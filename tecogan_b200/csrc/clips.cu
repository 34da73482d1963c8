// Frames to float32: the pixel half of HRClipLoader.sample() -- crop, left-right flip, convert_image_dtype -- on the GPU
// for training clips cut from the device-resident frame store (tecogan_b200/lib/dataloader.py::FrameStore), and the
// reference's `frame / 255` of LR inference input (lib/dataloader.py:38-43).  The draws (which frames, where, whether
// flipped) are made on the host and arrive as one table row per output frame.
#include "teco_common.cuh"

namespace {

// One block per (output row, output frame).  Row y of output frame n reads Sw pixels of one source row, mirrored when
// flip != 0, and writes them as 3*Sw contiguous floats.  With cols == 3 the table rows are {byte offset from base,
// row pitch in elements of T, flip}; with cols == 1 they are the byte offsets from base of packed, unflipped frames.
// __fdiv_rn: the correctly rounded quotient, which is what numpy's float32 division of the host path computes, whatever
// -use_fast_math or -prec-div say.
template <typename T>
__global__ void gather_rgb_kernel(uintptr_t base, const int64_t* __restrict__ table, int cols, int Sh, int Sw,
                                  float* __restrict__ out) {
  const int y = blockIdx.x, n = blockIdx.y;
  const int64_t src0 = table[cols * n], pitch = cols == 3 ? table[3 * n + 1] : 3 * (int64_t)Sw;
  const bool flip = cols == 3 && table[3 * n + 2] != 0;
  const T* row = reinterpret_cast<const T*>(base + (uintptr_t)src0) + (int64_t)y * pitch;
  float* dst = out + ((int64_t)n * Sh + y) * (int64_t)Sw * 3;
  for (int e = threadIdx.x; e < 3 * Sw; e += blockDim.x) {
    const int x = e / 3, c = e - 3 * x;
    const int sx = flip ? Sw - 1 - x : x;
    dst[e] = __fdiv_rn((float)row[3 * sx + c], 255.0f);
  }
}

// The same windows as gather_rgb_kernel<uint8_t> with cols == 3, read from host memory mapped into the device's address
// space (cudaHostRegister + cudaHostGetDevicePointer), where every load is a read request over PCIe.  One block per
// output window.  A row is cut into segments of at most kHostSegPixels pixels; the 16-byte-aligned span covering a
// segment's bytes is at most 32 uint4 (3 * 160 + 15 <= 512), so one warp reads it in one instruction.  Each warp issues
// the spans of kHostRows segments before it consumes any, stages them in shared memory, and writes each segment's
// 3 * len contiguous output floats as aligned float4 stores (scalar head and tail).  A flipped segment reads the
// mirrored source range and reverses it in shared memory.
constexpr int kHostWarps = 8, kHostRows = 4, kHostSegPixels = 160;

__global__ void __launch_bounds__(kHostWarps * 32) gather_clips_host_kernel(uintptr_t base,
                                                                            const int64_t* __restrict__ table, int S,
                                                                            float* __restrict__ out) {
  __shared__ __align__(16) uint8_t stage[kHostWarps][kHostRows][512];
  const int n = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t src0 = table[3 * n], pitch = table[3 * n + 1];
  const bool flip = table[3 * n + 2] != 0;
  const int nseg = (S + kHostSegPixels - 1) / kHostSegPixels;
  const int64_t items = (int64_t)S * nseg;
  float* const win = out + (int64_t)n * S * S * 3;
  for (int64_t i0 = (int64_t)warp * kHostRows; i0 < items; i0 += kHostWarps * kHostRows) {
    uint4 v[kHostRows];
#pragma unroll
    for (int r = 0; r < kHostRows; ++r) {
      const int64_t it = i0 + r;
      if (it < items) {
        const int y = (int)(it / nseg), x0 = (int)(it % nseg) * kHostSegPixels, len = min(kHostSegPixels, S - x0);
        const uintptr_t g = base + (uintptr_t)(src0 + (int64_t)y * pitch + 3 * (flip ? S - x0 - len : x0));
        const uintptr_t a = g & ~(uintptr_t)15;
        if (lane < (int)((g - a + 3 * len + 15) >> 4)) v[r] = __ldg(reinterpret_cast<const uint4*>(a) + lane);
      }
    }
#pragma unroll
    for (int r = 0; r < kHostRows; ++r) {
      const int64_t it = i0 + r;
      if (it < items) {
        const int y = (int)(it / nseg), x0 = (int)(it % nseg) * kHostSegPixels, len = min(kHostSegPixels, S - x0);
        const uintptr_t g = base + (uintptr_t)(src0 + (int64_t)y * pitch + 3 * (flip ? S - x0 - len : x0));
        if (lane < (int)((g - (g & ~(uintptr_t)15) + 3 * len + 15) >> 4))
          *reinterpret_cast<uint4*>(&stage[warp][r][16 * lane]) = v[r];
      }
    }
    __syncwarp();
    for (int r = 0; r < kHostRows; ++r) {
      const int64_t it = i0 + r;
      if (it >= items) break;
      const int y = (int)(it / nseg), x0 = (int)(it % nseg) * kHostSegPixels, len = min(kHostSegPixels, S - x0);
      const uintptr_t g = base + (uintptr_t)(src0 + (int64_t)y * pitch + 3 * (flip ? S - x0 - len : x0));
      const uint8_t* sm = &stage[warp][r][g & 15];
      float* d = win + ((int64_t)y * S + x0) * 3;
      const int m = 3 * len;
      auto val = [&](int e) {
        const int px = e / 3, c = e - 3 * px;
        return __fdiv_rn((float)sm[3 * (flip ? len - 1 - px : px) + c], 255.0f);
      };
      const int head = min(m, (int)((0u - (unsigned)(uintptr_t)d) >> 2 & 3u));   // floats before a 16-byte boundary
      const int nv = (m - head) >> 2, tail = head + 4 * nv;
      if (lane < head) d[lane] = val(lane);
      for (int j = lane; j < nv; j += 32) {
        const int e = head + 4 * j;
        *reinterpret_cast<float4*>(d + e) = make_float4(val(e), val(e + 1), val(e + 2), val(e + 3));
      }
      if (lane < m - tail) d[tail + lane] = val(tail + lane);
    }
    __syncwarp();
  }
}

}  // namespace

extern "C" int teco_gather_clips_host_u8(uint64_t store_dev_addr, const int64_t* table, int32_t n, int32_t S,
                                         float* out, void* stream) {
  TECO_CHECK_ARG(store_dev_addr && table && out, "teco_gather_clips_host_u8: NULL pointer");
  TECO_CHECK_ARG(n > 0 && n <= 65535 && S > 0, "teco_gather_clips_host_u8: need 0 < n <= 65535 and S > 0 (got n=%d, S=%d)",
                 n, S);
  gather_clips_host_kernel<<<(unsigned)n, kHostWarps * 32, 0, (cudaStream_t)stream>>>((uintptr_t)store_dev_addr, table,
                                                                                      S, out);
  TECO_CUDA_LAUNCH_CHECK("teco_gather_clips_host_u8");
  return TECO_OK;
}

extern "C" int teco_gather_clips_u8(const uint8_t* store, const int64_t* table, int32_t n, int32_t S, float* out,
                                    void* stream) {
  TECO_CHECK_ARG(store && table && out, "teco_gather_clips_u8: NULL pointer");
  TECO_CHECK_ARG(n > 0 && n <= 65535 && S > 0, "teco_gather_clips_u8: need 0 < n <= 65535 and S > 0 (got n=%d, S=%d)", n, S);
  gather_rgb_kernel<uint8_t><<<dim3((unsigned)S, (unsigned)n), 128, 0, (cudaStream_t)stream>>>((uintptr_t)store, table,
                                                                                               3, S, S, out);
  TECO_CUDA_LAUNCH_CHECK("teco_gather_clips_u8");
  return TECO_OK;
}

extern "C" int teco_frames_to_f32(const int64_t* frames, int32_t bits, int32_t N, int32_t H, int32_t W, float* out,
                                  void* stream) {
  TECO_CHECK_ARG(frames && out, "teco_frames_to_f32: NULL pointer");
  TECO_CHECK_ARG(bits == 8 || bits == 16, "teco_frames_to_f32: bits must be 8 or 16 (got %d)", bits);
  TECO_CHECK_ARG(N > 0 && N <= 65535 && H > 0 && W > 0, "teco_frames_to_f32: need 0 < N <= 65535 and H, W > 0 "
                 "(got N=%d, %dx%d)", N, H, W);
  const dim3 grid((unsigned)H, (unsigned)N);
  if (bits == 8)
    gather_rgb_kernel<uint8_t><<<grid, 128, 0, (cudaStream_t)stream>>>(0, frames, 1, H, W, out);
  else
    gather_rgb_kernel<uint16_t><<<grid, 128, 0, (cudaStream_t)stream>>>(0, frames, 1, H, W, out);
  TECO_CUDA_LAUNCH_CHECK("teco_frames_to_f32");
  return TECO_OK;
}
