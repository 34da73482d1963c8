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

}  // namespace

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
