// The reference's training-frame down-sample (lib/data/video.py:168-173): cv2.resize(frame, (0, 0), fx=0.5, fy=0.5,
// interpolation=INTER_AREA) on uint8 3-channel frames, bit for bit with cv2 4.13 (DESIGN.md section 4.10;
// tests/golden/area_oracle.py restates it).  The scale is exactly 2 on both axes whatever the parity of H and W, so cv2
// runs its integer-scale path on every size: an output whose 2 x 2 block lies inside the frame is (a + b + c + d + 2) >> 2;
// the extra last row (H = 4k + 3) or column (W = 4k + 3) averages the 2 sources it has, or takes the 1 at the corner,
// rounding half to even.  Integer arithmetic throughout: there is no float to round differently.
#include "teco_common.cuh"

namespace {

constexpr int kThreads = 256;

// cvRound(n * 0.5): halves to even.
__host__ __device__ __forceinline__ int half_size(int n) {
  const int k = n >> 1;
  return (n & 1) ? k + (k & 1) : k;
}

// cvRound(p / 2.0f) for an integer p >= 0: halves to even.
__device__ __forceinline__ int avg2_even(int p) { return (p + ((p >> 1) & 1)) >> 1; }

// One thread per output pixel; block (x: 256 output columns, y: output row, z: frame).  frames[n] is the device address
// of frame n, a packed [H, W, 3] uint8 array.  swap_rb stores channel 2 - c at c (BGR in, RGB out).
__global__ void __launch_bounds__(kThreads) area_half_u8_kernel(const int64_t* __restrict__ frames, int H, int W,
                                                               int oh, int ow, int swap_rb, uint8_t* __restrict__ out) {
  const int ox = blockIdx.x * kThreads + threadIdx.x, oy = blockIdx.y, n = blockIdx.z;
  if (ox >= ow) return;
  const uint8_t* src = reinterpret_cast<const uint8_t*>(frames[n]);
  const int64_t pitch = 3 * (int64_t)W;
  const bool row_in = oy < (H >> 1), col_in = ox < (W >> 1);
  const int y0 = row_in ? 2 * oy : H - 1, x0 = col_in ? 2 * ox : W - 1;
  const uint8_t* p0 = src + y0 * pitch + 3 * (int64_t)x0;
  const uint8_t* p1 = p0 + (row_in ? pitch : 0);          // second row, or the first again on the last row
  const int dx = col_in ? 3 : 0;                          // second column, or the first again on the last column
  int v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (row_in && col_in) {
      v[c] = (__ldg(p0 + c) + __ldg(p0 + dx + c) + __ldg(p1 + c) + __ldg(p1 + dx + c) + 2) >> 2;
    } else if (row_in || col_in) {
      v[c] = avg2_even(__ldg(p0 + c) + (row_in ? __ldg(p1 + c) : __ldg(p0 + dx + c)));
    } else {
      v[c] = __ldg(p0 + c);
    }
  }
  uint8_t* o = out + (((int64_t)n * oh + oy) * ow + ox) * 3;
  o[0] = (uint8_t)v[swap_rb ? 2 : 0];
  o[1] = (uint8_t)v[1];
  o[2] = (uint8_t)v[swap_rb ? 0 : 2];
}

}  // namespace

extern "C" int teco_area_half_u8(const int64_t* frames, int32_t N, int32_t H, int32_t W, uint8_t* out, int32_t swap_rb,
                                 void* stream) {
  TECO_CHECK_ARG(frames && out, "teco_area_half_u8: NULL pointer");
  TECO_CHECK_ARG(N > 0 && N <= 65535, "teco_area_half_u8: need 0 < N <= 65535 (got %d)", N);
  TECO_CHECK_ARG(H >= 2 && W >= 2 && H <= 65535 && W <= 65535,
                 "teco_area_half_u8: frames need 2 <= H, W <= 65535 (got %dx%d)", H, W);
  const int oh = half_size(H), ow = half_size(W);
  const dim3 grid((unsigned)(ow + kThreads - 1) / kThreads, (unsigned)oh, (unsigned)N);
  area_half_u8_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(frames, H, W, oh, ow, swap_rb != 0, out);
  TECO_CUDA_LAUNCH_CHECK("teco_area_half_u8");
  return TECO_OK;
}
