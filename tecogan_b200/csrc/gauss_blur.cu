// The reference's HR -> LR inference input (lib/dataloader.py:38-43): cv2.GaussianBlur(frame, (0, 0), sigmaX=1.5)
// sampled at [::4, ::4] and divided by 255, on uint8 or uint16 RGB frames, bit for bit with cv2 4.13's float32 filter
// (DESIGN.md section 4.9; tests/golden/gauss_blur_oracle.py restates the arithmetic).  Only the sampled outputs are
// computed: the row pass runs at every 4th column for the rows the column pass of one tile of output rows needs, and
// neighbouring output rows share those row results through shared memory.
#include "teco_common.cuh"

namespace {

constexpr int kRadius = 6;
constexpr int kTileX = 32;                                   // output columns per block
constexpr int kTileY = 16;                                   // output rows per block
constexpr int kRows = 4 * (kTileY - 1) + 2 * kRadius + 1;    // HR rows the tile's column pass reads: 73
constexpr int kCols = 3 * kTileX;                            // row-pass results per HR row: 96 floats
constexpr int kThreads = 256;

// cv2.getGaussianKernel(13, 1.5, CV_32F)
__constant__ float kTap[2 * kRadius + 1] = {
    0x1.763864p-14f, 0x1.0d891ap-10f, 0x1.f1e742p-8f, 0x1.26dd9ep-5f, 0x1.bfdc88p-4f, 0x1.b42852p-3f, 0x1.1058fp-2f,
    0x1.b42852p-3f,  0x1.bfdc88p-4f,  0x1.26dd9ep-5f, 0x1.f1e742p-8f, 0x1.0d891ap-10f, 0x1.763864p-14f};

// cv2::borderInterpolate(p, n, BORDER_REFLECT_101) for n >= 2: the reflection repeats until p is inside.
__device__ __forceinline__ int reflect101(int p, int n) {
  while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

// One block per (32 output columns, 16 output rows, frame).  frames[n] is the device address of frame n, a packed
// [H, W, 3] RGB array of T.  The fused/unfused choice follows element e = 3x + (2 - c) of cv2's BGR row of 3W floats:
// the row pass fuses on its 8-wide body plus one 4-wide step, the column pass on its 8-wide body only.
template <typename T>
__global__ void __launch_bounds__(kThreads) gauss_blur_down4_kernel(const int64_t* __restrict__ frames, int H, int W,
                                                                    float* __restrict__ out) {
  __shared__ float rows[kRows][kCols];
  const int h = (H + 3) / 4, w = (W + 3) / 4;
  const int ox0 = blockIdx.x * kTileX, oy0 = blockIdx.y * kTileY, n = blockIdx.z;
  const int tw = min(kTileX, w - ox0), th = min(kTileY, h - oy0);
  const int nrows = 4 * (th - 1) + 2 * kRadius + 1;
  const int nf = 3 * W;
  const int row_fused = 8 * (nf / 8) + (nf % 8 >= 4 ? 4 : 0), col_fused = 8 * (nf / 8);
  const T* src = reinterpret_cast<const T*>(frames[n]);

  // Row pass: local row j holds HR row 4*oy0 - 6 + j, reflected into the frame.
  for (int i = threadIdx.x; i < nrows * kCols; i += kThreads) {
    const int j = i / kCols, q = i - j * kCols, lx = q / 3, c = q - 3 * lx;
    if (lx >= tw) continue;
    const int X = 4 * (ox0 + lx);
    const T* row = src + (int64_t)reflect101(4 * oy0 - kRadius + j, H) * nf + c;
    const bool fused = 3 * X + 2 - c < row_fused;
    float s = 0.f;
#pragma unroll
    for (int t = 0; t <= 2 * kRadius; ++t) {
      const float x = (float)row[3 * reflect101(X + t - kRadius, W)];
      s = fused ? fmaf(kTap[t], x, s) : __fadd_rn(__fmul_rn(kTap[t], x), s);
    }
    rows[j][q] = s;
  }
  __syncthreads();

  // Column pass, symmetric: the centre tap, then each pair of rows summed first.
  for (int i = threadIdx.x; i < th * kCols; i += kThreads) {
    const int j = i / kCols, q = i - j * kCols, lx = q / 3, c = q - 3 * lx;
    if (lx >= tw) continue;
    const bool fused = 3 * 4 * (ox0 + lx) + 2 - c < col_fused;
    const int m = 4 * j + kRadius;
    float acc = __fmul_rn(kTap[kRadius], rows[m][q]);
#pragma unroll
    for (int t = 1; t <= kRadius; ++t) {
      const float pair = __fadd_rn(rows[m + t][q], rows[m - t][q]);
      acc = fused ? fmaf(kTap[kRadius + t], pair, acc) : __fadd_rn(__fmul_rn(kTap[kRadius + t], pair), acc);
    }
    // __fdiv_rn: numpy's correctly rounded float32 division, whatever -use_fast_math or -prec-div say
    out[(((int64_t)n * h + oy0 + j) * w + ox0 + lx) * 3 + c] = __fdiv_rn(acc, 255.0f);
  }
}

}  // namespace

extern "C" int teco_gauss_blur_down4(const int64_t* frames, int32_t bits, int32_t N, int32_t H, int32_t W, float* out,
                                     void* stream) {
  TECO_CHECK_ARG(frames && out, "teco_gauss_blur_down4: NULL pointer");
  TECO_CHECK_ARG(bits == 8 || bits == 16, "teco_gauss_blur_down4: bits must be 8 or 16 (got %d)", bits);
  TECO_CHECK_ARG(N > 0 && N <= 65535, "teco_gauss_blur_down4: need 0 < N <= 65535 (got %d)", N);
  TECO_CHECK_ARG(H >= 2 && W >= 2 && H <= 65535 && W <= 65535,
                 "teco_gauss_blur_down4: frames need 2 <= H, W <= 65535 (got %dx%d); cv2's blur of a 1-pixel side is "
                 "not reproduced", H, W);
  const dim3 grid((unsigned)((W + 3) / 4 + kTileX - 1) / kTileX, (unsigned)((H + 3) / 4 + kTileY - 1) / kTileY,
                  (unsigned)N);
  if (bits == 8)
    gauss_blur_down4_kernel<uint8_t><<<grid, kThreads, 0, (cudaStream_t)stream>>>(frames, H, W, out);
  else
    gauss_blur_down4_kernel<uint16_t><<<grid, kThreads, 0, (cudaStream_t)stream>>>(frames, H, W, out);
  TECO_CUDA_LAUNCH_CHECK("teco_gauss_blur_down4");
  return TECO_OK;
}
