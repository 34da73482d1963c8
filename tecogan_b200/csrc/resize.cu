// `main.py --outscale`: cv2.resize(frame, (W_out, H_out), interpolation=INTER_LANCZOS4) on a uint8 RGB frame, byte for
// byte with cv2 4.13's fixed-point path (DESIGN.md section 4.11; tests/golden/resize_oracle.py restates it).  The
// coefficients need libm's double sin / cos, so the host computes them once per (input size, output size)
// (tecogan_b200/resize.py) and the kernel does integer work only:
//   horizontal  h[r][x][c] = sum_j src[r][clamp(sx[x] - 3 + j)][c] * alpha[x][j]           (int32)
//   vertical    v[y][x][c] = sum_k beta[y][k] * h[clamp(sy[y] - 3 + k)][x][c]              (int32)
//   store       clamp((v + (1 << 21)) >> 22, 0, 255)
// Each axis table is int32 [n_out, 9]: the base index s, then the eight int16 weights widened to int32.
#include "teco_common.cuh"

namespace {

constexpr int kTileW = 64;              // output columns per tile
constexpr int kThreads = kTileW * 3;    // one thread per output byte of a tile row
constexpr int kMaxRows = 56;            // source rows of a tile's horizontal results in shared memory
constexpr int kMaxTileH = 64;
constexpr int kMaxDown = 4;             // H_in <= 4 H_out, W_in <= 4 W_out

// Output rows per tile for a vertical scale H_in / H_out: (th - 1) * scale + 10 <= kMaxRows.  A tile's source rows are
// sy[y0 + th - 1] + 4 - (sy[y0] - 3) + 1 <= floor((th - 1) * scale + float rounding) + 9, which leaves a row to spare;
// the kernel clamps the count to kMaxRows all the same, so a table that breaks the bound cannot overrun the buffer.
int tile_rows(int H_in, int H_out) {
  const double scale = (double)H_in / (double)H_out;
  const int th = (int)((kMaxRows - 10) / scale) + 1;
  return th < kMaxTileH ? th : kMaxTileH;
}

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// One CTA per tile of th output rows x kTileW output columns, the tiles taken grid-stride.  Thread t owns byte t of each
// tile row (column t / 3, channel t % 3): its eight taps and weights stay in registers through the tile.
__global__ void __launch_bounds__(kThreads, 4) resize_lanczos4_u8_kernel(
    const uint8_t* __restrict__ src, int64_t src_pitch, int H_in, int W_in, uint8_t* __restrict__ dst,
    int64_t dst_pitch, int H_out, int W_out, const int* __restrict__ xtab, const int* __restrict__ ytab, int th,
    int tiles_x, int ntiles) {
  __shared__ int hbuf[kMaxRows][kThreads];
  __shared__ int yrow[kMaxTileH][8];
  __shared__ int ycoef[kMaxTileH][8];
  const int t = threadIdx.x, xl = t / 3, c = t - 3 * xl;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int x0 = (tile % tiles_x) * kTileW, y0 = (tile / tiles_x) * th;
    const int nx = min(kTileW, W_out - x0), ny = min(th, H_out - y0);
    const bool live = xl < nx;
    const int lo = clampi(__ldg(ytab + (int64_t)y0 * 9) - 3, 0, H_in - 1);
    const int hi = clampi(__ldg(ytab + (int64_t)(y0 + ny - 1) * 9) + 4, 0, H_in - 1);
    const int nrows = clampi(hi - lo + 1, 1, kMaxRows);
    __syncthreads();                                     // the previous tile is done with yrow / hbuf
    for (int i = t; i < ny * 8; i += kThreads) {
      const int y = i >> 3, k = i & 7;
      const int* e = ytab + (int64_t)(y0 + y) * 9;
      yrow[y][k] = clampi(clampi(__ldg(e) - 3 + k, 0, H_in - 1) - lo, 0, nrows - 1);
      ycoef[y][k] = __ldg(e + 1 + k);
    }
    int off[8], alpha[8];
    if (live) {
      const int* e = xtab + (int64_t)(x0 + xl) * 9;
      const int sx = __ldg(e);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        off[j] = 3 * clampi(sx - 3 + j, 0, W_in - 1) + c;
        alpha[j] = __ldg(e + 1 + j);
      }
      const uint8_t* row = src + (int64_t)lo * src_pitch;
#pragma unroll 2   // two rows of loads in flight in 64 registers: four CTAs per SM, as shared memory allows
      for (int r = 0; r < nrows; ++r, row += src_pitch) {
        int acc = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += (int)__ldg(row + off[j]) * alpha[j];
        hbuf[r][t] = acc;
      }
    }
    __syncthreads();
    if (live) {
      uint8_t* out = dst + (int64_t)y0 * dst_pitch + 3 * (int64_t)x0 + t;
      for (int y = 0; y < ny; ++y, out += dst_pitch) {
        int acc = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) acc += ycoef[y][k] * hbuf[yrow[y][k]][t];
        *out = (uint8_t)clampi((acc + (1 << 21)) >> 22, 0, 255);
      }
    }
  }
}

}  // namespace

extern "C" int teco_resize_lanczos4_u8(const uint8_t* src, int64_t src_pitch, int32_t H_in, int32_t W_in, uint8_t* dst,
                                       int64_t dst_pitch, int32_t H_out, int32_t W_out, const int32_t* xtab,
                                       const int32_t* ytab, void* stream) {
  TECO_CHECK_ARG(src && dst && xtab && ytab, "teco_resize_lanczos4_u8: NULL pointer");
  TECO_CHECK_ARG(H_in >= 1 && W_in >= 1 && H_out >= 1 && W_out >= 1 && H_in <= 65535 && W_in <= 65535 &&
                     H_out <= 65535 && W_out <= 65535,
                 "teco_resize_lanczos4_u8: sides must be 1..65535 (got %dx%d -> %dx%d)", H_in, W_in, H_out, W_out);
  TECO_CHECK_ARG(H_in <= kMaxDown * H_out && W_in <= kMaxDown * W_out,
                 "teco_resize_lanczos4_u8: at most a 4x down-scale per axis (got %dx%d -> %dx%d)", H_in, W_in, H_out,
                 W_out);
  TECO_CHECK_ARG(src_pitch >= 3 * (int64_t)W_in && dst_pitch >= 3 * (int64_t)W_out,
                 "teco_resize_lanczos4_u8: row pitches %lld, %lld below 3 * width", (long long)src_pitch,
                 (long long)dst_pitch);
  const int th = tile_rows(H_in, H_out);
  const int tiles_x = teco_ceil_div(W_out, kTileW);
  const int ntiles = tiles_x * teco_ceil_div(H_out, th);
  static int per_sm = 0;
  if (per_sm == 0) TECO_CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, resize_lanczos4_u8_kernel,
                                                                                kThreads, 0));
  const int grid = min(ntiles, max(per_sm, 1) * teco_sm_count());
  resize_lanczos4_u8_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(src, src_pitch, H_in, W_in, dst, dst_pitch,
                                                                          H_out, W_out, xtab, ytab, th, tiles_x,
                                                                          ntiles);
  TECO_CUDA_LAUNCH_CHECK("teco_resize_lanczos4_u8");
  return TECO_OK;
}
