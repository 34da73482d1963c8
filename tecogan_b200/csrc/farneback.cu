// farneback.cu -- tOF of the reference's evaluation (metrics.py:143-169) on the device: cv2.cvtColor(RGB2GRAY) and
// cv2.calcOpticalFlowFarneback(prev, next, None, 0.5, 3, 15, 3, 5, 1.2, 0) broken into its stages, each batched over
// frames or frame pairs, and the per-pair tOF reduction.  The stages and their arithmetic follow Farneback (2003) and the
// black-box probes of cv2 4.13 recorded in DESIGN.md section 4.4.  Only the reference's parameters exist here.
//
// Everything that cv2 keeps in float Mats is fp32 and is evaluated one correctly rounded operation at a time (explicit
// __f*_rn intrinsics: no FMA contraction), so each stage reproduces the host restatement tests/golden/farneback_oracle.py
// operation for operation.  Where cv2 sums in double -- the horizontal half of the polynomial expansion, the 15x15 box
// filter and the 2x2 solve -- this does too: the solve divides by g11 g22 - g12^2 + 1e-3, which cancels badly in fp32.
#include <cmath>

#include "teco_common.cuh"

namespace {
constexpr int TPB = 256;
constexpr int POLY_N = 5;                       // poly_n = 5: taps -5 .. 5
constexpr int MAX_TAPS = 19;                    // Gaussian of the coarsest level (sigma 3.5): cvRound(17.5) | 1 = 19
constexpr int WIN_R = 7;                        // winsize 15
constexpr int MAX_PAIRS = 256;                  // frame pairs per teco_farneback_iterate_f32 launch
constexpr int MAX_LEVEL = 3;                    // levels = 3
constexpr int RED_CHUNKS = 32;                  // row chunks per pair of teco_tof_reduce_f32

// Polyexp tile: 32 x 8 outputs, 5-pixel halo on each side.
constexpr int PX = 32, PY = 8, PHX = PX + 2 * POLY_N, PHY = PY + 2 * POLY_N;
// Iteration tile: 32 x 16 outputs, 7-pixel halo (the box filter) on each side.
constexpr int IX = 32, IY = 16, IHX = IX + 2 * WIN_R, IHY = IY + 2 * WIN_R;
constexpr size_t ITER_SMEM = 5 * (size_t)IHY * IHX * sizeof(float) + 5 * (size_t)IY * IHX * sizeof(double);

struct GaussTaps {
  float k[MAX_TAPS];
  int r;
};
struct PolyTaps {
  float g[POLY_N + 1], xg[POLY_N + 1], xxg[POLY_N + 1];
  double ig11, ig03, ig33, ig55;
};
struct PairIdx {
  int32_t a[MAX_PAIRS], b[MAX_PAIRS];
};

__device__ __forceinline__ float fadd(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fmul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }
__device__ __forceinline__ int reflect101(int i, int n) {
  if (n == 1) return 0;
  i = i < 0 ? -i : i;
  return i >= n ? 2 * (n - 1) - i : i;
}

// INTER_LINEAR source index pair and weight of destination index d (half-pixel centres, clamp at both ends):
// f = float((d + 0.5) * (1 / (dst / src)) - 0.5), s = floor(f), f -= s; s < 0 or s >= src - 1 -> weight 0 on s.
__device__ __forceinline__ void linear_coeff(int d, int src, int dst, int& s0, int& s1, float& f) {
  const double scale = 1.0 / ((double)dst / (double)src);
  f = (float)((d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f = fsub(f, (float)s);
  if (s < 0) f = 0.f, s = 0;
  if (s >= src - 1) f = 0.f, s = src - 1;
  s0 = s;
  s1 = min(s + 1, src - 1);
}

// ---- RGB -> grey ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TPB) grey_kernel(const uint8_t* __restrict__ img, int H, int W, int y0, int x0, int h,
                                                   int w, long long total, uint8_t* __restrict__ g) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int col = (int)(i % w);
    const long long t = i / w;
    const int row = (int)(t % h);
    const long long n = t / h;
    const uint8_t* p = img + ((n * H + y0 + row) * W + x0 + col) * 3;
    g[i] = (uint8_t)((9798 * p[0] + 19235 * p[1] + 3735 * p[2] + 16384) >> 15);
  }
}

// ---- pyramid level -------------------------------------------------------------------------------------------------
// Gaussian of the full-resolution grey image at (y, x): horizontal then vertical symmetric pass with reflect-101
// borders, each k_0 v_0 then += k_j (v_-j + v_j), in fp32.
__device__ __noinline__ float blurred_at(const uint8_t* __restrict__ img, int H, int W, int y, int x,
                                         const float* __restrict__ k, int r) {
  auto row = [&](int yy) {
    const uint8_t* p = img + (size_t)yy * W;
    float s = fmul(k[r], (float)p[x]);
    for (int j = 1; j <= r; ++j)
      s = fadd(s, fmul(k[r + j], fadd((float)p[reflect101(x - j, W)], (float)p[reflect101(x + j, W)])));
    return s;
  };
  float s = fmul(k[r], row(y));
  for (int j = 1; j <= r; ++j) s = fadd(s, fmul(k[r + j], fadd(row(reflect101(y - j, H)), row(reflect101(y + j, H)))));
  return s;
}

__global__ void __launch_bounds__(TPB) pyramid_kernel(const uint8_t* __restrict__ grey, int H, int W, int lh, int lw,
                                                      long long total, const GaussTaps gk, float* __restrict__ out) {
  __shared__ float k[MAX_TAPS];                  // taps in shared memory: indexing the parameter struct would copy it to the stack
  if (threadIdx.x < MAX_TAPS) k[threadIdx.x] = gk.k[threadIdx.x];
  __syncthreads();
  const int r = gk.r;
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int x = (int)(i % lw);
    const long long t = i / lw;
    const int y = (int)(t % lh);
    const uint8_t* img = grey + (size_t)(t / lh) * H * W;
    float v;
    if (lh == H && lw == W) {
      v = blurred_at(img, H, W, y, x, k, r);                                 // same size: resize is a copy
    } else if (H == 2 * lh && W == 2 * lw) {                               // exact halving: cv2's fast area path
      const float a = blurred_at(img, H, W, 2 * y, 2 * x, k, r), b = blurred_at(img, H, W, 2 * y, 2 * x + 1, k, r);
      const float c = blurred_at(img, H, W, 2 * y + 1, 2 * x, k, r), d = blurred_at(img, H, W, 2 * y + 1, 2 * x + 1, k, r);
      v = fmul(fadd(fadd(fadd(a, b), c), d), 0.25f);
    } else {
      int sx0, sx1, sy0, sy1;
      float fx, fy;
      linear_coeff(x, W, lw, sx0, sx1, fx);
      linear_coeff(y, H, lh, sy0, sy1, fy);
      const float r0 = fadd(fmul(blurred_at(img, H, W, sy0, sx0, k, r), 1.f - fx), fmul(blurred_at(img, H, W, sy0, sx1, k, r), fx));
      const float r1 = fadd(fmul(blurred_at(img, H, W, sy1, sx0, k, r), 1.f - fx), fmul(blurred_at(img, H, W, sy1, sx1, k, r), fx));
      v = fadd(fmul(r0, 1.f - fy), fmul(r1, fy));
    }
    out[i] = v;
  }
}

// ---- polynomial expansion ------------------------------------------------------------------------------------------
// One CTA per 32 x 8 tile of one image: the tile and its 5-pixel halo (rows / columns clamped) in shared memory, the
// vertical 11-tap pass (1, y, y^2 weights) in fp32 over the halo width, the horizontal pass in float64 per output.
// Output channels: y, x, yy, xx, xy coefficients.
__global__ void __launch_bounds__(TPB) polyexp_kernel(const float* __restrict__ src, int h, int w, const PolyTaps pt,
                                                      float* __restrict__ dst) {
  __shared__ float tile[PHY][PHX];
  __shared__ float vp[3][PY][PHX];
  const int n = blockIdx.z, tx0 = blockIdx.x * PX, ty0 = blockIdx.y * PY;
  const float* img = src + (size_t)n * h * w;
  for (int i = threadIdx.x; i < PHY * PHX; i += TPB) {
    const int r = i / PHX, c = i % PHX;
    tile[r][c] = img[(size_t)clampi(ty0 - POLY_N + r, 0, h - 1) * w + clampi(tx0 - POLY_N + c, 0, w - 1)];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < PY * PHX; i += TPB) {
    const int r = i / PHX, c = i % PHX;
    const float centre = tile[r + POLY_N][c];
    float v0 = fmul(centre, pt.g[0]), v1 = 0.f, v2 = 0.f;
#pragma unroll
    for (int k = 1; k <= POLY_N; ++k) {
      const float lo = tile[r + POLY_N - k][c], hi = tile[r + POLY_N + k][c];
      const float p = fadd(lo, hi);
      v0 = fadd(v0, fmul(pt.g[k], p));
      v1 = fadd(v1, fmul(pt.xg[k], fsub(hi, lo)));
      v2 = fadd(v2, fmul(pt.xxg[k], p));
    }
    vp[0][r][c] = v0;
    vp[1][r][c] = v1;
    vp[2][r][c] = v2;
  }
  __syncthreads();
  const int r = threadIdx.x / PX, c = threadIdx.x % PX;
  const int y = ty0 + r, x = tx0 + c;
  if (y >= h || x >= w) return;
  const int cc = c + POLY_N;
  const double g0 = pt.g[0];
  double b1 = dmul(vp[0][r][cc], g0), b2 = 0.0, b3 = dmul(vp[1][r][cc], g0), b4 = 0.0, b5 = dmul(vp[2][r][cc], g0), b6 = 0.0;
#pragma unroll
  for (int k = 1; k <= POLY_N; ++k) {
    // columns beyond the image: the tile loaded clamped columns, whose vertical sums are the edge column's
    const double l0 = vp[0][r][cc - k], r0 = vp[0][r][cc + k], l1 = vp[1][r][cc - k], r1 = vp[1][r][cc + k];
    const double l2 = vp[2][r][cc - k], r2 = vp[2][r][cc + k];
    const double g = pt.g[k], xg = pt.xg[k], xxg = pt.xxg[k];
    const double tg = dadd(r0, l0);
    b1 = dadd(b1, dmul(tg, g));
    b4 = dadd(b4, dmul(tg, xxg));
    b2 = dadd(b2, dmul(dsub(r0, l0), xg));
    b3 = dadd(b3, dmul(dadd(r1, l1), g));
    b6 = dadd(b6, dmul(dsub(r1, l1), xg));
    b5 = dadd(b5, dmul(dadd(r2, l2), g));
  }
  float* o = dst + (((size_t)n * h + y) * w + x) * 5;
  o[0] = (float)dmul(b3, pt.ig11);
  o[1] = (float)dmul(b2, pt.ig11);
  o[2] = (float)dadd(dmul(b1, pt.ig03), dmul(b5, pt.ig33));
  o[3] = (float)dadd(dmul(b1, pt.ig03), dmul(b4, pt.ig33));
  o[4] = (float)dmul(b6, pt.ig55);
}

// ---- one update iteration ------------------------------------------------------------------------------------------
__device__ __forceinline__ float border_weight(int i) {
  return i == 0 || i == 1 ? 0.14f : 0.4472f;
}

// The 5-term field (G11, G12, G22, h1, h2) at pixel (x, y) of a pair, from R0 (first frame), R1 (second frame) sampled
// bilinearly at (x, y) + flow, and the border weights -- fp32, one rounded operation at a time.
__device__ __forceinline__ void field_at(const float* __restrict__ R0, const float* __restrict__ R1,
                                         const float* __restrict__ flow, int h, int w, int x, int y, float m[5]) {
  const float* r0 = R0 + ((size_t)y * w + x) * 5;
  float dx = 0.f, dy = 0.f;
  if (flow) {
    dx = flow[((size_t)y * w + x) * 2];
    dy = flow[((size_t)y * w + x) * 2 + 1];
  }
  float fx = fadd((float)x, dx), fy = fadd((float)y, dy);
  const int x1 = (int)floorf(fx), y1 = (int)floorf(fy);
  fx = fsub(fx, (float)x1);
  fy = fsub(fy, (float)y1);
  float r2, r3, r4, r5, r6;
  if ((unsigned)x1 < (unsigned)(w - 1) && (unsigned)y1 < (unsigned)(h - 1)) {
    const float a00 = fmul(1.f - fx, 1.f - fy), a01 = fmul(fx, 1.f - fy), a10 = fmul(1.f - fx, fy), a11 = fmul(fx, fy);
    const float* p = R1 + ((size_t)y1 * w + x1) * 5;
    const float* q = p + (size_t)w * 5;
    float s[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) s[c] = fadd(fadd(fadd(fmul(a00, p[c]), fmul(a01, p[5 + c])), fmul(a10, q[c])), fmul(a11, q[5 + c]));
    r2 = s[0];
    r3 = s[1];
    r4 = fmul(fadd(r0[2], s[2]), 0.5f);
    r5 = fmul(fadd(r0[3], s[3]), 0.5f);
    r6 = fmul(fadd(r0[4], s[4]), 0.25f);
  } else {                                       // the sample square leaves the frame: R0 alone
    r2 = r3 = 0.f;
    r4 = r0[2];
    r5 = r0[3];
    r6 = fmul(r0[4], 0.5f);
  }
  r2 = fmul(fsub(r0[0], r2), 0.5f);
  r3 = fmul(fsub(r0[1], r3), 0.5f);
  r2 = fadd(r2, fadd(fmul(r4, dy), fmul(r6, dx)));
  r3 = fadd(r3, fadd(fmul(r6, dy), fmul(r5, dx)));
  if (x < 5 || x >= w - 5 || y < 5 || y >= h - 5) {
    const float sc = fmul(fmul(fmul(x < 5 ? border_weight(x) : 1.f, x >= w - 5 ? border_weight(w - 1 - x) : 1.f),
                               y < 5 ? border_weight(y) : 1.f),
                          y >= h - 5 ? border_weight(h - 1 - y) : 1.f);
    r2 = fmul(r2, sc);
    r3 = fmul(r3, sc);
    r4 = fmul(r4, sc);
    r5 = fmul(r5, sc);
    r6 = fmul(r6, sc);
  }
  m[0] = fadd(fmul(r4, r4), fmul(r6, r6));
  m[1] = fmul(fadd(r4, r5), r6);
  m[2] = fadd(fmul(r5, r5), fmul(r6, r6));
  m[3] = fadd(fmul(r4, r2), fmul(r6, r3));
  m[4] = fadd(fmul(r6, r2), fmul(r5, r3));
}

// One CTA per 32 x 16 tile of one pair.  The field of the tile and its 7-pixel halo (rows / columns clamped, i.e. the
// box filter's replicated border) is computed straight into shared memory, so it never reaches global memory; the 15-row
// sums (float64) go to shared memory as well, and each output pixel finishes its 15-column sums and solves
//   flow = (g11 h2 - g12 h1, g22 h1 - g12 h2) / (g11 g22 - g12^2 + 1e-3)      (g, h = box means)
// in float64.  flow_in == NULL is the zero flow of the coarsest level.  flow_out must not alias flow_in.
__global__ void __launch_bounds__(TPB) iterate_kernel(const float* __restrict__ R, int h, int w, const PairIdx pi,
                                                      const float* __restrict__ flow_in, float* __restrict__ flow_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  double* vs = reinterpret_cast<double*>(smem_raw);                        // [5][IY][IHX]
  float* ms = reinterpret_cast<float*>(vs + 5 * IY * IHX);                 // [5][IHY][IHX]
  const int p = blockIdx.z, tx0 = blockIdx.x * IX, ty0 = blockIdx.y * IY;
  const size_t plane = (size_t)h * w;
  const float* R0 = R + (size_t)pi.a[p] * plane * 5;
  const float* R1 = R + (size_t)pi.b[p] * plane * 5;
  const float* fin = flow_in ? flow_in + (size_t)p * plane * 2 : nullptr;
  for (int i = threadIdx.x; i < IHY * IHX; i += TPB) {
    const int r = i / IHX, c = i % IHX;
    float m[5];
    field_at(R0, R1, fin, h, w, clampi(tx0 - WIN_R + c, 0, w - 1), clampi(ty0 - WIN_R + r, 0, h - 1), m);
#pragma unroll
    for (int k = 0; k < 5; ++k) ms[(k * IHY + r) * IHX + c] = m[k];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 5 * IY * IHX; i += TPB) {
    const int k = i / (IY * IHX), rc = i % (IY * IHX), r = rc / IHX, c = rc % IHX;
    const float* col = ms + (k * IHY + r) * IHX + c;
    double s = 0.0;
#pragma unroll
    for (int d = 0; d < 2 * WIN_R + 1; ++d) s = dadd(s, (double)col[d * IHX]);
    vs[i] = s;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < IY * IX; i += TPB) {
    const int r = i / IX, c = i % IX;
    const int y = ty0 + r, x = tx0 + c;
    if (y >= h || x >= w) continue;
    double g[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      const double* row = vs + (k * IY + r) * IHX + c;
      double s = 0.0;
#pragma unroll
      for (int d = 0; d < 2 * WIN_R + 1; ++d) s = dadd(s, row[d]);
      g[k] = dmul(s, 1.0 / 225.0);
    }
    const double idet = 1.0 / dadd(dsub(dmul(g[0], g[2]), dmul(g[1], g[1])), 1e-3);
    float* o = flow_out + ((size_t)p * plane + (size_t)y * w + x) * 2;
    o[0] = (float)dmul(dsub(dmul(g[0], g[4]), dmul(g[1], g[3])), idet);
    o[1] = (float)dmul(dsub(dmul(g[2], g[3]), dmul(g[1], g[4])), idet);
  }
}

// ---- flow to the next level ----------------------------------------------------------------------------------------
__global__ void __launch_bounds__(TPB) flow_up_kernel(const float* __restrict__ src, int sh, int sw, int h, int w,
                                                      long long total, float* __restrict__ dst) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int x = (int)(i % w);
    const long long t = i / w;
    const int y = (int)(t % h);
    const float* f = src + (size_t)(t / h) * sh * sw * 2;
    int sx0, sx1, sy0, sy1;
    float fx, fy;
    linear_coeff(x, sw, w, sx0, sx1, fx);
    linear_coeff(y, sh, h, sy0, sy1, fy);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float r0 = fadd(fmul(f[((size_t)sy0 * sw + sx0) * 2 + c], 1.f - fx), fmul(f[((size_t)sy0 * sw + sx1) * 2 + c], fx));
      const float r1 = fadd(fmul(f[((size_t)sy1 * sw + sx0) * 2 + c], 1.f - fx), fmul(f[((size_t)sy1 * sw + sx1) * 2 + c], fx));
      dst[i * 2 + c] = fmul(fadd(fmul(r0, 1.f - fy), fmul(r1, fy)), 2.f);   // x 1 / pyr_scale
    }
  }
}

// ---- tOF reduction -------------------------------------------------------------------------------------------------
// CTA (chunk, pair) sums rows chunk, chunk + RED_CHUNKS, ... of the window in float64 with a fixed-shape tree; a second
// kernel adds the chunks of each pair in order.  No atomics: the result is the same on every run.
__global__ void __launch_bounds__(TPB) tof_partial_kernel(const float* __restrict__ fa, const float* __restrict__ fb, int H,
                                                          int W, int y0, int x0, int h, int w, double* __restrict__ part) {
  const int p = blockIdx.y;
  const float* A = fa + (size_t)p * H * W * 2;
  const float* B = fb + (size_t)p * H * W * 2;
  double acc = 0.0;
  for (int r = blockIdx.x; r < h; r += RED_CHUNKS)
    for (int c = threadIdx.x; c < w; c += TPB) {
      const size_t o = ((size_t)(y0 + r) * W + x0 + c) * 2;
      const float dx = fabsf(fsub(A[o], B[o])), dy = fabsf(fsub(A[o + 1], B[o + 1]));
      acc += (double)__fsqrt_rn(fadd(fmul(dx, dx), fmul(dy, dy)));
    }
  __shared__ double red[TPB];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = TPB / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[(size_t)p * RED_CHUNKS + blockIdx.x] = red[0];
}

__global__ void tof_finish_kernel(const double* __restrict__ part, int P, double inv_n, double* __restrict__ out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  double s = 0.0;
  for (int c = 0; c < RED_CHUNKS; ++c) s += part[(size_t)p * RED_CHUNKS + c];
  out[p] = s * inv_n;
}

int grid_for(long long total) {
  return (int)max(1LL, min((total + TPB - 1) / TPB, (long long)(16 * teco_sm_count())));
}

bool level_size(int H, int W, int level, int& lh, int& lw) {
  const double scale = std::ldexp(1.0, -level);
  lh = (int)std::lrint(H * scale);               // cvRound: half to even
  lw = (int)std::lrint(W * scale);
  return lh > 0 && lw > 0;
}

GaussTaps gauss_taps(int level) {
  GaussTaps gk{};
  if (level == 0) {                              // sigma 0, ksize 3: cv2's fixed small kernel
    gk.r = 1;
    gk.k[0] = 0.25f, gk.k[1] = 0.5f, gk.k[2] = 0.25f;
    return gk;
  }
  const double scale = std::ldexp(1.0, -level), sigma = (1.0 / scale - 1.0) * 0.5;
  const int ksize = std::max((int)std::lrint(sigma * 5) | 1, 3);
  gk.r = ksize / 2;
  double v[MAX_TAPS], s = 0.0;
  for (int i = 0; i < ksize; ++i) {
    const double x = i - (ksize - 1) * 0.5;
    v[i] = std::exp(-x * x / (2 * sigma * sigma));
    s += v[i];
  }
  for (int i = 0; i < ksize; ++i) gk.k[i] = (float)(v[i] / s);
  return gk;
}

// Normalised Gaussian (sigma 1.2, taps -5..5) with its x and x^2 moments in float, and the entries of the inverse of the
// 6x6 moment matrix (basis 1, x, y, x^2, y^2, xy) that map the weighted sums to coefficients.  That matrix only couples
// {1, x^2, y^2}; the 3x3 block is inverted by cofactors, and the x and xy entries are reciprocals.
PolyTaps poly_taps() {
  PolyTaps pt{};
  const double sigma = 1.2;
  float g[2 * POLY_N + 1];
  double s = 0.0;
  for (int x = -POLY_N; x <= POLY_N; ++x) {
    g[x + POLY_N] = (float)std::exp(-x * x / (2 * sigma * sigma));
    s += g[x + POLY_N];
  }
  s = 1.0 / s;
  for (int x = -POLY_N; x <= POLY_N; ++x) g[x + POLY_N] = (float)(g[x + POLY_N] * s);
  for (int k = 0; k <= POLY_N; ++k) {
    pt.g[k] = g[POLY_N + k];
    pt.xg[k] = (float)(k * g[POLY_N + k]);
    pt.xxg[k] = (float)(k * k * g[POLY_N + k]);
  }
  double G00 = 0, G11 = 0, G33 = 0, G55 = 0;
  for (int y = -POLY_N; y <= POLY_N; ++y)
    for (int x = -POLY_N; x <= POLY_N; ++x) {
      const double wgt = (double)g[y + POLY_N] * g[x + POLY_N];
      G00 += wgt;
      G11 += wgt * x * x;
      G33 += wgt * x * x * x * x;
      G55 += wgt * x * x * y * y;
    }
  // block [[G00, G11, G11], [G11, G33, G55], [G11, G55, G33]]
  const double a = G00, b = G11, c = G33, d = G55;
  const double det = a * (c * c - d * d) - b * (b * c - d * b) + b * (b * d - c * b);
  pt.ig11 = 1.0 / G11;
  pt.ig03 = -(b * c - d * b) / det;
  pt.ig33 = (a * c - b * b) / det;
  pt.ig55 = 1.0 / G55;
  return pt;
}
}  // namespace

extern "C" {

int teco_tof_grey_u8(const uint8_t* img, int32_t N, int32_t H, int32_t W, int32_t y0, int32_t x0, int32_t h, int32_t w,
                     uint8_t* grey, void* stream) {
  TECO_CHECK_ARG(img && grey, "teco_tof_grey_u8: NULL tensor");
  TECO_CHECK_ARG(N > 0 && H > 0 && W > 0 && h > 0 && w > 0, "teco_tof_grey_u8: bad size N=%d %dx%d window %dx%d", N, H, W, h, w);
  TECO_CHECK_ARG(y0 >= 0 && x0 >= 0 && y0 + h <= H && x0 + w <= W,
                 "teco_tof_grey_u8: window %d+%d x %d+%d does not fit a %dx%d frame", y0, h, x0, w, H, W);
  const long long total = (long long)N * h * w;
  grey_kernel<<<grid_for(total), TPB, 0, (cudaStream_t)stream>>>(img, H, W, y0, x0, h, w, total, grey);
  TECO_CUDA_LAUNCH_CHECK("teco_tof_grey_u8");
  return TECO_OK;
}

int teco_farneback_pyramid_u8(const uint8_t* grey, int32_t N, int32_t H, int32_t W, int32_t level, int32_t lh, int32_t lw,
                              float* out, void* stream) {
  TECO_CHECK_ARG(grey && out, "teco_farneback_pyramid_u8: NULL tensor");
  TECO_CHECK_ARG(N > 0 && H >= 2 && W >= 2, "teco_farneback_pyramid_u8: bad size N=%d %dx%d (at least 2x2)", N, H, W);
  TECO_CHECK_ARG(level >= 0 && level <= MAX_LEVEL, "teco_farneback_pyramid_u8: level %d outside 0..%d", level, MAX_LEVEL);
  int eh, ew;
  TECO_CHECK_ARG(level_size(H, W, level, eh, ew) && eh == lh && ew == lw,
                 "teco_farneback_pyramid_u8: level %d of %dx%d is %dx%d, not %dx%d", level, H, W, eh, ew, lh, lw);
  const GaussTaps gk = gauss_taps(level);
  TECO_CHECK_ARG(H > gk.r && W > gk.r, "teco_farneback_pyramid_u8: %dx%d is too small for level %d", H, W, level);
  const long long total = (long long)N * lh * lw;
  pyramid_kernel<<<grid_for(total), TPB, 0, (cudaStream_t)stream>>>(grey, H, W, lh, lw, total, gk, out);
  TECO_CUDA_LAUNCH_CHECK("teco_farneback_pyramid_u8");
  return TECO_OK;
}

int teco_farneback_polyexp_f32(const float* img, int32_t N, int32_t h, int32_t w, float* R, void* stream) {
  TECO_CHECK_ARG(img && R, "teco_farneback_polyexp_f32: NULL tensor");
  TECO_CHECK_ARG(N > 0 && N <= 65535 && h > 0 && w > 0, "teco_farneback_polyexp_f32: bad size N=%d %dx%d", N, h, w);
  static const PolyTaps pt = poly_taps();
  const dim3 grid(teco_ceil_div(w, PX), teco_ceil_div(h, PY), N);
  polyexp_kernel<<<grid, TPB, 0, (cudaStream_t)stream>>>(img, h, w, pt, R);
  TECO_CUDA_LAUNCH_CHECK("teco_farneback_polyexp_f32");
  return TECO_OK;
}

int teco_farneback_iterate_f32(const float* R, int32_t Nf, int32_t h, int32_t w, const int32_t* i0_host,
                               const int32_t* i1_host, int32_t P, const float* flow_in, float* flow_out, void* stream) {
  TECO_CHECK_ARG(R && flow_out && i0_host && i1_host, "teco_farneback_iterate_f32: NULL argument");
  TECO_CHECK_ARG(P > 0 && P <= MAX_PAIRS, "teco_farneback_iterate_f32: %d pairs (1..%d per launch)", P, MAX_PAIRS);
  TECO_CHECK_ARG(Nf > 0 && h >= 2 && w >= 2, "teco_farneback_iterate_f32: bad size Nf=%d %dx%d (at least 2x2)", Nf, h, w);
  TECO_CHECK_ARG(flow_in != flow_out, "teco_farneback_iterate_f32: flow_out must not alias flow_in");
  PairIdx pi;
  for (int p = 0; p < P; ++p) {
    TECO_CHECK_ARG(i0_host[p] >= 0 && i0_host[p] < Nf && i1_host[p] >= 0 && i1_host[p] < Nf,
                   "teco_farneback_iterate_f32: pair %d = (%d, %d) outside %d frames", p, i0_host[p], i1_host[p], Nf);
    pi.a[p] = i0_host[p];
    pi.b[p] = i1_host[p];
  }
  static bool attr = false;
  if (!attr) {
    TECO_CUDA_CALL(cudaFuncSetAttribute(iterate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ITER_SMEM));
    attr = true;
  }
  const dim3 grid(teco_ceil_div(w, IX), teco_ceil_div(h, IY), P);
  iterate_kernel<<<grid, TPB, ITER_SMEM, (cudaStream_t)stream>>>(R, h, w, pi, flow_in, flow_out);
  TECO_CUDA_LAUNCH_CHECK("teco_farneback_iterate_f32");
  return TECO_OK;
}

int teco_farneback_flow_up_f32(const float* flow_in, int32_t P, int32_t sh, int32_t sw, float* flow_out, int32_t h,
                               int32_t w, void* stream) {
  TECO_CHECK_ARG(flow_in && flow_out, "teco_farneback_flow_up_f32: NULL tensor");
  TECO_CHECK_ARG(P > 0 && sh > 0 && sw > 0 && h > 0 && w > 0, "teco_farneback_flow_up_f32: bad size P=%d %dx%d -> %dx%d", P,
                 sh, sw, h, w);
  const long long total = (long long)P * h * w;
  flow_up_kernel<<<grid_for(total), TPB, 0, (cudaStream_t)stream>>>(flow_in, sh, sw, h, w, total, flow_out);
  TECO_CUDA_LAUNCH_CHECK("teco_farneback_flow_up_f32");
  return TECO_OK;
}

int teco_tof_reduce_f32(const float* flow_a, const float* flow_b, int32_t P, int32_t H, int32_t W, int32_t y0, int32_t x0,
                        int32_t h, int32_t w, double* partial, double* out, void* stream) {
  TECO_CHECK_ARG(flow_a && flow_b && partial && out, "teco_tof_reduce_f32: NULL tensor");
  TECO_CHECK_ARG(P > 0 && P <= 65535 && H > 0 && W > 0, "teco_tof_reduce_f32: bad size P=%d %dx%d", P, H, W);
  TECO_CHECK_ARG(h > 0 && w > 0 && y0 >= 0 && x0 >= 0 && y0 + h <= H && x0 + w <= W,
                 "teco_tof_reduce_f32: window %d+%d x %d+%d does not fit a %dx%d flow", y0, h, x0, w, H, W);
  tof_partial_kernel<<<dim3(RED_CHUNKS, P), TPB, 0, (cudaStream_t)stream>>>(flow_a, flow_b, H, W, y0, x0, h, w, partial);
  TECO_CUDA_LAUNCH_CHECK("teco_tof_reduce_f32");
  tof_finish_kernel<<<teco_ceil_div(P, 128), 128, 0, (cudaStream_t)stream>>>(partial, P, 1.0 / ((double)h * w), out);
  TECO_CUDA_LAUNCH_CHECK("teco_tof_reduce_f32");
  return TECO_OK;
}

}  // extern "C"
