// Elementwise / conversion kernels, discriminator batch-norm, fused loss reductions and Adam.
// Reference call sites are cited in include/teco.h.
#include "teco_common.cuh"

namespace {

constexpr int TPB = 256;

inline unsigned grid_for(long long n, int per_block = TPB) {
  long long b = (n + per_block - 1) / per_block;
  long long cap = (long long)teco_sm_count() * 16;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

#define GRID_STRIDE(i, n) \
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (n); i += (long long)gridDim.x * blockDim.x)

__global__ void affine_act_kernel(const float* __restrict__ x, float* __restrict__ y, long long n, float a, float b, int act) {
  GRID_STRIDE(i, n) y[i] = teco_act(a * x[i] + b, act);
}

__global__ void act_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx,
                               long long n, int act) {
  GRID_STRIDE(i, n) {
    float v = y[i], g = dy[i];
    switch (act) {
      case TECO_ACT_RELU: g = v > 0.f ? g : 0.f; break;
      case TECO_ACT_LRELU02: g = v >= 0.f ? g : 0.2f * g; break;
      case TECO_ACT_TANH24: { float t = v * (1.0f / 24.0f); g = g * 24.0f * (1.f - t * t); break; }
      case TECO_ACT_SIGMOID: g = g * v * (1.f - v); break;
      default: break;
    }
    dx[i] = g;
  }
}

__global__ void f32_to_bf16_pad_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long npix,
                                       int C, int src_cpitch, int dst_cpitch, int c_off, float scale, float shift) {
  long long total = npix * C;
  GRID_STRIDE(i, total) {
    long long p = i / C;
    int c = (int)(i - p * C);
    dst[p * dst_cpitch + c_off + c] = __float2bfloat16_rn(src[p * src_cpitch + c] * scale + shift);
  }
}

__global__ void bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ src, float* __restrict__ dst, long long npix, int C,
                                   int src_cpitch, int dst_cpitch) {
  long long total = npix * C;
  GRID_STRIDE(i, total) {
    long long p = i / C;
    int c = (int)(i - p * C);
    dst[p * dst_cpitch + c] = __bfloat162float(src[p * src_cpitch + c]);
  }
}

__global__ void to_u8_kernel(const float* __restrict__ x, uint8_t* __restrict__ y, long long n) {
  GRID_STRIDE(i, n) {
    float v = fminf(fmaxf(x[i] * 255.0f, 0.f), 255.f);
    y[i] = (uint8_t)v;  // numpy astype(uint8) truncates (reference lib/ops.py:522)
  }
}

// deprocess + save_img quantisation in one pass (reference lib/ops.py:17-22, 521-523): y01 = (x+1)/2, y8 = u8(clip(255*y01))
__global__ void deprocess_u8_kernel(const float* __restrict__ x, float* __restrict__ y01, uint8_t* __restrict__ y8, long long n4,
                                    long long n) {
  GRID_STRIDE(i, n4) {
    const float4 v = reinterpret_cast<const float4*>(x)[i];
    float4 o;
    o.x = 0.5f * v.x + 0.5f; o.y = 0.5f * v.y + 0.5f; o.z = 0.5f * v.z + 0.5f; o.w = 0.5f * v.w + 0.5f;
    if (y01) reinterpret_cast<float4*>(y01)[i] = o;
    uchar4 q;
    q.x = (uint8_t)fminf(fmaxf(o.x * 255.0f, 0.f), 255.f); q.y = (uint8_t)fminf(fmaxf(o.y * 255.0f, 0.f), 255.f);
    q.z = (uint8_t)fminf(fmaxf(o.z * 255.0f, 0.f), 255.f); q.w = (uint8_t)fminf(fmaxf(o.w * 255.0f, 0.f), 255.f);
    reinterpret_cast<uchar4*>(y8)[i] = q;
  }
  if (blockIdx.x == 0 && threadIdx.x < (int)(n - 4 * n4)) {   // tail (n not a multiple of 4)
    const long long i = 4 * n4 + threadIdx.x;
    const float o = 0.5f * x[i] + 0.5f;
    if (y01) y01[i] = o;
    y8[i] = (uint8_t)fminf(fmaxf(o * 255.0f, 0.f), 255.f);
  }
}

// ------------------------------------------------------------------ batch norm (per channel over pixels)
// Thread (c = tid % C, lane ps = tid / C) of a block sums pixels p0 + ps, p0 + ps + ppar, ... of its block's range.
// Default: each lane adds its sum into acc[c] with an atomic.  kDet: the lanes' sums meet in shared memory and lane 0 adds
// them in lane order into part[block][c] (the fixed-order path of the *_det entry points), with every product and sum
// rounded explicitly so the order can be restated on the host.
template <bool kDet>
__device__ __forceinline__ void bn_lane_out(float* sh, float v, int ppar, int C, float* acc, float* part) {
  const int c = threadIdx.x % C, ps = threadIdx.x / C;
  if (!kDet) {
    if (ps < ppar) atomicAdd(&acc[c], v);
    return;
  }
  sh[threadIdx.x] = v;
  __syncthreads();
  if (ps == 0) {
    for (int k = 1; k < ppar; ++k) v = __fadd_rn(v, sh[k * C + c]);
    part[c] = v;
  }
  __syncthreads();
}

// pass 1: per-block partial sums into acc[0,C) via atomics (or part[block][C]); C <= 256.
template <bool kDet>
__global__ void bn_partial_kernel(const float* __restrict__ x, float* __restrict__ acc, long long npix, int C,
                                  long long pix_per_block, float* __restrict__ part) {
  __shared__ float sh[TPB];
  int ppar = TPB / C;
  int c = threadIdx.x % C, ps = threadIdx.x / C;
  if (!kDet && ps >= ppar) return;
  long long p0 = (long long)blockIdx.x * pix_per_block, p1 = min(npix, p0 + pix_per_block);
  float s = 0.f;
  if (ps < ppar)
    for (long long p = p0 + ps; p < p1; p += ppar) s = kDet ? __fadd_rn(s, x[p * C + c]) : s + x[p * C + c];
  bn_lane_out<kDet>(sh, s, ppar, C, acc, part + (kDet ? (size_t)blockIdx.x * C : 0));
}
// two-pass variance for accuracy: pass 2 accumulates sum (x-mean)^2
template <bool kDet>
__global__ void bn_var_kernel(const float* __restrict__ x, const float* __restrict__ acc, float* __restrict__ var_acc,
                              long long npix, int C, long long pix_per_block, float* __restrict__ part) {
  __shared__ float sh[TPB];
  int ppar = TPB / C;
  int c = threadIdx.x % C, ps = threadIdx.x / C;
  if (!kDet && ps >= ppar) return;
  float mean = kDet ? __fdiv_rn(acc[c], (float)npix) : acc[c] / (float)npix;
  long long p0 = (long long)blockIdx.x * pix_per_block, p1 = min(npix, p0 + pix_per_block);
  float q = 0.f;
  if (ps < ppar)
    for (long long p = p0 + ps; p < p1; p += ppar) {
      if (kDet) {
        const float v = __fsub_rn(x[p * C + c], mean);
        q = __fadd_rn(q, __fmul_rn(v, v));
      } else {
        float v = x[p * C + c] - mean;
        q += v * v;
      }
    }
  bn_lane_out<kDet>(sh, q, ppar, C, var_acc, part + (kDet ? (size_t)blockIdx.x * C : 0));
}
__global__ void bn_finalize_kernel(const float* __restrict__ acc, const float* __restrict__ var_acc,
                                   float* __restrict__ stats, long long npix, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) {
    stats[c] = acc[c] / (float)npix;
    stats[C + c] = var_acc[c] / (float)npix;
  }
}
__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ beta, const float* __restrict__ stats,
                                float* __restrict__ y, long long npix, int C, float eps, int lrelu02) {
  long long total = npix * C;
  GRID_STRIDE(i, total) {
    int c = (int)(i % C);
    float v = (x[i] - stats[c]) * rsqrtf(stats[C + c] + eps) + beta[c];
    if (lrelu02) v = v >= 0.f ? v : 0.2f * v;
    y[i] = v;
  }
}
// backward: g = dy * lrelu'(y); dbeta = sum g; dx = rstd * (g - mean(g) - xhat * mean(g*xhat))
template <bool kDet>
__global__ void bn_bwd_partial_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                      const float* __restrict__ stats, float* __restrict__ acc, long long npix, int C,
                                      float eps, int lrelu02, long long pix_per_block, float* __restrict__ part) {
  __shared__ float sh[TPB];
  int ppar = TPB / C;
  int c = threadIdx.x % C, ps = threadIdx.x / C;
  if (!kDet && ps >= ppar) return;
  float mean = stats[c], rstd = rsqrtf(stats[C + c] + eps);
  long long p0 = (long long)blockIdx.x * pix_per_block, p1 = min(npix, p0 + pix_per_block);
  float s = 0.f, q = 0.f;
  if (ps < ppar)
    for (long long p = p0 + ps; p < p1; p += ppar) {
      float g = dy[p * C + c];
      if (lrelu02 && y[p * C + c] < 0.f) g *= 0.2f;
      if (kDet) {
        s = __fadd_rn(s, g);
        q = __fadd_rn(q, __fmul_rn(__fmul_rn(g, __fsub_rn(x[p * C + c], mean)), rstd));
      } else {
        s += g;
        q += g * (x[p * C + c] - mean) * rstd;
      }
    }
  float* pb = part + (kDet ? (size_t)blockIdx.x * 2 * C : 0);
  bn_lane_out<kDet>(sh, s, ppar, C, acc, pb);
  bn_lane_out<kDet>(sh, q, ppar, C, acc + C, pb + C);
}
__global__ void bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ dy,
                                    const float* __restrict__ stats, const float* __restrict__ acc, float* __restrict__ dx,
                                    long long npix, int C, float eps, int lrelu02) {
  long long total = npix * C;
  float inv = 1.0f / (float)npix;
  GRID_STRIDE(i, total) {
    int c = (int)(i % C);
    float mean = stats[c], rstd = rsqrtf(stats[C + c] + eps);
    float g = dy[i];
    if (lrelu02 && y[i] < 0.f) g *= 0.2f;
    float xhat = (x[i] - mean) * rstd;
    dx[i] = rstd * (g - acc[c] * inv - xhat * acc[C + c] * inv);
  }
}

// ------------------------------------------------------------------ loss reductions
// warp-shuffle -> block -> one atomic per block into out[k].  With part != NULL (the *_det entry points) block b stores
// its value to part[b * K + k] instead, and the per-thread sums round every product and sum explicitly.
__device__ __forceinline__ void loss_block_out(float* out, float* part, int K, int k, float v) {
  if (part) part[(size_t)blockIdx.x * K + k] = v;
  else atomicAdd(out + k, v);
}

__global__ void loss_l2_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                               float* __restrict__ da, long long n, float inv_npix, float gscale, float* __restrict__ part) {
  __shared__ float sm[32];
  float s = 0.f;
  GRID_STRIDE(i, n) {
    float d = a[i] - b[i];
    if (part) s = __fadd_rn(s, __fmul_rn(d, d));
    else s += d * d;
    if (da) da[i] = 2.f * d * inv_npix * gscale;
  }
  s = block_sum(s, sm);
  if (threadIdx.x == 0) loss_block_out(out, part, 1, 0, s * inv_npix);
}

__global__ void loss_l1_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                               float* __restrict__ da, float* __restrict__ db, long long n, float inv_den, float gscale,
                               float* __restrict__ part) {
  __shared__ float sm[32];
  float s = 0.f;
  GRID_STRIDE(i, n) {
    float d = a[i] - b[i];
    s += fabsf(d);
    float g = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * inv_den * gscale;
    if (da) da[i] = g;
    if (db) db[i] = -g;
  }
  s = block_sum(s, sm);
  if (threadIdx.x == 0) loss_block_out(out, part, 1, 0, s * inv_den);
}

// one warp per pixel: cos = <f,g> / (sqrt(|f|^2+eps) sqrt(|g|^2+eps)), eps=1e-12 (reference lib/Teco.py:20)
__global__ void loss_cosine_kernel(const float* __restrict__ f, const float* __restrict__ g, float* __restrict__ out,
                                   float* __restrict__ df, long long npix, int C, float gscale, float* __restrict__ part) {
  __shared__ float sm[32];
  int lane = threadIdx.x & 31;
  long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  float local = 0.f;
  float inv = 1.0f / (float)npix;
  for (long long p = warp; p < npix; p += nwarps) {
    const float* fp = f + p * C;
    const float* gp = g + p * C;
    float ff = 0.f, gg = 0.f, fg = 0.f;
    for (int c = lane; c < C; c += 32) {
      float x = fp[c], y = gp[c];
      if (part) {
        ff = __fadd_rn(ff, __fmul_rn(x, x));
        gg = __fadd_rn(gg, __fmul_rn(y, y));
        fg = __fadd_rn(fg, __fmul_rn(x, y));
      } else {
        ff += x * x;
        gg += y * y;
        fg += x * y;
      }
    }
    ff = warp_sum(ff);
    gg = warp_sum(gg);
    fg = warp_sum(fg);
    float nf = sqrtf(ff + 1e-12f), ng = sqrtf(gg + 1e-12f);
    float cosv = fg / (nf * ng);
    if (lane == 0) local = part ? __fadd_rn(local, cosv) : local + cosv;
    if (df) {
      // d(1 - mean cos)/df = -(1/npix) * ( g/(nf ng) - cos * f / nf^2 )
      float k1 = -inv * gscale / (nf * ng), k2 = inv * gscale * cosv / (nf * nf);
      for (int c = lane; c < C; c += 32) df[p * C + c] = k1 * gp[c] + k2 * fp[c];
    }
  }
  float s = block_sum(local, sm);
  if (threadIdx.x == 0) loss_block_out(out, part, 1, 0, -s * inv);
}
__global__ void add_const_kernel(float* p, float v) { p[0] += v; }

__global__ void loss_gan_kernel(const float* __restrict__ dfk, const float* __restrict__ drl, float* __restrict__ out,
                                float* __restrict__ g_adv, float* __restrict__ g_dis_f, float* __restrict__ g_dis_r,
                                long long n, float eps, float s_adv, float s_dis, float* __restrict__ part) {
  __shared__ float sm[32];
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
  float inv = 1.0f / (float)n;
  GRID_STRIDE(i, n) {
    float f = dfk[i], r = drl[i];
    float lf = logf(f + eps), l1f = logf(1.f - f + eps), lr = logf(r + eps);
    if (part) {
      a0 = __fadd_rn(a0, -lf);
      a1 = __fadd_rn(a1, -__fadd_rn(l1f, lr));
      a2 = __fadd_rn(a2, lr);
      a3 = __fadd_rn(a3, r);
      a4 = __fadd_rn(a4, f);
    } else {
      a0 += -lf;
      a1 += -(l1f + lr);
      a2 += lr;
      a3 += r;
      a4 += f;
    }
    if (g_adv) g_adv[i] = -inv * s_adv / (f + eps);
    if (g_dis_f) g_dis_f[i] = inv * s_dis / (1.f - f + eps);
    if (g_dis_r) g_dis_r[i] = -inv * s_dis / (r + eps);
  }
  a0 = block_sum(a0, sm);
  a1 = block_sum(a1, sm);
  a2 = block_sum(a2, sm);
  a3 = block_sum(a3, sm);
  a4 = block_sum(a4, sm);
  if (threadIdx.x == 0) {
    loss_block_out(out, part, 5, 0, a0 * inv);
    loss_block_out(out, part, 5, 1, a1 * inv);
    loss_block_out(out, part, 5, 2, a2 * inv);
    loss_block_out(out, part, 5, 3, a3 * inv);
    loss_block_out(out, part, 5, 4, a4 * inv);
  }
}

// out[e] (+)= part[0][e] + part[1][e] + ... + part[S-1][e], summed in split order (the fixed-order reductions).
__global__ void reduce_splits_kernel(const float* __restrict__ part, int S, long long E, float* __restrict__ out, int accumulate) {
  GRID_STRIDE(e, E) {
    float t = part[e];
    for (int s = 1; s < S; ++s) t = __fadd_rn(t, part[(long long)s * E + e]);
    out[e] = accumulate ? __fadd_rn(out[e], t) : t;
  }
}

__global__ void adam_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                            const float* __restrict__ g, long long n, float lr_t, float b1, float b2, float eps,
                            float gscale) {
  GRID_STRIDE(i, n) {
    float gi = g[i] * gscale;
    float mi = b1 * m[i] + (1.f - b1) * gi;
    float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] = p[i] - lr_t * mi / (sqrtf(vi) + eps);
  }
}

}  // namespace

#define ST ((cudaStream_t)stream)

extern "C" {

int teco_affine_act_f32(const float* x, float* y, int64_t n, float a, float b, int32_t act, void* stream) {
  TECO_CHECK_ARG(x && y && n > 0, "teco_affine_act_f32: bad argument");
  affine_act_kernel<<<grid_for(n), TPB, 0, ST>>>(x, y, n, a, b, act);
  TECO_CUDA_LAUNCH_CHECK("teco_affine_act_f32");
  return TECO_OK;
}

int teco_act_bwd_f32(const float* y, const float* dy, float* dx, int64_t n, int32_t act, void* stream) {
  TECO_CHECK_ARG(y && dy && dx && n > 0, "teco_act_bwd_f32: bad argument");
  act_bwd_kernel<<<grid_for(n), TPB, 0, ST>>>(y, dy, dx, n, act);
  TECO_CUDA_LAUNCH_CHECK("teco_act_bwd_f32");
  return TECO_OK;
}

int teco_f32_to_bf16_pad(const float* src, void* dst, int64_t npix, int32_t C, int32_t src_cpitch, int32_t dst_cpitch,
                         int32_t c_off, float scale, float shift, void* stream) {
  TECO_CHECK_ARG(src && dst && npix > 0 && C > 0 && src_cpitch >= C && c_off >= 0 && c_off + C <= dst_cpitch,
                 "teco_f32_to_bf16_pad: bad argument");
  f32_to_bf16_pad_kernel<<<grid_for(npix * C), TPB, 0, ST>>>(src, (__nv_bfloat16*)dst, npix, C, src_cpitch, dst_cpitch,
                                                              c_off, scale, shift);
  TECO_CUDA_LAUNCH_CHECK("teco_f32_to_bf16_pad");
  return TECO_OK;
}

int teco_bf16_to_f32(const void* src, float* dst, int64_t npix, int32_t C, int32_t src_cpitch, int32_t dst_cpitch,
                     void* stream) {
  TECO_CHECK_ARG(src && dst && npix > 0 && C > 0 && src_cpitch >= C && dst_cpitch >= C, "teco_bf16_to_f32: bad argument");
  bf16_to_f32_kernel<<<grid_for(npix * C), TPB, 0, ST>>>((const __nv_bfloat16*)src, dst, npix, C, src_cpitch, dst_cpitch);
  TECO_CUDA_LAUNCH_CHECK("teco_bf16_to_f32");
  return TECO_OK;
}

int teco_to_u8(const float* x, uint8_t* y, int64_t n, void* stream) {
  TECO_CHECK_ARG(x && y && n > 0, "teco_to_u8: bad argument");
  to_u8_kernel<<<grid_for(n), TPB, 0, ST>>>(x, y, n);
  TECO_CUDA_LAUNCH_CHECK("teco_to_u8");
  return TECO_OK;
}

int teco_deprocess_u8(const float* x, float* y01, uint8_t* y8, int64_t n, void* stream) {
  TECO_CHECK_ARG(x && y8 && n > 0, "teco_deprocess_u8: bad argument");   // y01 may be NULL: uint8 frame only
  TECO_CHECK_ARG((((uintptr_t)x) & 15) == 0 && (((uintptr_t)y01) & 15) == 0 && (((uintptr_t)y8) & 3) == 0,
                 "teco_deprocess_u8: x / y01 must be 16-byte aligned, y8 4-byte aligned");
  const long long n4 = n / 4;
  deprocess_u8_kernel<<<grid_for(n4 > 0 ? n4 : 1), TPB, 0, ST>>>(x, y01, y8, n4, n);
  TECO_CUDA_LAUNCH_CHECK("teco_deprocess_u8");
  return TECO_OK;
}

// stats doubles as scratch: caller provides stats[4C]: [0,2C) outputs (mean,var), [2C,3C) sum x, [3C,4C) sum (x-mean)^2
int teco_bn_train_f32(const float* x, const float* beta, float* y, float* stats, int64_t npix, int32_t C, float eps,
                      int32_t lrelu02, void* stream) {
  TECO_CHECK_ARG(x && beta && y && stats && npix > 0, "teco_bn_train_f32: bad argument");
  TECO_CHECK_ARG(C > 0 && C <= 256, "teco_bn_train_f32: C must be in [1,256] (got %d)", C);
  float* acc = stats + 2 * C;
  TECO_CUDA_CALL(cudaMemsetAsync(acc, 0, sizeof(float) * 2 * C, ST));
  long long blocks = (npix + 1023) / 1024;
  if (blocks > 2 * teco_sm_count()) blocks = 2 * teco_sm_count();
  long long ppb = (npix + blocks - 1) / blocks;
  blocks = (npix + ppb - 1) / ppb;
  bn_partial_kernel<false><<<(unsigned)blocks, TPB, 0, ST>>>(x, acc, npix, C, ppb, nullptr);
  bn_var_kernel<false><<<(unsigned)blocks, TPB, 0, ST>>>(x, acc, acc + C, npix, C, ppb, nullptr);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_f32(stats)");
  bn_finalize_kernel<<<teco_ceil_div(C, 128), 128, 0, ST>>>(acc, acc + C, stats, npix, C);
  bn_apply_kernel<<<grid_for(npix * C), TPB, 0, ST>>>(x, beta, stats, y, npix, C, eps, lrelu02);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_f32");
  return TECO_OK;
}

int teco_bn_train_bwd_f32(const float* x, const float* y, const float* dy, const float* stats, float* dx, float* dbeta,
                          int64_t npix, int32_t C, float eps, int32_t lrelu02, void* stream) {
  TECO_CHECK_ARG(x && y && dy && stats && dx && dbeta && npix > 0, "teco_bn_train_bwd_f32: bad argument");
  TECO_CHECK_ARG(C > 0 && C <= 256, "teco_bn_train_bwd_f32: C must be in [1,256] (got %d)", C);
  // dbeta[2C]: [0,C) = sum g (the beta gradient), [C,2C) scratch = sum g*xhat
  TECO_CUDA_CALL(cudaMemsetAsync(dbeta, 0, sizeof(float) * 2 * C, ST));
  long long blocks = (npix + 1023) / 1024;
  if (blocks > 2 * teco_sm_count()) blocks = 2 * teco_sm_count();
  long long ppb = (npix + blocks - 1) / blocks;
  blocks = (npix + ppb - 1) / ppb;
  bn_bwd_partial_kernel<false><<<(unsigned)blocks, TPB, 0, ST>>>(x, y, dy, stats, dbeta, npix, C, eps, lrelu02, ppb, nullptr);
  bn_bwd_apply_kernel<<<grid_for(npix * C), TPB, 0, ST>>>(x, y, dy, stats, dbeta, dx, npix, C, eps, lrelu02);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_bwd_f32");
  return TECO_OK;
}

int teco_loss_l2_f32(const float* a, const float* b, float* out, float* da, int64_t npix, int32_t C, float gscale,
                     void* stream) {
  TECO_CHECK_ARG(a && b && out && npix > 0 && C > 0, "teco_loss_l2_f32: bad argument");
  TECO_CUDA_CALL(cudaMemsetAsync(out, 0, sizeof(float), ST));
  loss_l2_kernel<<<grid_for(npix * C, TPB * 4), TPB, 0, ST>>>(a, b, out, da, npix * C, 1.0f / (float)npix, gscale, nullptr);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_l2_f32");
  return TECO_OK;
}

int teco_loss_l1_f32(const float* a, const float* b, float* out, float* da, float* db, int64_t npix, int32_t C,
                     int32_t per_pixel, float gscale, void* stream) {
  TECO_CHECK_ARG(a && b && out && npix > 0 && C > 0, "teco_loss_l1_f32: bad argument");
  TECO_CUDA_CALL(cudaMemsetAsync(out, 0, sizeof(float), ST));
  float inv_den = per_pixel ? 1.0f / (float)npix : 1.0f / ((float)npix * (float)C);
  loss_l1_kernel<<<grid_for(npix * C, TPB * 4), TPB, 0, ST>>>(a, b, out, da, db, npix * C, inv_den, gscale, nullptr);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_l1_f32");
  return TECO_OK;
}

int teco_loss_cosine_f32(const float* f, const float* g, float* out, float* df, int64_t npix, int32_t C, float gscale,
                         void* stream) {
  TECO_CHECK_ARG(f && g && out && npix > 0 && C > 0, "teco_loss_cosine_f32: bad argument");
  TECO_CUDA_CALL(cudaMemsetAsync(out, 0, sizeof(float), ST));
  loss_cosine_kernel<<<grid_for(npix * 32), TPB, 0, ST>>>(f, g, out, df, npix, C, gscale, nullptr);
  add_const_kernel<<<1, 1, 0, ST>>>(out, 1.0f);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_cosine_f32");
  return TECO_OK;
}

int teco_loss_gan_f32(const float* d_fake, const float* d_real, float* out, float* g_adv, float* g_dis_f,
                      float* g_dis_r, int64_t n, float eps, float s_adv, float s_dis, void* stream) {
  TECO_CHECK_ARG(d_fake && d_real && out && n > 0, "teco_loss_gan_f32: bad argument");
  TECO_CUDA_CALL(cudaMemsetAsync(out, 0, sizeof(float) * 5, ST));
  loss_gan_kernel<<<grid_for(n, TPB * 4), TPB, 0, ST>>>(d_fake, d_real, out, g_adv, g_dis_f, g_dis_r, n, eps, s_adv, s_dis, nullptr);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_gan_f32");
  return TECO_OK;
}

int teco_adam_f32(float* p, float* m, float* v, const float* g, int64_t n, float lr_t, float b1, float b2, float eps,
                  float gscale, void* stream) {
  TECO_CHECK_ARG(p && m && v && g && n > 0, "teco_adam_f32: bad argument");
  adam_kernel<<<grid_for(n), TPB, 0, ST>>>(p, m, v, g, n, lr_t, b1, b2, eps, gscale);
  TECO_CUDA_LAUNCH_CHECK("teco_adam_f32");
  return TECO_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// Fixed-order (deterministic) variants.  Every partition below is a function of the call's shapes alone, never of the
// device: block b of a reduction writes its partial to the caller's workspace and reduce_splits_kernel sums the partials
// in block order.  DESIGN.md section 4.3 gives the orders and the workspace sizes.
namespace {
constexpr long long DET_BN_BLOCKS = 264;     // batch-norm statistics: at most this many blocks of >= 1024 pixels
constexpr long long DET_LOSS_BLOCKS = 2112;  // loss reductions: at most this many blocks

long long det_bn_blocks(long long npix, long long* ppb) {
  long long blocks = (npix + 1023) / 1024;
  if (blocks > DET_BN_BLOCKS) blocks = DET_BN_BLOCKS;
  *ppb = (npix + blocks - 1) / blocks;
  return (npix + *ppb - 1) / *ppb;
}

unsigned det_grid(long long n, int per_block) {
  long long b = (n + per_block - 1) / per_block;
  if (b > DET_LOSS_BLOCKS) b = DET_LOSS_BLOCKS;
  if (b < 1) b = 1;
  return (unsigned)b;
}

// blocks of each loss: l2 / l1 (kind 0 / 1) over npix * C elements, cosine (2) one warp per pixel, gan (3) over npix values
unsigned det_loss_blocks(int kind, long long npix, int C) {
  if (kind == 2) return det_grid(npix * 32, TPB);
  if (kind == 3) return det_grid(npix, TPB * 4);
  return det_grid(npix * C, TPB * 4);
}
}  // namespace

int teco_reduce_splits(const float* part, int S, long long E, float* out, int accumulate, cudaStream_t stream) {
  reduce_splits_kernel<<<grid_for(E), TPB, 0, stream>>>(part, S, E, out, accumulate);
  TECO_CUDA_LAUNCH_CHECK("reduce_splits_kernel");
  return TECO_OK;
}

#define DET_WS_CHECK(who, need) \
  TECO_CHECK_ARG(ws && ws_bytes >= (int64_t)(need) && (((uintptr_t)ws) & 15) == 0, \
                 "%s: workspace of %lld bytes (16-byte aligned) needed, got %lld", who, (long long)(need), (long long)ws_bytes)

extern "C" {

int teco_bn_det_plan_bytes(int64_t npix, int32_t C, int64_t* ws_bytes_host) {
  TECO_CHECK_ARG(ws_bytes_host && npix > 0 && C > 0 && C <= 256, "teco_bn_det_plan_bytes: bad argument");
  long long ppb;
  *ws_bytes_host = (int64_t)det_bn_blocks(npix, &ppb) * 2 * C * (int64_t)sizeof(float);
  return TECO_OK;
}

int teco_bn_train_f32_det(const float* x, const float* beta, float* y, float* stats, int64_t npix, int32_t C, float eps,
                          int32_t lrelu02, void* ws, int64_t ws_bytes, void* stream) {
  TECO_CHECK_ARG(x && beta && y && stats && npix > 0, "teco_bn_train_f32_det: bad argument");
  TECO_CHECK_ARG(C > 0 && C <= 256, "teco_bn_train_f32_det: C must be in [1,256] (got %d)", C);
  long long ppb;
  const long long blocks = det_bn_blocks(npix, &ppb);
  DET_WS_CHECK("teco_bn_train_f32_det", blocks * 2 * C * sizeof(float));
  float* acc = stats + 2 * C;
  float* part = (float*)ws;
  bn_partial_kernel<true><<<(unsigned)blocks, TPB, 0, ST>>>(x, nullptr, npix, C, ppb, part);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_f32_det(sum)");
  int rc = teco_reduce_splits(part, (int)blocks, C, acc, 0, ST);
  if (rc) return rc;
  bn_var_kernel<true><<<(unsigned)blocks, TPB, 0, ST>>>(x, acc, nullptr, npix, C, ppb, part);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_f32_det(var)");
  rc = teco_reduce_splits(part, (int)blocks, C, acc + C, 0, ST);
  if (rc) return rc;
  bn_finalize_kernel<<<teco_ceil_div(C, 128), 128, 0, ST>>>(acc, acc + C, stats, npix, C);
  bn_apply_kernel<<<grid_for(npix * C), TPB, 0, ST>>>(x, beta, stats, y, npix, C, eps, lrelu02);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_f32_det");
  return TECO_OK;
}

int teco_bn_train_bwd_f32_det(const float* x, const float* y, const float* dy, const float* stats, float* dx, float* dbeta,
                              int64_t npix, int32_t C, float eps, int32_t lrelu02, void* ws, int64_t ws_bytes, void* stream) {
  TECO_CHECK_ARG(x && y && dy && stats && dx && dbeta && npix > 0, "teco_bn_train_bwd_f32_det: bad argument");
  TECO_CHECK_ARG(C > 0 && C <= 256, "teco_bn_train_bwd_f32_det: C must be in [1,256] (got %d)", C);
  long long ppb;
  const long long blocks = det_bn_blocks(npix, &ppb);
  DET_WS_CHECK("teco_bn_train_bwd_f32_det", blocks * 2 * C * sizeof(float));
  float* part = (float*)ws;
  bn_bwd_partial_kernel<true><<<(unsigned)blocks, TPB, 0, ST>>>(x, y, dy, stats, nullptr, npix, C, eps, lrelu02, ppb, part);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_bwd_f32_det(partial)");
  const int rc = teco_reduce_splits(part, (int)blocks, 2 * C, dbeta, 0, ST);
  if (rc) return rc;
  bn_bwd_apply_kernel<<<grid_for(npix * C), TPB, 0, ST>>>(x, y, dy, stats, dbeta, dx, npix, C, eps, lrelu02);
  TECO_CUDA_LAUNCH_CHECK("teco_bn_train_bwd_f32_det");
  return TECO_OK;
}

int teco_loss_det_plan_bytes(int64_t npix, int32_t C, int64_t* ws_bytes_host) {
  TECO_CHECK_ARG(ws_bytes_host && npix > 0 && C > 0, "teco_loss_det_plan_bytes: bad argument");
  unsigned most = 0;
  for (int kind = 0; kind < 4; ++kind) {
    const unsigned b = det_loss_blocks(kind, npix, C) * (kind == 3 ? 5 : 1);
    if (b > most) most = b;
  }
  *ws_bytes_host = (int64_t)most * (int64_t)sizeof(float);
  return TECO_OK;
}

int teco_loss_l2_f32_det(const float* a, const float* b, float* out, float* da, int64_t npix, int32_t C, float gscale,
                         void* ws, int64_t ws_bytes, void* stream) {
  TECO_CHECK_ARG(a && b && out && npix > 0 && C > 0, "teco_loss_l2_f32_det: bad argument");
  const unsigned blocks = det_loss_blocks(0, npix, C);
  DET_WS_CHECK("teco_loss_l2_f32_det", blocks * sizeof(float));
  loss_l2_kernel<<<blocks, TPB, 0, ST>>>(a, b, out, da, npix * C, 1.0f / (float)npix, gscale, (float*)ws);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_l2_f32_det");
  return teco_reduce_splits((float*)ws, (int)blocks, 1, out, 0, ST);
}

int teco_loss_l1_f32_det(const float* a, const float* b, float* out, float* da, float* db, int64_t npix, int32_t C,
                         int32_t per_pixel, float gscale, void* ws, int64_t ws_bytes, void* stream) {
  TECO_CHECK_ARG(a && b && out && npix > 0 && C > 0, "teco_loss_l1_f32_det: bad argument");
  const unsigned blocks = det_loss_blocks(1, npix, C);
  DET_WS_CHECK("teco_loss_l1_f32_det", blocks * sizeof(float));
  float inv_den = per_pixel ? 1.0f / (float)npix : 1.0f / ((float)npix * (float)C);
  loss_l1_kernel<<<blocks, TPB, 0, ST>>>(a, b, out, da, db, npix * C, inv_den, gscale, (float*)ws);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_l1_f32_det");
  return teco_reduce_splits((float*)ws, (int)blocks, 1, out, 0, ST);
}

int teco_loss_cosine_f32_det(const float* f, const float* g, float* out, float* df, int64_t npix, int32_t C, float gscale,
                             void* ws, int64_t ws_bytes, void* stream) {
  TECO_CHECK_ARG(f && g && out && npix > 0 && C > 0, "teco_loss_cosine_f32_det: bad argument");
  const unsigned blocks = det_loss_blocks(2, npix, C);
  DET_WS_CHECK("teco_loss_cosine_f32_det", blocks * sizeof(float));
  loss_cosine_kernel<<<blocks, TPB, 0, ST>>>(f, g, out, df, npix, C, gscale, (float*)ws);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_cosine_f32_det");
  const int rc = teco_reduce_splits((float*)ws, (int)blocks, 1, out, 0, ST);
  if (rc) return rc;
  add_const_kernel<<<1, 1, 0, ST>>>(out, 1.0f);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_cosine_f32_det");
  return TECO_OK;
}

int teco_loss_gan_f32_det(const float* d_fake, const float* d_real, float* out, float* g_adv, float* g_dis_f,
                          float* g_dis_r, int64_t n, float eps, float s_adv, float s_dis, void* ws, int64_t ws_bytes,
                          void* stream) {
  TECO_CHECK_ARG(d_fake && d_real && out && n > 0, "teco_loss_gan_f32_det: bad argument");
  const unsigned blocks = det_loss_blocks(3, n, 1);
  DET_WS_CHECK("teco_loss_gan_f32_det", blocks * 5 * sizeof(float));
  loss_gan_kernel<<<blocks, TPB, 0, ST>>>(d_fake, d_real, out, g_adv, g_dis_f, g_dis_r, n, eps, s_adv, s_dis, (float*)ws);
  TECO_CUDA_LAUNCH_CHECK("teco_loss_gan_f32_det");
  return teco_reduce_splits((float*)ws, (int)blocks, 5, out, 0, ST);
}

int teco_sum_ranks_f32(const float* src, int32_t R, int64_t n, float* dst, void* stream) {
  TECO_CHECK_ARG(src && dst && R > 0 && n > 0, "teco_sum_ranks_f32: bad argument");
  return teco_reduce_splits(src, R, n, dst, 0, ST);
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------
// per-pixel channel L2 normalisation of VGG features (reference lib/Teco.py:19-21): y = f / sqrt(sum_c f^2 + 1e-12)
namespace {
__global__ void l2norm_channels_kernel(const float* __restrict__ f, float* __restrict__ y, long long npix, int C) {
  int lane = threadIdx.x & 31;
  long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long p = warp; p < npix; p += nwarps) {
    float ss = 0.f;
    for (int c = lane; c < C; c += 32) { float v = f[p * C + c]; ss += v * v; }
    ss = warp_sum(ss);
    float inv = 1.0f / sqrtf(ss + 1e-12f);
    for (int c = lane; c < C; c += 32) y[p * C + c] = f[p * C + c] * inv;
  }
}
}  // namespace

extern "C" int teco_l2norm_channels_f32(const float* f, float* y, int64_t npix, int32_t C, void* stream) {
  TECO_CHECK_ARG(f && y && npix > 0 && C > 0, "teco_l2norm_channels_f32: bad argument");
  l2norm_channels_kernel<<<grid_for(npix * 32), TPB, 0, (cudaStream_t)stream>>>(f, y, npix, C);
  TECO_CUDA_LAUNCH_CHECK("teco_l2norm_channels_f32");
  return TECO_OK;
}

// ---------------------------------------------------------------------------------------------------
// conversions used by the bf16 tensor-core training path
namespace {
__global__ void bf16_to_f32_add_kernel(const __nv_bfloat16* __restrict__ src, const float* __restrict__ add,
                                       float* __restrict__ dst, long long npix, int C, int src_cpitch, int dst_cpitch) {
  long long total = npix * C;
  GRID_STRIDE(i, total) {
    long long p = i / C;
    int c = (int)(i - p * C);
    float v = __bfloat162float(src[p * src_cpitch + c]);
    if (add) v += add[p * dst_cpitch + c];
    dst[p * dst_cpitch + c] = v;
  }
}
__global__ void f32_to_bf16_rowpad_kernel(const float* __restrict__ src, __nv_bfloat16* __restrict__ dst, long long npix,
                                          int C, int src_cpitch, int dst_cpitch) {
  long long total = npix * dst_cpitch;
  GRID_STRIDE(i, total) {
    long long p = i / dst_cpitch;
    int c = (int)(i - p * dst_cpitch);
    dst[i] = __float2bfloat16_rn(c < C ? src[p * src_cpitch + c] : 0.f);
  }
}

// Offset, in 4-channel groups, of full-resolution pixel (n, y, x) group c4 in the space-to-depth-2 image [N,H/2,W/2,4C]
// whose channel (py*2 + px)*C + c holds pixel (2i + py, 2j + px) channel c; g indexes the full-resolution image's groups.
__device__ __forceinline__ long long s2d2_group(long long g, int H, int W, int C4) {
  const long long p = g / C4;
  const int c4 = (int)(g - p * C4);
  const int x = (int)(p % W);
  const long long r = p / W;
  const int y = (int)(r % H);
  const long long n = r / H;
  return ((n * (H / 2) + (y >> 1)) * (W / 2) + (x >> 1)) * (4LL * C4) + ((y & 1) * 2 + (x & 1)) * C4 + c4;
}

__global__ void f32_to_bf16_s2d2_kernel(const float4* __restrict__ x, uint2* __restrict__ xs, long long groups, int H, int W,
                                        int C4) {
  GRID_STRIDE(g, groups) {
    const float4 v = x[g];
    __nv_bfloat162 lo = __floats2bfloat162_rn(v.x, v.y), hi = __floats2bfloat162_rn(v.z, v.w);
    uint2 o;
    o.x = *reinterpret_cast<uint32_t*>(&lo);
    o.y = *reinterpret_cast<uint32_t*>(&hi);
    xs[s2d2_group(g, H, W, C4)] = o;
  }
}

__global__ void bf16_d2s2_to_f32_kernel(const uint2* __restrict__ xs, float4* __restrict__ x, long long groups, int H, int W,
                                        int C4) {
  GRID_STRIDE(g, groups) {
    const uint2 v = xs[s2d2_group(g, H, W, C4)];
    const float2 lo = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.x));
    const float2 hi = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&v.y));
    x[g] = make_float4(lo.x, lo.y, hi.x, hi.y);
  }
}

int s2d2_check(const void* a, const void* b, int N, int H, int W, int C, const char* who) {
  TECO_CHECK_ARG(a && b && N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0 && C > 0 && C % 4 == 0,
                 "%s: needs even H, W and C a multiple of 4 (got N=%d H=%d W=%d C=%d)", who, N, H, W, C);
  TECO_CHECK_ARG((((uintptr_t)a) & 15) == 0 && (((uintptr_t)b) & 15) == 0, "%s: tensors must be 16-byte aligned", who);
  return TECO_OK;
}
}  // namespace

extern "C" int teco_f32_to_bf16_s2d2(const float* x, void* xs, int32_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  const int rc = s2d2_check(x, xs, N, H, W, C, "teco_f32_to_bf16_s2d2");
  if (rc != TECO_OK) return rc;
  const long long groups = (long long)N * H * W * (C / 4);
  f32_to_bf16_s2d2_kernel<<<grid_for(groups), TPB, 0, (cudaStream_t)stream>>>((const float4*)x, (uint2*)xs, groups, H, W, C / 4);
  TECO_CUDA_LAUNCH_CHECK("teco_f32_to_bf16_s2d2");
  return TECO_OK;
}

extern "C" int teco_bf16_d2s2_to_f32(const void* xs, float* x, int32_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  const int rc = s2d2_check(xs, x, N, H, W, C, "teco_bf16_d2s2_to_f32");
  if (rc != TECO_OK) return rc;
  const long long groups = (long long)N * H * W * (C / 4);
  bf16_d2s2_to_f32_kernel<<<grid_for(groups), TPB, 0, (cudaStream_t)stream>>>((const uint2*)xs, (float4*)x, groups, H, W, C / 4);
  TECO_CUDA_LAUNCH_CHECK("teco_bf16_d2s2_to_f32");
  return TECO_OK;
}

extern "C" int teco_bf16_to_f32_add(const void* src, const float* add, float* dst, int64_t npix, int32_t C,
                                    int32_t src_cpitch, int32_t dst_cpitch, void* stream) {
  TECO_CHECK_ARG(src && dst && npix > 0 && C > 0 && src_cpitch >= C && dst_cpitch >= C, "teco_bf16_to_f32_add: bad argument");
  bf16_to_f32_add_kernel<<<grid_for(npix * C), TPB, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)src, add, dst, npix, C,
                                                                            src_cpitch, dst_cpitch);
  TECO_CUDA_LAUNCH_CHECK("teco_bf16_to_f32_add");
  return TECO_OK;
}

extern "C" int teco_f32_to_bf16_rowpad(const float* src, void* dst, int64_t npix, int32_t C, int32_t src_cpitch,
                                       int32_t dst_cpitch, void* stream) {
  TECO_CHECK_ARG(src && dst && npix > 0 && C > 0 && src_cpitch >= C && dst_cpitch >= C, "teco_f32_to_bf16_rowpad: bad argument");
  f32_to_bf16_rowpad_kernel<<<grid_for(npix * dst_cpitch), TPB, 0, (cudaStream_t)stream>>>(src, (__nv_bfloat16*)dst, npix, C,
                                                                                        src_cpitch, dst_cpitch);
  TECO_CUDA_LAUNCH_CHECK("teco_f32_to_bf16_rowpad");
  return TECO_OK;
}
