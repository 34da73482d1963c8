// fp32 direct convolution as an implicit GEMM on the CUDA cores (exact-parity path), plus the
// weight-gradient kernel.  Reference arithmetic replaced: slim.conv2d / slim.conv2d_transpose
// behind conv2()/conv2_tran() (reference lib/ops.py:35-56) and their TF autodiff gradients.
//
// Forward:  M = N*OH*OW output pixels, N = Cout, K = KH*KW*Cin.  CTA tile 64x64, BK = 16,
// 256 threads, 4x4 register tile per thread, register-prefetched double buffering.
#include "teco_common.cuh"

namespace {

constexpr int BM = 64, BN = 64, BK = 16, PADM = 4;

struct PixCoord {
  int n, iy0, ix0;
  bool valid;
};

__global__ void __launch_bounds__(256)
conv2d_f32_kernel(const teco_conv_desc d, const float* __restrict__ x, const float* __restrict__ w,
                  const float* __restrict__ bias, const float* __restrict__ res, float* __restrict__ y) {
  __shared__ __align__(16) float As[2][BK][BM + PADM];
  __shared__ __align__(16) float Bs[2][BK][BN + PADM];

  const int tid = threadIdx.x;
  const long long M = (long long)d.N * d.OH * d.OW;
  const long long m0 = (long long)blockIdx.x * BM;
  const int co0 = blockIdx.y * BN;

  // ---- loader roles
  const int a_m = tid >> 2;          // pixel within tile 0..63
  const int a_k = (tid & 3) * 4;     // cin sub-offset 0,4,8,12
  const int b_k = tid >> 4;          // 0..15
  const int b_n = (tid & 15) * 4;    // 0..60

  PixCoord pc;
  {
    long long pm = m0 + a_m;
    pc.valid = pm < M;
    long long t = pc.valid ? pm : 0;
    int ox = (int)(t % d.OW);
    t /= d.OW;
    int oy = (int)(t % d.OH);
    pc.n = (int)(t / d.OH);
    pc.iy0 = oy * d.stride - d.pad_t;
    pc.ix0 = ox * d.stride - d.pad_l;
  }
  const bool a_vec = ((d.Cin & 3) == 0) && ((d.in_cpitch & 3) == 0);
  const bool b_vec = ((d.Cout & 3) == 0);
  const int cchunks = (d.Cin + BK - 1) / BK;
  const int iters = d.KH * d.KW * cchunks;

  float4 a_reg, b_reg;
  auto load_tiles = [&](int it) {
    int tap = it / cchunks;
    int c0 = (it - tap * cchunks) * BK;
    int ky = tap / d.KW, kx = tap - ky * d.KW;
    // A
    a_reg = make_float4(0.f, 0.f, 0.f, 0.f);
    int iy = pc.iy0 + ky, ix = pc.ix0 + kx;
    if (pc.valid && iy >= 0 && iy < d.H && ix >= 0 && ix < d.W) {
      const float* p = x + (((long long)pc.n * d.H + iy) * d.W + ix) * d.in_cpitch + c0 + a_k;
      int c = c0 + a_k;
      if (a_vec && c + 3 < d.Cin) {
        a_reg = *reinterpret_cast<const float4*>(p);
      } else {
        if (c + 0 < d.Cin) a_reg.x = p[0];
        if (c + 1 < d.Cin) a_reg.y = p[1];
        if (c + 2 < d.Cin) a_reg.z = p[2];
        if (c + 3 < d.Cin) a_reg.w = p[3];
      }
    }
    // B
    b_reg = make_float4(0.f, 0.f, 0.f, 0.f);
    int ci = c0 + b_k;
    if (ci < d.Cin) {
      const float* p = w + ((long long)tap * d.Cin + ci) * d.Cout + co0 + b_n;
      int co = co0 + b_n;
      if (b_vec && co + 3 < d.Cout) {
        b_reg = *reinterpret_cast<const float4*>(p);
      } else {
        if (co + 0 < d.Cout) b_reg.x = p[0];
        if (co + 1 < d.Cout) b_reg.y = p[1];
        if (co + 2 < d.Cout) b_reg.z = p[2];
        if (co + 3 < d.Cout) b_reg.w = p[3];
      }
    }
  };
  auto store_tiles = [&](int buf) {
    As[buf][a_k + 0][a_m] = a_reg.x;
    As[buf][a_k + 1][a_m] = a_reg.y;
    As[buf][a_k + 2][a_m] = a_reg.z;
    As[buf][a_k + 3][a_m] = a_reg.w;
    *reinterpret_cast<float4*>(&Bs[buf][b_k][b_n]) = b_reg;
  };

  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int it = 0; it < iters; ++it) {
    int buf = it & 1;
    if (it + 1 < iters) load_tiles(it + 1);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (it + 1 < iters) store_tiles(buf ^ 1);
    __syncthreads();
  }

  // ---- epilogue
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    long long pm = m0 + ty * 4 + i;
    if (pm >= M) continue;
    long long t = pm;
    int ox = (int)(t % d.OW);
    t /= d.OW;
    int oy = (int)(t % d.OH);
    int n = (int)(t / d.OH);
    long long base = (((long long)n * d.out_H + (oy * d.out_sy + d.out_oy)) * d.out_W + (ox * d.out_sx + d.out_ox)) *
                     d.out_cpitch;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int co = co0 + tx * 4 + j;
      if (co >= d.Cout) continue;
      float v = acc[i][j] + (bias ? bias[co] : 0.f);
      v = teco_act(v, d.act);
      if (res) v += res[base + co];
      y[base + co] = v * d.post_scale + d.post_shift;
    }
  }
}

// ---------------------------------------------------------------------------------------
// Weight gradient: for one tap, GEMM [Cin x pixels] * [pixels x Cout], split over pixels
// (blockIdx.z) with fp32 atomics into dw.  grid = (ci tiles * taps, co tiles, splits).  With part != NULL split z stores
// its sums to part[z][tap][ci][co] instead (the fixed-order entry point reduces them in split order).
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
conv2d_wgrad_f32_kernel(const teco_conv_desc d, const float* __restrict__ x, const float* __restrict__ dy,
                        float* __restrict__ dw, int ci_tiles, long long pix_per_split, float* __restrict__ part) {
  __shared__ __align__(16) float As[BK][BM + PADM];  // [pixel][ci]
  __shared__ __align__(16) float Bs[BK][BN + PADM];  // [pixel][co]
  const int tid = threadIdx.x;
  const int tap = blockIdx.x / ci_tiles;
  const int ci0 = (blockIdx.x - tap * ci_tiles) * BM;
  const int co0 = blockIdx.y * BN;
  const int ky = tap / d.KW, kx = tap - ky * d.KW;
  const long long M = (long long)d.N * d.OH * d.OW;
  const long long p_begin = (long long)blockIdx.z * pix_per_split;
  const long long p_end = min(M, p_begin + pix_per_split);

  const int l_k = tid >> 4;         // pixel within chunk 0..15
  const int l_c = (tid & 15) * 4;   // channel offset 0..60
  const bool a_vec = ((d.Cin & 3) == 0) && ((d.in_cpitch & 3) == 0);
  const bool b_vec = ((d.Cout & 3) == 0) && ((d.out_cpitch & 3) == 0);
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (long long p0 = p_begin; p0 < p_end; p0 += BK) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    long long pm = p0 + l_k;
    if (pm < p_end) {
      long long t = pm;
      int ox = (int)(t % d.OW);
      t /= d.OW;
      int oy = (int)(t % d.OH);
      int n = (int)(t / d.OH);
      int iy = oy * d.stride - d.pad_t + ky, ix = ox * d.stride - d.pad_l + kx;
      if (iy >= 0 && iy < d.H && ix >= 0 && ix < d.W) {
        int c = ci0 + l_c;
        const float* p = x + (((long long)n * d.H + iy) * d.W + ix) * d.in_cpitch + c;
        if (a_vec && c + 3 < d.Cin) {
          a = *reinterpret_cast<const float4*>(p);
        } else {
          if (c + 0 < d.Cin) a.x = p[0];
          if (c + 1 < d.Cin) a.y = p[1];
          if (c + 2 < d.Cin) a.z = p[2];
          if (c + 3 < d.Cin) a.w = p[3];
        }
      }
      {
        int co = co0 + l_c;
        const float* p = dy + (((long long)n * d.out_H + (oy * d.out_sy + d.out_oy)) * d.out_W +
                               (ox * d.out_sx + d.out_ox)) * d.out_cpitch + co;
        if (b_vec && co + 3 < d.Cout) {
          b = *reinterpret_cast<const float4*>(p);
        } else {
          if (co + 0 < d.Cout) b.x = p[0];
          if (co + 1 < d.Cout) b.y = p[1];
          if (co + 2 < d.Cout) b.z = p[2];
          if (co + 3 < d.Cout) b.w = p[3];
        }
      }
    }
    __syncthreads();
    *reinterpret_cast<float4*>(&As[l_k][l_c]) = a;
    *reinterpret_cast<float4*>(&Bs[l_k][l_c]) = b;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float4 av4 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 bv4 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      float av[4] = {av4.x, av4.y, av4.z, av4.w}, bv[4] = {bv4.x, bv4.y, bv4.z, bv4.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int ci = ci0 + ty * 4 + i;
    if (ci >= d.Cin) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int co = co0 + tx * 4 + j;
      if (co >= d.Cout) continue;
      const long long e = ((long long)tap * d.Cin + ci) * d.Cout + co;
      if (part) part[(long long)blockIdx.z * d.KH * d.KW * d.Cin * d.Cout + e] = acc[i][j];
      else atomicAdd(&dw[e], acc[i][j]);
    }
  }
}

// db[c] += sum over pixels of dy[pixel, c] (dy addressed through the output mapping).  Threads are laid out
// channel-fastest (coalesced), 256 / C pixel lanes per block, shared-memory reduce, one atomic per channel per block
// (kDet: part[block][c] stored instead, every sum rounded explicitly).
// Many small blocks (16-64 pixels each): the first version gave a 4096-pixel layer 16 blocks of 64 serial iterations with
// two 64-bit divisions each and cost 46 us per call -- 27 % of an FRVSR training step.
template <bool kContig, bool kDet = false>
__global__ void __launch_bounds__(256)
bias_grad_kernel(const teco_conv_desc d, const float* __restrict__ dy, float* __restrict__ db, int pix_per_block,
                 float* __restrict__ part = nullptr) {
  __shared__ float lanes[256];
  const int M = d.N * d.OH * d.OW;
  const int p_begin = blockIdx.x * pix_per_block;
  const int p_end = min(M, p_begin + pix_per_block);
  const int C = d.Cout;
  const int ppar = 256 / C;                 // C <= 256
  const int c = threadIdx.x % C, ps = threadIdx.x / C;
  float s = 0.f;
  if (ps < ppar) {
    for (int pm = p_begin + ps; pm < p_end; pm += ppar) {
      if (kContig) {
        s = kDet ? __fadd_rn(s, dy[(size_t)pm * d.out_cpitch + c]) : s + dy[(size_t)pm * d.out_cpitch + c];
      } else {
        int t = pm;
        const int ox = t % d.OW;
        t /= d.OW;
        const int oy = t % d.OH;
        const int n = t / d.OH;
        const float v = dy[(((size_t)n * d.out_H + (oy * d.out_sy + d.out_oy)) * d.out_W + (ox * d.out_sx + d.out_ox)) * d.out_cpitch + c];
        s = kDet ? __fadd_rn(s, v) : s + v;
      }
    }
  }
  lanes[threadIdx.x] = s;
  __syncthreads();
  if (ps == 0) {
    if (kDet) {
      for (int k = 1; k < ppar; ++k) s = __fadd_rn(s, lanes[k * C + c]);
      part[(size_t)blockIdx.x * C + c] = s;
    } else {
      for (int k = 1; k < ppar; ++k) s += lanes[k * C + c];
      atomicAdd(&db[c], s);
    }
  }
}

// Fixed-order partitions (the *_det entry points): functions of the shapes alone.  The weight gradient splits the pixels
// as the default path does on a device of DET_SMS SMs; the bias gradient takes blocks of 8 * (256 / C) pixels, at most
// DET_BIAS_BLOCKS of them.
constexpr int DET_SMS = 132;
constexpr long long DET_BIAS_BLOCKS = 16LL * DET_SMS;

long long wgrad_splits(long long M, int base, int target, long long* pps) {
  long long splits = (target + base - 1) / base;
  long long max_splits = (M + 255) / 256;  // at least 256 pixels per split
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  if (splits > 65535) splits = 65535;
  *pps = (M + splits - 1) / splits;
  *pps = (*pps + BK - 1) / BK * BK;
  return (M + *pps - 1) / *pps;
}

long long det_bias_blocks(long long M, int C, int* ppb) {
  *ppb = 8 * (256 / C);
  long long blocks = (M + *ppb - 1) / *ppb;
  if (blocks > DET_BIAS_BLOCKS) { blocks = DET_BIAS_BLOCKS; *ppb = (int)((M + blocks - 1) / blocks); blocks = (M + *ppb - 1) / *ppb; }
  return blocks;
}

int check_desc(const teco_conv_desc* d, const char* who) {
  TECO_CHECK_ARG(d != nullptr, "%s: descriptor is NULL", who);
  TECO_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0 && d->Cin > 0 && d->Cout > 0 && d->OH > 0 && d->OW > 0,
                 "%s: non-positive dimension N=%d H=%d W=%d Cin=%d Cout=%d OH=%d OW=%d", who, d->N, d->H, d->W, d->Cin,
                 d->Cout, d->OH, d->OW);
  TECO_CHECK_ARG(d->KH > 0 && d->KW > 0 && d->stride > 0, "%s: bad kernel/stride", who);
  TECO_CHECK_ARG(d->in_cpitch >= d->Cin && d->out_cpitch >= d->Cout, "%s: channel pitch smaller than channels", who);
  TECO_CHECK_ARG(d->out_sy > 0 && d->out_sx > 0 && d->out_oy >= 0 && d->out_ox >= 0 &&
                     (d->OH - 1) * d->out_sy + d->out_oy < d->out_H && (d->OW - 1) * d->out_sx + d->out_ox < d->out_W,
                 "%s: output mapping exceeds out_H/out_W", who);
  return TECO_OK;
}

}  // namespace

extern "C" int teco_conv2d_f32(const teco_conv_desc* d, const float* x, const float* w, const float* bias,
                               const float* res, float* y, void* stream) {
  int rc = check_desc(d, "teco_conv2d_f32");
  if (rc) return rc;
  TECO_CHECK_ARG(x && w && y, "teco_conv2d_f32: NULL tensor");
  TECO_CHECK_ARG(d->act >= 0 && d->act <= TECO_ACT_SIGMOID, "teco_conv2d_f32: unknown activation %d", d->act);
  long long M = (long long)d->N * d->OH * d->OW;
  dim3 grid(teco_ceil_div(M, BM), teco_ceil_div(d->Cout, BN));
  conv2d_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(*d, x, w, bias, res, y);
  TECO_CUDA_LAUNCH_CHECK("teco_conv2d_f32");
  return TECO_OK;
}

extern "C" int teco_conv2d_wgrad_f32(const teco_conv_desc* d, const float* x, const float* dy, float* dw, float* db,
                                     int accumulate, void* stream) {
  int rc = check_desc(d, "teco_conv2d_wgrad_f32");
  if (rc) return rc;
  TECO_CHECK_ARG(x && dy && dw, "teco_conv2d_wgrad_f32: NULL tensor");
  cudaStream_t s = (cudaStream_t)stream;
  long long M = (long long)d->N * d->OH * d->OW;
  // Every check comes before the first write: a rejected call leaves dw and db as they were.
  if (db) {
    TECO_CHECK_ARG(d->Cout <= 256, "teco_conv2d_wgrad_f32: bias gradient supports Cout <= 256 (got %d)", d->Cout);
    TECO_CHECK_ARG(M < (1LL << 31), "teco_conv2d_wgrad_f32: too many output pixels for the bias gradient");
  }
  if (!accumulate) {
    TECO_CUDA_CALL(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)d->KH * d->KW * d->Cin * d->Cout, s));
    if (db) TECO_CUDA_CALL(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)d->Cout, s));
  }
  int ci_tiles = teco_ceil_div(d->Cin, BM);
  int co_tiles = teco_ceil_div(d->Cout, BN);
  int base = ci_tiles * d->KH * d->KW * co_tiles;
  long long pps;
  const long long splits = wgrad_splits(M, base, 4 * teco_sm_count(), &pps);
  dim3 grid(ci_tiles * d->KH * d->KW, co_tiles, (unsigned)splits);
  conv2d_wgrad_f32_kernel<<<grid, 256, 0, s>>>(*d, x, dy, dw, ci_tiles, pps, nullptr);
  TECO_CUDA_LAUNCH_CHECK("teco_conv2d_wgrad_f32");
  if (db) {
    const int ppar = 256 / d->Cout;
    int ppb = 8 * ppar;                                          // eight pixels per thread
    long long blocks = (M + ppb - 1) / ppb;
    if (blocks > 16LL * teco_sm_count()) { blocks = 16LL * teco_sm_count(); ppb = (int)((M + blocks - 1) / blocks); blocks = (M + ppb - 1) / ppb; }
    const bool contig = d->out_sy == 1 && d->out_sx == 1 && d->out_oy == 0 && d->out_ox == 0 && d->out_H == d->OH && d->out_W == d->OW;
    if (contig) bias_grad_kernel<true><<<(unsigned)blocks, 256, 0, s>>>(*d, dy, db, ppb);
    else bias_grad_kernel<false><<<(unsigned)blocks, 256, 0, s>>>(*d, dy, db, ppb);
    TECO_CUDA_LAUNCH_CHECK("teco_conv2d_wgrad_f32(bias)");
  }
  return TECO_OK;
}

extern "C" int teco_bias_grad_f32(const float* dy, float* db, int64_t npix, int32_t C, int32_t cpitch, int32_t accumulate, void* stream) {
  TECO_CHECK_ARG(dy && db && npix > 0 && C > 0 && C <= 256 && cpitch >= C && npix < (1LL << 31), "teco_bias_grad_f32: bad argument");
  cudaStream_t s = (cudaStream_t)stream;
  if (!accumulate) TECO_CUDA_CALL(cudaMemsetAsync(db, 0, sizeof(float) * (size_t)C, s));
  teco_conv_desc d = {};
  d.N = 1; d.OH = 1; d.OW = (int)npix; d.Cout = C; d.out_cpitch = cpitch;
  const int ppar = 256 / C;
  int ppb = 8 * ppar;
  long long blocks = (npix + ppb - 1) / ppb;
  if (blocks > 16LL * teco_sm_count()) { blocks = 16LL * teco_sm_count(); ppb = (int)((npix + blocks - 1) / blocks); blocks = (npix + ppb - 1) / ppb; }
  bias_grad_kernel<true><<<(unsigned)blocks, 256, 0, s>>>(d, dy, db, ppb);
  TECO_CUDA_LAUNCH_CHECK("teco_bias_grad_f32");
  return TECO_OK;
}

// ---------------------------------------------------------------------------------------------------
// Fixed-order weight and bias gradients.  Workspace: [splits][KH][KW][Cin][Cout] fp32 partials of the weight gradient,
// then (db != NULL) [blocks][Cout] partials of the bias gradient; each is summed in split order into dw / db.
namespace {
struct WgradDetPlan {
  long long splits, pps, bias_blocks, w_floats, bytes;
  int ci_tiles, co_tiles, ppb;
};
WgradDetPlan wgrad_det_plan(const teco_conv_desc* d, bool with_bias) {
  WgradDetPlan p;
  const long long M = (long long)d->N * d->OH * d->OW;
  p.ci_tiles = teco_ceil_div(d->Cin, BM);
  p.co_tiles = teco_ceil_div(d->Cout, BN);
  p.splits = wgrad_splits(M, p.ci_tiles * d->KH * d->KW * p.co_tiles, 4 * DET_SMS, &p.pps);
  p.w_floats = (long long)d->KH * d->KW * d->Cin * d->Cout;
  p.bias_blocks = with_bias ? det_bias_blocks(M, d->Cout, &p.ppb) : 0;
  p.bytes = (p.splits * p.w_floats + p.bias_blocks * d->Cout) * (long long)sizeof(float);
  return p;
}

int bias_grad_det_launch(const teco_conv_desc& d, const float* dy, float* db, long long blocks, int ppb, float* part,
                         int accumulate, cudaStream_t s) {
  const bool contig = d.out_sy == 1 && d.out_sx == 1 && d.out_oy == 0 && d.out_ox == 0 && d.out_H == d.OH && d.out_W == d.OW;
  if (contig) bias_grad_kernel<true, true><<<(unsigned)blocks, 256, 0, s>>>(d, dy, db, ppb, part);
  else bias_grad_kernel<false, true><<<(unsigned)blocks, 256, 0, s>>>(d, dy, db, ppb, part);
  TECO_CUDA_LAUNCH_CHECK("bias_grad_kernel(det)");
  return teco_reduce_splits(part, (int)blocks, d.Cout, db, accumulate, s);
}
}  // namespace

#define DET_WS_CHECK(who, need) \
  TECO_CHECK_ARG(ws && ws_bytes >= (int64_t)(need) && (((uintptr_t)ws) & 15) == 0, \
                 "%s: workspace of %lld bytes (16-byte aligned) needed, got %lld", who, (long long)(need), (long long)ws_bytes)

extern "C" int teco_conv2d_wgrad_f32_det_plan_bytes(const teco_conv_desc* d, int32_t with_bias, int64_t* ws_bytes_host) {
  int rc = check_desc(d, "teco_conv2d_wgrad_f32_det_plan_bytes");
  if (rc) return rc;
  TECO_CHECK_ARG(ws_bytes_host, "teco_conv2d_wgrad_f32_det_plan_bytes: NULL output");
  TECO_CHECK_ARG(!with_bias || d->Cout <= 256, "teco_conv2d_wgrad_f32_det_plan_bytes: bias gradient supports Cout <= 256");
  *ws_bytes_host = wgrad_det_plan(d, with_bias != 0).bytes;
  return TECO_OK;
}

extern "C" int teco_conv2d_wgrad_f32_det(const teco_conv_desc* d, const float* x, const float* dy, float* dw, float* db,
                                         int32_t accumulate, void* ws, int64_t ws_bytes, void* stream) {
  int rc = check_desc(d, "teco_conv2d_wgrad_f32_det");
  if (rc) return rc;
  TECO_CHECK_ARG(x && dy && dw, "teco_conv2d_wgrad_f32_det: NULL tensor");
  const long long M = (long long)d->N * d->OH * d->OW;
  if (db) {
    TECO_CHECK_ARG(d->Cout <= 256, "teco_conv2d_wgrad_f32_det: bias gradient supports Cout <= 256 (got %d)", d->Cout);
    TECO_CHECK_ARG(M < (1LL << 31), "teco_conv2d_wgrad_f32_det: too many output pixels for the bias gradient");
  }
  const WgradDetPlan p = wgrad_det_plan(d, db != nullptr);
  DET_WS_CHECK("teco_conv2d_wgrad_f32_det", p.bytes);
  cudaStream_t s = (cudaStream_t)stream;
  float* part = (float*)ws;
  dim3 grid(p.ci_tiles * d->KH * d->KW, p.co_tiles, (unsigned)p.splits);
  conv2d_wgrad_f32_kernel<<<grid, 256, 0, s>>>(*d, x, dy, dw, p.ci_tiles, p.pps, part);
  TECO_CUDA_LAUNCH_CHECK("teco_conv2d_wgrad_f32_det");
  rc = teco_reduce_splits(part, (int)p.splits, p.w_floats, dw, accumulate, s);
  if (rc || !db) return rc;
  return bias_grad_det_launch(*d, dy, db, p.bias_blocks, p.ppb, part + p.splits * p.w_floats, accumulate, s);
}

extern "C" int teco_bias_grad_f32_det_plan_bytes(int64_t npix, int32_t C, int64_t* ws_bytes_host) {
  TECO_CHECK_ARG(ws_bytes_host && npix > 0 && C > 0 && C <= 256 && npix < (1LL << 31), "teco_bias_grad_f32_det_plan_bytes: bad argument");
  int ppb;
  *ws_bytes_host = det_bias_blocks(npix, C, &ppb) * C * (int64_t)sizeof(float);
  return TECO_OK;
}

extern "C" int teco_bias_grad_f32_det(const float* dy, float* db, int64_t npix, int32_t C, int32_t cpitch, int32_t accumulate,
                                      void* ws, int64_t ws_bytes, void* stream) {
  TECO_CHECK_ARG(dy && db && npix > 0 && C > 0 && C <= 256 && cpitch >= C && npix < (1LL << 31), "teco_bias_grad_f32_det: bad argument");
  int ppb;
  const long long blocks = det_bias_blocks(npix, C, &ppb);
  DET_WS_CHECK("teco_bias_grad_f32_det", blocks * C * sizeof(float));
  teco_conv_desc d = {};
  d.N = 1; d.OH = 1; d.OW = (int)npix; d.Cout = C; d.out_cpitch = cpitch;
  d.out_H = 1; d.out_W = (int)npix; d.out_sy = 1; d.out_sx = 1;
  return bias_grad_det_launch(d, dy, db, blocks, ppb, (float*)ws, accumulate, (cudaStream_t)stream);
}
