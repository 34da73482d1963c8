// bf16 3x3 convolution / 3x3-stride-2 transposed convolution on the Hopper tensor cores (sm_90a):
// TMA halo tiles -> shared memory -> wgmma (m64nNk16, bf16 operands, fp32 accumulators in registers) -> register
// epilogue (bias, activation, residual, bf16 store; or fp32 "+bicubic, *2-1" output stage).
//
// Replaces, layer by layer, the cuDNN convolutions behind conv2()/conv2_tran() of the reference
// (lib/ops.py:35-56) as used by generator_F (lib/frvsr.py:44-88) and fnet (lib/frvsr.py:4-41).
//
// Implicit GEMM, no im2col buffer:
//   CTA tile  = 16 image rows x 8 pixels = 128 output pixels; warpgroup g (two per CTA) owns rows 8g..8g+7, i.e. one
//               M = 64 accumulator (8 image rows x 8 pixels).
//   A operand = NHWC bf16 activations, 64 channels = one 128-byte row per pixel.  Per 64-channel block the halo (18 rows x
//               10 pixels) is staged by ONE 4-D TMA box with SWIZZLE_128B; TMA out-of-bounds zero fill implements TF
//               'SAME' padding.  Tap (ky, kx) is the descriptor start address of halo row ky, pixel kx: 8 pixels of one
//               image row are one 8 x 128 B core-matrix group, SBO = one halo row (10 x 128 B).
//   B operand = weights pre-packed on the device as [cin/64][tap][cout][64 cin] bf16 in the same SW128 image, fetched by
//               1-D bulk copies: once per CTA when the layer's Cout slice fits next to the halo ring (every 64 -> 64 layer),
//               otherwise with each 64-channel block.
//   D         = fp32 registers, NT / 2 per thread per accumulator (NT = output channels per CTA: 64, 32 or 16).
// Transposed conv (stride 2, TF 'SAME', y[i] = sum_j x[j] w[i-2j]) is the same loop with the nine taps routed to four
// sub-pixel phase accumulators (SURVEY.md A.3) and a 2x interleaving epilogue.
//
// Persistent CTAs walk tiles c, c + G, ...; the halo (and weight) ring has two stages, so the TMA of the next 64-channel
// block or tile is in flight while the warpgroups run the MMAs and the epilogue of the current one.
#include <cuda.h>
#include "teco_common.cuh"
#include "tc_ptx.cuh"

namespace {

using namespace tcptx;

constexpr int TILE_ROWS = 16;
constexpr int TILE_COLS = 8;
constexpr int HALO_ROWS = TILE_ROWS + 2;
constexpr int HALO_COLS = TILE_COLS + 2;
constexpr int CB = 64;                                                 // channels per K block = one 128-byte swizzled row
constexpr uint32_t HALO_BYTES = HALO_ROWS * HALO_COLS * 128;           // 23040
constexpr uint32_t HALO_STAGE = (HALO_BYTES + 1023u) & ~1023u;         // 24576: stages stay 1024-byte aligned
constexpr int NUM_THREADS = 256;                                       // two warpgroups
constexpr size_t SMEM_MAX = 232448;                                    // 227 KB: opt-in maximum per block on sm_90

struct TcParams {
  int N, H, W, Cout;          // Cout = channel pitch of y / res / bias (all output channels)
  int nblk, act, out_f32_c;   // Cin / 64
  int tiles_x, tiles_y, num_tiles, resident;
  float post_scale, post_shift;
  uint32_t w_blk_bytes, stage_bytes;   // 9 taps x NT x 128 B; one ring stage (halo, + weights unless resident)
  const uint8_t* wpk;
  const float* bias;
  const __nv_bfloat16* res;
  __nv_bfloat16* y;
  const float* res_f32;
  float* out_f32;
};

// tap (ky, kx) -> halo offset (ry, rx) and accumulator.  Transposed conv: output pixel (2i + py, 2j + px) collects the taps
// with ky == 1 (py = 1) or ky in {0, 2} (py = 0), reading input row i (ky != 2) or i - 1 (ky == 2); the same for x.
template <int MODE>
__device__ __forceinline__ void tap_route(int t, int& ry, int& rx, int& ph) {
  const int ky = t / 3, kx = t % 3;
  if (MODE == 1) {
    ry = ky == 2 ? 0 : 1;
    rx = kx == 2 ? 0 : 1;
    ph = (ky == 1 ? 2 : 0) + (kx == 1 ? 1 : 0);
  } else {
    ry = ky; rx = kx; ph = 0;
  }
}

// The nine taps x four K-steps of one 64-channel block for warpgroup wg: halo stage at halo_a, the block's packed
// weights [tap][NT][64] at w_a.
template <int MODE, int NT, int NACC>
__device__ __forceinline__ void mma_block(float (&acc)[NACC][NT / 2], uint32_t halo_a, uint32_t w_a, int wg) {
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    int ry, rx, ph;
    tap_route<MODE>(t, ry, rx, ph);
    const uint32_t a0 = halo_a + (uint32_t)(((8 * wg + ry) * HALO_COLS + rx) * 128);
    const uint32_t b0 = w_a + (uint32_t)t * (uint32_t)NT * 128u;
#pragma unroll
    for (int k = 0; k < CB / 16; ++k)
      Wgmma<NT, 0, 0>::run(acc[ph], gmma_desc_sw128(a0 + 32u * k, 16u, HALO_COLS * 128u), gmma_desc_sw128(b0 + 32u * k, 16u, 1024u), 1u);
  }
  wgmma_commit();
  wgmma_wait_all();
}

// Epilogue of one tile: this thread holds pixels (row 8 wg + 2 wq + i, column lane / 4), channels 8 j + 2 (lane % 4) + {0, 1}
// of the NT-channel slice starting at n0.  bias points at that slice.
template <int MODE, int NT, int NACC>
__device__ __forceinline__ void epilogue(const float (&acc)[NACC][NT / 2], const TcParams& p, const float* bias, int n0, int n,
                                         int y0, int x0) {
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int ox_in = x0 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int oy_in = y0 + 8 * wg + 2 * wq + i;
    const bool in_img = oy_in < p.H && ox_in < p.W;
#pragma unroll
    for (int ph = 0; ph < NACC; ++ph) {
      const int OH = MODE == 1 ? 2 * p.H : p.H, OW = MODE == 1 ? 2 * p.W : p.W;
      const int oy = MODE == 1 ? 2 * oy_in + (ph >> 1) : oy_in, ox = MODE == 1 ? 2 * ox_in + (ph & 1) : ox_in;
      const size_t pix = ((size_t)n * OH + oy) * OW + ox;
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int c = 8 * j + 2 * (lane & 3);
        float v0 = teco_act(acc[ph][4 * j + 2 * i] + bias[c], p.act);
        float v1 = teco_act(acc[ph][4 * j + 2 * i + 1] + bias[c + 1], p.act);
        if (!in_img) continue;
        if (p.out_f32) {
          const int C = p.out_f32_c, ch = n0 + c;
          if (ch < C)
            p.out_f32[pix * C + ch] = (v0 + (p.res_f32 ? p.res_f32[pix * C + ch] : 0.f)) * p.post_scale + p.post_shift;
          if (ch + 1 < C)
            p.out_f32[pix * C + ch + 1] = (v1 + (p.res_f32 ? p.res_f32[pix * C + ch + 1] : 0.f)) * p.post_scale + p.post_shift;
        }
        if (p.y) {
          const size_t o = pix * p.Cout + n0 + c;
          if (p.res) {   // in-place residual (res == y) is safe: this thread reads the element before it writes it
            const float2 r = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(p.res + o));
            v0 += r.x;
            v1 += r.y;
          }
          *reinterpret_cast<__nv_bfloat162*>(p.y + o) = __floats2bfloat162_rn(v0, v1);
        }
      }
    }
  }
}

template <int MODE, int NT>
__global__ void __launch_bounds__(NUM_THREADS, MODE == 1 ? 1 : 2)
conv3x3_wgmma_kernel(const __grid_constant__ CUtensorMap tmap, const TcParams p) {
  constexpr int NACC = MODE == 1 ? 4 : 1;
  constexpr int NR = NT / 2;                    // accumulator registers per thread
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                                        // 2 stages
  uint8_t* w_res = smem + 2 * (size_t)p.stage_bytes;                           // resident weights, all blocks
  uint64_t* bars = reinterpret_cast<uint64_t*>(w_res + (p.resident ? (size_t)p.nblk * p.w_blk_bytes : 0));
  uint64_t* full = bars;                                                       // [2]
  uint64_t* w_full = bars + 2;
  float* s_bias = reinterpret_cast<float*>(bars + 4);                          // [NT]

  const int tid = threadIdx.x, wg = tid >> 7;
  const int n0 = blockIdx.y * NT;
  const int G = gridDim.x;
  const int my_tiles = (int)blockIdx.x < p.num_tiles ? (p.num_tiles - (int)blockIdx.x + G - 1) / G : 0;
  const int nsteps = my_tiles * p.nblk;

  for (int c = tid; c < NT; c += NUM_THREADS) s_bias[c] = p.bias ? p.bias[n0 + c] : 0.f;
  if (tid == 0) {
    mbar_init(smem_u32(&full[0]), 1);
    mbar_init(smem_u32(&full[1]), 1);
    mbar_init(smem_u32(w_full), 1);
    fence_mbar_init();
  }
  __syncthreads();

  auto tile_coords = [&](int it, int& n, int& y0, int& x0) {
    int tile = (int)blockIdx.x + it * G;
    const int tx = tile % p.tiles_x;
    tile /= p.tiles_x;
    const int ty = tile % p.tiles_y;
    n = tile / p.tiles_y;
    x0 = tx * TILE_COLS;
    y0 = ty * TILE_ROWS;
  };
  const uint32_t tap_bytes = (uint32_t)NT * 128u;
  // step s = (tile s / nblk, channel block s % nblk) into ring stage s & 1; issued by thread 0
  auto issue = [&](int s) {
    const int st = s & 1, it = s / p.nblk, b = s - it * p.nblk;
    int n, y0, x0;
    tile_coords(it, n, y0, x0);
    uint8_t* base = ring + (size_t)st * p.stage_bytes;
    const uint32_t bar = smem_u32(&full[st]);
    mbar_expect_tx(bar, HALO_BYTES + (p.resident ? 0u : p.w_blk_bytes));
    tma_load_4d(smem_u32(base), &tmap, bar, b * CB, x0 - 1, y0 - 1, n);
    if (!p.resident)
      for (int t = 0; t < 9; ++t)
        bulk_load_1d(smem_u32(base + HALO_STAGE + t * tap_bytes), p.wpk + ((size_t)(b * 9 + t) * p.Cout + n0) * 128, tap_bytes, bar);
  };
  if (tid == 0 && nsteps > 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap) : "memory");
    if (p.resident) {
      mbar_expect_tx(smem_u32(w_full), (uint32_t)p.nblk * p.w_blk_bytes);
      for (int bt = 0; bt < 9 * p.nblk; ++bt)
        bulk_load_1d(smem_u32(w_res + (size_t)bt * tap_bytes), p.wpk + ((size_t)bt * p.Cout + n0) * 128, tap_bytes, smem_u32(w_full));
    }
    issue(0);
  }
  if (p.resident && nsteps > 0) mbar_wait(smem_u32(w_full), 0);

  float acc[NACC][NR];
  for (int s = 0; s < nsteps; ++s) {
    const int it = s / p.nblk, b = s - it * p.nblk;
    if (tid == 0 && s + 1 < nsteps) issue(s + 1);   // its stage was released by the __syncthreads() closing step s - 1
    if (b == 0) {
#pragma unroll
      for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int r = 0; r < NR; ++r) acc[a][r] = 0.f;
    }
    mbar_wait(smem_u32(&full[s & 1]), (uint32_t)((s >> 1) & 1));
    uint8_t* base = ring + (size_t)(s & 1) * p.stage_bytes;
    const uint32_t halo_a = smem_u32(base);
    const uint32_t w_a = p.resident ? smem_u32(w_res + (size_t)b * p.w_blk_bytes) : smem_u32(base + HALO_STAGE);
    mma_block<MODE, NT, NACC>(acc, halo_a, w_a, wg);
    if (b == p.nblk - 1) {
      int n, y0, x0;
      tile_coords(it, n, y0, x0);
      epilogue<MODE, NT, NACC>(acc, p, s_bias, n0, n, y0, x0);
    }
    __syncthreads();   // every warpgroup's MMAs on this stage have completed: it may be refilled
  }
}

// ------------------------------------------------------------------ multi-layer chain (generator trunk)
// L consecutive 3x3 64 -> 64 layers (bias, ReLU / LeakyReLU / none, optional residual) on 32-pixel-wide images in ONE
// launch.  CTA c owns images c, c + G, ... for EVERY layer, so the input tiles of layer l + 1 were written by this very
// CTA: a CTA-wide barrier (after a generic -> async proxy fence, because the next layer's halo arrives by TMA) is the only
// dependency between layers, there is no grid-wide one and no kernel boundary.  Weights of layer l + 1 are in flight in
// the second weight buffer while layer l computes; within a layer the halo of the next tile is in flight while the
// current one runs its MMAs and epilogue.  Same MMA and epilogue code as conv3x3_wgmma_kernel.
constexpr int LIN_W = 32, LIN_ROWS = 4, LIN_MAX_LAYERS = 40;
constexpr uint32_t LAYER_W_BYTES = 9u * 64u * 128u;   // one packed 64 x 64 layer: 73728

struct ChainParams {
  int N, H, L, tiles_y;
  int8_t plan[LIN_MAX_LAYERS][4];   // input buffer, output buffer, residual buffer or -1, activation
  __nv_bfloat16* bufs[3];
  const uint8_t* wpk;
  const float* bias;
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
conv3x3_chain_kernel(const __grid_constant__ CUtensorMap tmap0, const __grid_constant__ CUtensorMap tmap1,
                     const __grid_constant__ CUtensorMap tmap2, const ChainParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                   // 2 halo stages
  uint8_t* wbuf = smem + 2 * HALO_STAGE;                  // 2 layers of weights
  uint64_t* full = reinterpret_cast<uint64_t*>(wbuf + 2 * LAYER_W_BYTES);   // [2]
  uint64_t* w_full = full + 2;                                              // [2]
  const int tid = threadIdx.x, wg = tid >> 7;
  const int G = gridDim.x;
  const int tiles_per_image = (LIN_W / TILE_COLS) * p.tiles_y;
  const int my_images = (int)blockIdx.x < p.N ? (p.N - (int)blockIdx.x + G - 1) / G : 0;
  const int T = my_images * tiles_per_image;              // tiles of this CTA per layer
  const int nsteps = p.L * T;

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(smem_u32(&full[i]), 1);
      mbar_init(smem_u32(&w_full[i]), 1);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (T == 0) return;

  auto tile_coords = [&](int it, int& n, int& y0, int& x0) {
    const int k = it / tiles_per_image, r = it - k * tiles_per_image;
    n = (int)blockIdx.x + k * G;
    x0 = (r % (LIN_W / TILE_COLS)) * TILE_COLS;
    y0 = (r / (LIN_W / TILE_COLS)) * TILE_ROWS;
  };
  auto issue = [&](int s) {     // halo of step s = (layer s / T, tile s % T) into ring stage s & 1
    const int l = s / T;
    int n, y0, x0;
    tile_coords(s - l * T, n, y0, x0);
    const int in = p.plan[l][0];
    const CUtensorMap* map = in == 0 ? &tmap0 : (in == 1 ? &tmap1 : &tmap2);
    const uint32_t bar = smem_u32(&full[s & 1]);
    mbar_expect_tx(bar, HALO_BYTES);
    tma_load_4d(smem_u32(ring + (size_t)(s & 1) * HALO_STAGE), map, bar, 0, x0 - 1, y0 - 1, n);
  };
  auto issue_weights = [&](int l) {   // layer l into weight buffer l & 1
    const uint32_t bar = smem_u32(&w_full[l & 1]);
    mbar_expect_tx(bar, LAYER_W_BYTES);
    for (int t = 0; t < 9; ++t)
      bulk_load_1d(smem_u32(wbuf + (size_t)(l & 1) * LAYER_W_BYTES + t * 8192u), p.wpk + (size_t)l * LAYER_W_BYTES + t * 8192u,
                   8192u, bar);
  };
  if (tid == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap2) : "memory");
    issue_weights(0);
    if (p.L > 1) issue_weights(1);
    issue(0);
  }

  TcParams q = {};
  q.H = p.H; q.W = LIN_W; q.Cout = 64;
  float acc[1][32];
  for (int s = 0; s < nsteps; ++s) {
    const int l = s / T, it = s - l * T;
    // the next tile of the same layer: its input does not change during this layer, its stage was released at the end of
    // step s - 1.  The first tile of the next layer waits for this layer's last outputs (below).
    if (tid == 0 && it + 1 < T) issue(s + 1);
    if (it == 0) mbar_wait(smem_u32(&w_full[l & 1]), (uint32_t)((l >> 1) & 1));
#pragma unroll
    for (int r = 0; r < 32; ++r) acc[0][r] = 0.f;
    mbar_wait(smem_u32(&full[s & 1]), (uint32_t)((s >> 1) & 1));
    mma_block<0, 64, 1>(acc, smem_u32(ring + (size_t)(s & 1) * HALO_STAGE), smem_u32(wbuf + (size_t)(l & 1) * LAYER_W_BYTES), wg);
    q.act = p.plan[l][3];
    q.y = p.bufs[p.plan[l][1]];
    q.res = p.plan[l][2] >= 0 ? p.bufs[p.plan[l][2]] : nullptr;
    int n, y0, x0;
    tile_coords(it, n, y0, x0);
    epilogue<0, 64, 1>(acc, q, p.bias + 64 * l, 0, n, y0, x0);
    if (it == T - 1) fence_proxy_async_global();   // this layer's stores -> visible to the next layer's TMA loads
    __syncthreads();
    if (tid == 0 && it == T - 1) {
      if (l + 2 < p.L) issue_weights(l + 2);         // buffer l & 1 is free: every MMA of layer l has completed
      if (s + 1 < nsteps) issue(s + 1);
    }
  }
}

// ------------------------------------------------------------------ weight packing
// out[blk][tap][cout_pad][64] bf16 in the SWIZZLE_128B image (16-byte chunk j of row r stored at chunk j ^ (r & 7))
//   <- w[3,3,cin,cout] (or [3,3,cout,cin] when transpose_layout); packed input channel k reads cin_perm[k] (-1 = zero).
__global__ void pack_conv3x3_kernel(const float* __restrict__ w, int cin, int cout, int cin_pad, int cout_pad,
                                    int transpose_layout, const int* __restrict__ cin_perm, __nv_bfloat16* __restrict__ out) {
  long long total = 9LL * cin_pad * cout_pad;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int e = (int)(i & 7);
    int jpos = (int)((i >> 3) & 7);
    long long t = i >> 6;
    int co = (int)(t % cout_pad);
    t /= cout_pad;
    int tap = (int)(t % 9);
    int blk = (int)(t / 9);
    int j = jpos ^ (co & 7);
    int ci = blk * 64 + j * 8 + e;
    int src_ci = cin_perm ? cin_perm[ci] : (ci < cin ? ci : -1);
    float v = 0.f;
    const int stap = (transpose_layout & 2) ? 8 - tap : tap;   // bit 1: spatially flipped taps (input-gradient convolution)
    if (src_ci >= 0 && src_ci < cin && co < cout)
      v = (transpose_layout & 1) ? w[((long long)stap * cout + co) * cin + src_ci] : w[((long long)stap * cin + src_ci) * cout + co];
    out[i] = __float2bfloat16_rn(v);
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

// NHWC bf16 activations [N,H,W,C] as a 4-D map whose box is one tile's halo of 64 channels (SWIZZLE_128B, zero fill)
int encode_halo_map(CUtensorMap* map, const void* x, int N, int H, int W, int C, const char* who) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    teco_set_error("%s: cuTensorMapEncodeTiled is unavailable (no CUDA driver?)", who);
    return TECO_E_CUDA;
  }
  const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t gstr[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)CB, (cuuint32_t)HALO_COLS, (cuuint32_t)HALO_ROWS, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult cr = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), gdim, gstr, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    teco_set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d (N=%d H=%d W=%d C=%d)", who, (int)cr, N, H, W, C);
    return TECO_E_CUDA;
  }
  return TECO_OK;
}

using KernelT = void (*)(const CUtensorMap, const TcParams);

KernelT pick_kernel(int mode, int nt) {
  if (mode == 1) return nt == 32 ? conv3x3_wgmma_kernel<1, 32> : conv3x3_wgmma_kernel<1, 16>;
  if (nt == 64) return conv3x3_wgmma_kernel<0, 64>;
  if (nt == 32) return conv3x3_wgmma_kernel<0, 32>;
  return conv3x3_wgmma_kernel<0, 16>;
}

// CTAs of `kern` resident per SM at `smem` bytes of dynamic shared memory; the opt-in shared-memory attribute is set on
// first use and the answer cached per (kernel, size), so a launch costs no extra driver calls.
int resident_ctas(const void* kern, size_t smem, int* per_sm) {
  struct Entry { const void* kern; size_t smem; int per_sm; };
  static Entry cache[32];
  static int used = 0;
  for (int i = 0; i < used; ++i)
    if (cache[i].kern == kern && cache[i].smem == smem) { *per_sm = cache[i].per_sm; return TECO_OK; }
  bool attr_set = false;
  for (int i = 0; i < used; ++i) attr_set |= cache[i].kern == kern;
  if (!attr_set) TECO_CUDA_CALL(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX));
  int n = 0;
  TECO_CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, NUM_THREADS, smem));
  if (n < 1) n = 1;
  if (used < 32) cache[used++] = {kern, smem, n};
  *per_sm = n;
  return TECO_OK;
}

int launch_conv3x3(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, const void* res, void* y,
                   const float* res_f32, float* out_f32, cudaStream_t stream) {
  TcParams p;
  p.N = d->N; p.H = d->H; p.W = d->W; p.Cout = d->Cout;
  p.act = d->act; p.out_f32_c = d->out_f32_c;
  p.post_scale = d->post_scale; p.post_shift = d->post_shift;
  p.wpk = (const uint8_t*)wpk; p.bias = bias; p.res = (const __nv_bfloat16*)res; p.y = (__nv_bfloat16*)y;
  p.res_f32 = res_f32; p.out_f32 = out_f32;
  p.nblk = d->Cin / CB;
  // output channels per CTA: 64, or 32 for the transposed conv, whose four phase accumulators must stay in registers
  const int nt = (d->Cout % 64 == 0 && d->mode == 0) ? 64 : (d->Cout % 32 == 0 ? 32 : 16);
  const int nsplit = d->Cout / nt;
  p.w_blk_bytes = 9u * (uint32_t)nt * 128u;
  p.tiles_x = teco_ceil_div(d->W, TILE_COLS);
  p.tiles_y = teco_ceil_div(d->H, TILE_ROWS);
  const long long tiles = (long long)d->N * p.tiles_x * p.tiles_y;
  TECO_CHECK_ARG(tiles < (1LL << 31), "teco_conv3x3_tc: too many tiles");
  p.num_tiles = (int)tiles;
  const size_t fixed = 1024 + 64 + (size_t)nt * sizeof(float);
  p.resident = fixed + 2 * (size_t)HALO_STAGE + (size_t)p.nblk * p.w_blk_bytes <= SMEM_MAX ? 1 : 0;
  p.stage_bytes = HALO_STAGE + (p.resident ? 0u : p.w_blk_bytes);
  const size_t smem = fixed + 2 * (size_t)p.stage_bytes + (p.resident ? (size_t)p.nblk * p.w_blk_bytes : 0);
  TECO_CHECK_ARG(smem <= SMEM_MAX, "teco_conv3x3_tc: shared memory budget exceeded (Cin=%d Cout=%d)", d->Cin, d->Cout);

  CUtensorMap tmap;
  const int rc = encode_halo_map(&tmap, x, d->N, d->H, d->W, d->Cin, "teco_conv3x3_tc");
  if (rc != TECO_OK) return rc;
  const KernelT kern = pick_kernel(d->mode, nt);
  int per_sm = 0;
  const int rc_occ = resident_ctas((const void*)kern, smem, &per_sm);
  if (rc_occ != TECO_OK) return rc_occ;
  // persistent: as many CTAs as are resident at once, spread over the Cout splits
  const long long slots = ((long long)per_sm * teco_sm_count() + nsplit - 1) / nsplit;
  const unsigned gx = (unsigned)(tiles < slots ? tiles : slots);
  kern<<<dim3(gx, (unsigned)nsplit), NUM_THREADS, smem, stream>>>(tmap, p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_tc");
  return TECO_OK;
}

}  // namespace

extern "C" int64_t teco_packed_weight_bytes(int32_t cin_pad, int32_t cout_pad) {
  return 9LL * cin_pad * cout_pad * 2;
}

extern "C" int teco_pack_conv3x3_bf16(const float* w, int32_t cin, int32_t cout, int32_t cin_pad, int32_t cout_pad,
                                      int32_t transpose_layout, const int32_t* cin_perm, void* wpk, void* stream) {
  TECO_CHECK_ARG(w && wpk, "teco_pack_conv3x3_bf16: NULL tensor");
  TECO_CHECK_ARG(cin > 0 && cout > 0 && cin_pad >= cin && cout_pad >= cout && (cin_pad % 64) == 0 && (cout_pad % 16) == 0,
                 "teco_pack_conv3x3_bf16: cin_pad must be a multiple of 64 and cout_pad a multiple of 16, both >= the real channels");
  long long total = 9LL * cin_pad * cout_pad;
  int blocks = teco_ceil_div(total, 256);
  if (blocks > 4096) blocks = 4096;
  pack_conv3x3_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, cin, cout, cin_pad, cout_pad, transpose_layout, cin_perm,
                                                                (__nv_bfloat16*)wpk);
  TECO_CUDA_LAUNCH_CHECK("teco_pack_conv3x3_bf16");
  return TECO_OK;
}

extern "C" int teco_conv3x3_tc(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, const void* res,
                               void* y, const float* res_f32, float* out_f32, void* stream) {
  TECO_CHECK_ARG(d && x && wpk, "teco_conv3x3_tc: NULL argument");
  TECO_CHECK_ARG(y || out_f32, "teco_conv3x3_tc: no output buffer");
  TECO_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0, "teco_conv3x3_tc: bad shape N=%d H=%d W=%d", d->N, d->H, d->W);
  TECO_CHECK_ARG(d->Cin >= 64 && d->Cin % 64 == 0 && d->Cin <= 512, "teco_conv3x3_tc: Cin must be a multiple of 64 in [64,512] (got %d)", d->Cin);
  TECO_CHECK_ARG(d->Cout >= 16 && d->Cout % 16 == 0 && d->Cout <= 512, "teco_conv3x3_tc: Cout must be a multiple of 16 in [16,512] (got %d)", d->Cout);
  TECO_CHECK_ARG(d->mode == 0 || d->mode == 1, "teco_conv3x3_tc: unknown mode %d", d->mode);
  TECO_CHECK_ARG(d->act >= 0 && d->act <= TECO_ACT_SIGMOID, "teco_conv3x3_tc: unknown activation %d", d->act);
  TECO_CHECK_ARG(!out_f32 || (d->out_f32_c > 0 && d->out_f32_c <= d->Cout), "teco_conv3x3_tc: bad out_f32_c");
  TECO_CHECK_ARG((((uintptr_t)x) & 15) == 0 && (((uintptr_t)wpk) & 15) == 0 && (((uintptr_t)y) & 15) == 0 &&
                     (((uintptr_t)res) & 15) == 0,
                 "teco_conv3x3_tc: tensors must be 16-byte aligned");
  return launch_conv3x3(d, x, wpk, bias, res, y, res_f32, out_f32, (cudaStream_t)stream);
}

extern "C" int teco_conv3x3_lin_supported(int32_t N, int32_t H, int32_t W, int32_t num_layers) {
  return (N > 0 && W == LIN_W && H >= LIN_ROWS && H % LIN_ROWS == 0 && H <= 4096 && num_layers >= 1 && num_layers <= LIN_MAX_LAYERS) ? 1 : 0;
}

extern "C" int teco_conv3x3_lin_tc(int32_t N, int32_t H, int32_t W, int32_t num_layers, const void* x_in, void* buf_a, void* buf_b,
                                   const void* wpk_all, const float* bias_all, const int32_t* plan_host, void* stream) {
  TECO_CHECK_ARG(teco_conv3x3_lin_supported(N, H, W, num_layers),
                 "teco_conv3x3_lin_tc: needs W == 32, H a multiple of 4, 1..%d layers (got N=%d H=%d W=%d L=%d)", LIN_MAX_LAYERS, N, H, W, num_layers);
  TECO_CHECK_ARG(x_in && buf_a && buf_b && wpk_all && bias_all && plan_host, "teco_conv3x3_lin_tc: NULL argument");
  TECO_CHECK_ARG((((uintptr_t)x_in) & 15) == 0 && (((uintptr_t)buf_a) & 15) == 0 && (((uintptr_t)buf_b) & 15) == 0 &&
                     (((uintptr_t)wpk_all) & 15) == 0,
                 "teco_conv3x3_lin_tc: tensors must be 16-byte aligned");
  ChainParams p = {};
  p.N = N; p.H = H; p.L = num_layers; p.tiles_y = teco_ceil_div(H, TILE_ROWS);
  for (int l = 0; l < num_layers; ++l) {
    const int32_t* pl = plan_host + 4 * l;
    TECO_CHECK_ARG(pl[0] >= 0 && pl[0] <= 2 && (pl[1] == 1 || pl[1] == 2) && pl[0] != pl[1] && pl[2] >= -1 && pl[2] <= 2 &&
                       pl[3] >= 0 && pl[3] < TECO_ACT_TANH24,
                   "teco_conv3x3_lin_tc: bad plan row %d {%d, %d, %d, %d}", l, pl[0], pl[1], pl[2], pl[3]);
    for (int k = 0; k < 4; ++k) p.plan[l][k] = (int8_t)pl[k];
  }
  p.bufs[0] = (__nv_bfloat16*)const_cast<void*>(x_in); p.bufs[1] = (__nv_bfloat16*)buf_a; p.bufs[2] = (__nv_bfloat16*)buf_b;
  p.wpk = (const uint8_t*)wpk_all; p.bias = bias_all;
  CUtensorMap maps[3];
  for (int i = 0; i < 3; ++i) {
    const int rc = encode_halo_map(&maps[i], p.bufs[i], N, H, LIN_W, 64, "teco_conv3x3_lin_tc");
    if (rc != TECO_OK) return rc;
  }
  const size_t smem = 1024 + 2 * (size_t)HALO_STAGE + 2 * (size_t)LAYER_W_BYTES + 64;
  int per_sm = 0;
  const int rc = resident_ctas((const void*)conv3x3_chain_kernel, smem, &per_sm);
  if (rc != TECO_OK) return rc;
  const long long slots = (long long)per_sm * teco_sm_count();
  const unsigned grid = (unsigned)(N < slots ? N : slots);
  conv3x3_chain_kernel<<<grid, NUM_THREADS, smem, (cudaStream_t)stream>>>(maps[0], maps[1], maps[2], p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_lin_tc");
  return TECO_OK;
}
