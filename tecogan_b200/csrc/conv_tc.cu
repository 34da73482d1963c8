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
//   D         = fp32 registers, NT / 2 per thread (NT = output channels per CTA: 64, 32 or 16).
//
// Persistent CTAs walk tiles c, c + G, ...; the halo (and weight) ring has two stages, so the TMA of the next 64-channel
// block or tile is in flight while the warpgroups run the MMAs and the epilogue of the current one.  Layers with one
// 64-channel input block and 64-channel bf16 output slices run on conv3x3_ws_kernel<0> instead: the same MMAs and
// epilogue arithmetic behind a producer warp, a deeper ring and TMA-staged residuals and stores.
// The transposed conv (mode 1: stride 2, TF 'SAME', y[i] = sum_j x[j] w[i-2j]) runs only on conv3x3_ws_kernel<1>: the
// same MMAs with the nine taps routed to four sub-pixel phase accumulators (SURVEY.md A.3) and a 2x interleaving
// epilogue, for Cin = 64, 64-channel bf16 output slices and no residual.  teco_conv3x3_tc refuses any other mode-1 launch.
// The fp32 output stage (Cin = 64, Cout = 16, two or three fp32 channels) has its own entry point,
// teco_conv3x3_f32out_tc, on conv3x3_f32out_kernel: the same MMAs and epilogue arithmetic, pipelined the same way.
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
// weights [tap][NT][64] at w_a.  Issues and commits them; mma_block() also waits for them.  ZERO_INIT: the first MMA
// into each accumulator ignores its old contents (scale-d = 0) instead of the caller zeroing the registers.  Zeroing four
// accumulators in registers made ptxas interleave the zeroing moves with the MMAs and serialise every wgmma.
// KL < 4 issues only K-steps 0 .. KL - 1 of each tap, in the same order: for an input whose channels from 16 KL on are
// zero, the steps left out would add only zero products.
template <int MODE, int NT, int NACC, bool ZERO_INIT = false, int KL = CB / 16>
__device__ __forceinline__ void mma_issue(float (&acc)[NACC][NT / 2], uint32_t halo_a, uint32_t w_a, int wg) {
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    int ry, rx, ph;
    tap_route<MODE>(t, ry, rx, ph);
    bool first = true;                        // no earlier tap feeds accumulator ph
#pragma unroll
    for (int u = 0; u < t; ++u) {
      int uy, ux, uph;
      tap_route<MODE>(u, uy, ux, uph);
      first &= uph != ph;
    }
    const uint32_t a0 = halo_a + (uint32_t)(((8 * wg + ry) * HALO_COLS + rx) * 128);
    const uint32_t b0 = w_a + (uint32_t)t * (uint32_t)NT * 128u;
#pragma unroll
    for (int k = 0; k < KL; ++k)
      Wgmma<NT, 0, 0>::run(acc[ph], gmma_desc_sw128(a0 + 32u * k, 16u, HALO_COLS * 128u), gmma_desc_sw128(b0 + 32u * k, 16u, 1024u),
                           ZERO_INIT && first && k == 0 ? 0u : 1u);
  }
  wgmma_commit();
}

template <int NT>
__device__ __forceinline__ void mma_block(float (&acc)[1][NT / 2], uint32_t halo_a, uint32_t w_a, int wg) {
  mma_issue<0, NT, 1>(acc, halo_a, w_a, wg);
  wgmma_wait_all();
}

// Epilogue of one tile: this thread holds pixels (row 8 wg + 2 wq + i, column lane / 4), channels 8 j + 2 (lane % 4) + {0, 1}
// of the NT-channel slice starting at n0.  bias points at that slice.
template <int NT>
__device__ __forceinline__ void epilogue(const float (&acc)[NT / 2], const TcParams& p, const float* bias, int n0, int n,
                                         int y0, int x0) {
  const int tid = threadIdx.x, wg = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;
  const int ox = x0 + (lane >> 2);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int oy = y0 + 8 * wg + 2 * wq + i;
    const bool in_img = oy < p.H && ox < p.W;
    const size_t pix = ((size_t)n * p.H + oy) * p.W + ox;
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      float v0 = teco_act(acc[4 * j + 2 * i] + bias[c], p.act);
      float v1 = teco_act(acc[4 * j + 2 * i + 1] + bias[c + 1], p.act);
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

template <int NT>
__global__ void __launch_bounds__(NUM_THREADS, 2)
conv3x3_wgmma_kernel(const __grid_constant__ CUtensorMap tmap, const TcParams p) {
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

  float acc[1][NR];
  for (int s = 0; s < nsteps; ++s) {
    const int it = s / p.nblk, b = s - it * p.nblk;
    if (tid == 0 && s + 1 < nsteps) issue(s + 1);   // its stage was released by the __syncthreads() closing step s - 1
    if (b == 0) {
#pragma unroll
      for (int r = 0; r < NR; ++r) acc[0][r] = 0.f;
    }
    mbar_wait(smem_u32(&full[s & 1]), (uint32_t)((s >> 1) & 1));
    uint8_t* base = ring + (size_t)(s & 1) * p.stage_bytes;
    const uint32_t halo_a = smem_u32(base);
    const uint32_t w_a = p.resident ? smem_u32(w_res + (size_t)b * p.w_blk_bytes) : smem_u32(base + HALO_STAGE);
    mma_block<NT>(acc, halo_a, w_a, wg);
    if (b == p.nblk - 1) {
      int n, y0, x0;
      tile_coords(it, n, y0, x0);
      epilogue<NT>(acc[0], p, s_bias, n0, n, y0, x0);
    }
    __syncthreads();   // every warpgroup's MMAs on this stage have completed: it may be refilled
  }
}

// teco_conv3x3_lin_tc: chains of 3x3 64 -> 64 layers on 32 x 32 images
constexpr int LIN_W = 32, LIN_MAX_LAYERS = 40;
constexpr uint32_t LAYER_W_BYTES = 9u * 64u * 128u;   // one packed 64 x 64 layer: 73728

// ------------------------------------------------------------------ warp-specialised 64 -> 64 layer (one K block)
// Mode 0, Cin = 64, 64 output channels per CTA, bf16 output: the generator trunk, FNet's 64-channel layers and the
// 64-input-channel training convolutions.  The CTA tile (16 rows x 8 pixels), the products with their tap and K order,
// and the epilogue arithmetic are those of conv3x3_wgmma_kernel; what differs:
//   - the MMA operands are swapped, D[cout][pixel] = W_tap[cout][cin] X[cin][pixel] (mma_issue_tile): M = the 64 output
//     channels, A = the resident weight tap; N = the tile's 128 pixels, B = the halo at the tap's offset.  One
//     m64n128k16 reads 6 KB of shared-memory operands for 131072 MACs, where two m64n64k16 with the pixels as A read
//     8 KB, and at the tensor rate those reads alone would take all of the SM's shared-memory bandwidth;
//   - one consumer warpgroup owns a whole tile (64 accumulator registers per thread); the two take alternate tiles of the
//     CTA's walk;
//   - one producer warp bulk-copies the weights once and TMA-loads the halo of each tile into a WS_STAGES-deep ring; a
//     stage is refilled once the warps that read it have arrived on its `empty` barrier after their MMAs completed;
//   - the two consumer warpgroups alternate in *issuing* MMAs (named barriers 1 and 2): the warpgroup of tile k + 1 may
//     issue once the warpgroup of tile k has issued (not completed) its MMAs.  The barriers order only the issue; the
//     tensor pipe runs the two issue streams one after the other, so while it works on one warpgroup's MMAs the other,
//     its own MMAs complete, runs its epilogue.  The epilogues themselves are not ordered against each other;
//   - the epilogue does not wait on global loads or stores: each warpgroup has WS_OUT_BUFS SW128 staging tiles for its
//     output box (one tile, 16 rows x 8 pixels x 64 channels), used by its tiles in turn.  The residual box of its next
//     tile is TMA-loaded into the next staging tile while the MMAs of this one run, once the store of its previous tile
//     has read that staging tile; the epilogue overwrites the residual with the bf16 result and one TMA tensor store
//     writes it out (clipped at the image edges).  In-place residuals (res == y) are safe: each box is read and written
//     by one warpgroup of one CTA only, the load completing before the store is issued.
// MODE 1 (the transposed convolution) runs the same producer, ring, turn-taking and stores with the unswapped MMAs:
// both warpgroups work on every tile, warpgroup g on input rows 8g .. 8g + 7 with the four phase accumulators of
// mma_issue<1, 64, 4>.  Its 8 x 8 input pixels are a 16 x 16 pixel box of the interleaved 2H x 2W output, 32 KB, staged
// in one SW128 tile per warpgroup and written by one TMA store; there is no residual.
constexpr int WS_THREADS = NUM_THREADS + 32;          // two consumer warpgroups + the producer warp

template <int MODE>
struct WsCfg {
  static constexpr int S = MODE == 1 ? 2 : 1;                    // output pixels per input pixel, per axis
  static constexpr int NACC = S * S;                             // phase accumulators
  static constexpr int NR = MODE == 1 ? 32 : 64;                 // registers per accumulator and thread
  static constexpr int WARPS_PER_STAGE = MODE == 1 ? 8 : 4;      // consumer warps that read each halo stage
  static constexpr int STAGES = 3;                               // halo ring depth
  static constexpr int OUT_BUFS = MODE == 1 ? 1 : 2;             // staging tiles per warpgroup
  static constexpr int BOX_ROWS = TILE_ROWS, BOX_COLS = S * TILE_COLS;   // one warpgroup's output box
  static constexpr uint32_t OUT_BYTES = BOX_ROWS * BOX_COLS * 128;
  static constexpr size_t SMEM = 1024 + STAGES * (size_t)HALO_STAGE + LAYER_W_BYTES + 2 * OUT_BUFS * (size_t)OUT_BYTES +
                                 (2 * STAGES + 1 + 2 * OUT_BUFS) * sizeof(uint64_t) + 64 * sizeof(float);
  static_assert(SMEM <= SMEM_MAX, "conv3x3_ws_kernel: shared memory budget");
};

// MODE 0, one warpgroup per tile: the nine taps x four K-steps of mma_issue<0, …> with the operands swapped, A = weight
// tap t ([64 cout][64 cin], SBO = 8 rows of 128 B), B = the halo from (ky, kx) (8-pixel groups one halo row apart).  The
// first MMA runs with scale-d = 0.  Issues and commits them.  KL: K-steps per tap, as in mma_issue.
template <int KL>
__device__ __forceinline__ void mma_issue_tile(float (&acc)[64], uint32_t halo_a, uint32_t w_a) {
  wgmma_fence();
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const uint32_t a0 = w_a + (uint32_t)t * 64u * 128u;
    const uint32_t b0 = halo_a + (uint32_t)(((t / 3) * HALO_COLS + t % 3) * 128);
#pragma unroll
    for (int k = 0; k < KL; ++k)
      Wgmma<128, 0, 0>::run(acc, gmma_desc_sw128(a0 + 32u * k, 16u, 1024u), gmma_desc_sw128(b0 + 32u * k, 16u, HALO_COLS * 128u),
                            t == 0 && k == 0 ? 0u : 1u);
  }
  wgmma_commit();
}

// Epilogue of one warpgroup's box into its staging tile at out_a: bias -> activation -> (+ the residual already in the
// staging tile) -> bf16, the same fp32 operations as epilogue().  The box's pixel p (row p / 8 S, column p % 8 S) is the
// 128-byte row p of the tile; channel chunk q of it is stored at chunk q ^ (p & 7) (SWIZZLE_128B: the box is 8 S pixels
// wide, so p & 7 is the column's row index within its 1024-byte atom).
//   MODE 0: the thread holds channels 16 wq + lane / 4 + 8 i (bias b[i]) of pixels 8 j + 2 (lane % 4) + {0, 1}, i.e. of
//     tile row j.  Matrix (j, i), pixels 8 j .. 8 j + 7 by chunk 2 wq + i, is one 8 x 8 matrix of the transposed
//     ldmatrix / stmatrix; one x4 moves rows j, j + 1 of both chunks, each matrix conflict-free.
//   MODE 1: the thread holds input pixel (row 2 wq + i, column lane / 4) of the box, channels 8 j + 2 (lane % 4) + {0, 1};
//     accumulator ph goes to box pixel (S (2 wq + i) + ph / 2, S col + ph % 2).  A 4-byte store instruction's eight
//     columns hit four chunks, two lanes per bank.  There is no residual.
template <int ACT, int MODE, int NACC, int NR>
__device__ __forceinline__ void ws_epilogue(const float (&acc)[NACC][NR], const float* s_bias, const float (&b)[2],
                                            uint32_t out_a, bool res, int wq, int lane) {
  if constexpr (MODE == 0) {
    const int q = 2 * wq + ((lane >> 3) & 1);                        // lane supplies row lane % 8 of matrix lane / 8
    const uint32_t row_a = out_a + (uint32_t)((8 * (lane >> 4) + (lane & 7)) * 128 + ((q ^ (lane & 7)) << 4));
#pragma unroll
    for (int jj = 0; jj < TILE_ROWS / 2; ++jj) {
      const uint32_t a = row_a + (uint32_t)jj * 2u * TILE_COLS * 128u;
      uint32_t r[4];
      if (res) ldmatrix_x4_trans(r, a);
#pragma unroll
      for (int m = 0; m < 4; ++m) {                                  // matrix m = (row 2 jj + m / 2, chunk 2 wq + m % 2)
        const int j = 2 * jj + (m >> 1), i = m & 1;
        float v0 = teco_act(acc[0][4 * j + 2 * i] + b[i], ACT);
        float v1 = teco_act(acc[0][4 * j + 2 * i + 1] + b[i], ACT);
        if (res) {
          const float2 rf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&r[m]));
          v0 += rf.x;
          v1 += rf.y;
        }
        const __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
        r[m] = *reinterpret_cast<const uint32_t*>(&o);
      }
      stmatrix_x4_trans(a, r);
    }
  } else {
    constexpr int S = WsCfg<MODE>::S;
    const int col = lane >> 2;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int ph = 0; ph < NACC; ++ph) {
        const int oy = S * (2 * wq + i) + (ph >> 1), ox = S * col + (ph & 1);
        const uint32_t px = out_a + (uint32_t)((oy * 8 * S + ox) * 128 + 4 * (lane & 3));
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + 2 * (lane & 3);
          const float v0 = teco_act(acc[ph][4 * j + 2 * i] + s_bias[c], ACT);
          const float v1 = teco_act(acc[ph][4 * j + 2 * i + 1] + s_bias[c + 1], ACT);
          const __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
          const uint32_t e = px + (uint32_t)((j ^ (ox & 7)) << 4);
          asm volatile("st.shared.b32 [%0], %1;" ::"r"(e), "r"(*reinterpret_cast<const uint32_t*>(&o)) : "memory");
        }
      }
    }
  }
}

// MODE 0 followed by a 2x2 max-pool, into an 8 x 4 pixel box of the half-resolution output.  The thread's values of tile
// rows 2 jj, 2 jj + 1 and columns 2 (lane % 4) + {0, 1} are one pooling window for each of its channels 16 wq + lane / 4
// + 8 i.  Each value is rounded to bf16 as ws_epilogue stores it, and the window's max is taken as maxpool2_bf16_kernel
// takes it: max(max(TL, TR), max(BL, BR)) by __hmax2, channel i in half i of the pair.  Pooled pixel P = 4 jj + lane % 4
// is the 128-byte row P of the staging tile, channel chunk q stored at chunk q ^ (P & 7).
template <int ACT>
__device__ __forceinline__ void ws_epilogue_pool(const float (&acc)[64], const float (&b)[2], uint32_t out_a, int wq, int lane) {
#pragma unroll
  for (int jj = 0; jj < TILE_ROWS / 2; ++jj) {
    __nv_bfloat162 v[4];                                             // TL, TR, BL, BR
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int j = 2 * jj + r;
        v[2 * r + c] = __floats2bfloat162_rn(teco_act(acc[4 * j + c] + b[0], ACT), teco_act(acc[4 * j + 2 + c] + b[1], ACT));
      }
    const __nv_bfloat162 m = __hmax2(__hmax2(v[0], v[1]), __hmax2(v[2], v[3]));
    const int P = 4 * jj + (lane & 3);
    const uint32_t row = out_a + (uint32_t)(P * 128 + 2 * (lane >> 2));
    const uint32_t m32 = *reinterpret_cast<const uint32_t*>(&m);
    asm volatile("st.shared.b16 [%0], %1;" ::"r"(row + (uint32_t)(((2 * wq) ^ (P & 7)) << 4)), "h"((uint16_t)(m32 & 0xffffu))
                 : "memory");
    asm volatile("st.shared.b16 [%0], %1;" ::"r"(row + (uint32_t)(((2 * wq + 1) ^ (P & 7)) << 4)), "h"((uint16_t)(m32 >> 16))
                 : "memory");
  }
}

// The body of conv3x3_ws_kernel<MODE> (KL = 4, no pool) and of FNet's conv3x3_ws_live_kernel<KL, POOL> (MODE 0): KL
// K-steps per tap (mma_issue_tile), POOL the 2x2 max-pooled epilogue (ws_epilogue_pool).  Separate instances keep the
// generator's layers free of the variants' branches and registers.
template <int MODE, int KL, bool POOL>
__device__ __forceinline__ void ws_layer(const CUtensorMap& tmap, const CUtensorMap& ymap, const CUtensorMap& rmap,
                                         const TcParams& p) {
  static_assert(MODE == 0 || (KL == CB / 16 && !POOL), "conv3x3_ws_kernel<1> runs the full K without a pool");
  using Cfg = WsCfg<MODE>;
  constexpr int WS_STAGES = Cfg::STAGES, WS_OUT_BUFS = Cfg::OUT_BUFS, NACC = Cfg::NACC, S = Cfg::S;
  constexpr uint32_t WS_OUT_BYTES = Cfg::OUT_BYTES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                              // WS_STAGES halo stages
  uint8_t* w_s = ring + WS_STAGES * (size_t)HALO_STAGE;              // 9 taps x 64 x 64, resident
  uint8_t* outs = w_s + LAYER_W_BYTES;                               // [2][WS_OUT_BUFS] staging tiles
  uint64_t* full = reinterpret_cast<uint64_t*>(outs + 2 * WS_OUT_BUFS * (size_t)WS_OUT_BYTES);   // [WS_STAGES]
  uint64_t* empty = full + WS_STAGES;                                      // [WS_STAGES]
  uint64_t* w_full = empty + WS_STAGES;
  uint64_t* r_full = w_full + 1;                                           // [2][WS_OUT_BUFS] residual arrived
  float* s_bias = reinterpret_cast<float*>(r_full + 2 * WS_OUT_BUFS);      // [64]
  const bool has_res = MODE == 0 && p.res != nullptr;                      // the dispatch sends no mode-1 residual here

  const int tid = threadIdx.x, wg = tid >> 7;
  const int n0 = blockIdx.y * 64;
  const int G = gridDim.x;
  const int my_tiles = (int)blockIdx.x < p.num_tiles ? (p.num_tiles - (int)blockIdx.x + G - 1) / G : 0;

  for (int c = tid; c < 64; c += WS_THREADS) s_bias[c] = p.bias ? p.bias[n0 + c] : 0.f;
  if (tid == 0) {
    for (int s = 0; s < WS_STAGES; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), Cfg::WARPS_PER_STAGE);   // one arrival per consumer warp reading the stage
    }
    for (int i = 0; i < 1 + 2 * WS_OUT_BUFS; ++i) mbar_init(smem_u32(&w_full[i]), 1);   // w_full, r_full[]
    fence_mbar_init();
  }
  __syncthreads();
  if (my_tiles == 0) return;

  auto tile_coords = [&](int it, int& n, int& y0, int& x0) {
    int tile = (int)blockIdx.x + it * G;
    const int tx = tile % p.tiles_x;
    tile /= p.tiles_x;
    const int ty = tile % p.tiles_y;
    n = tile / p.tiles_y;
    x0 = tx * TILE_COLS;
    y0 = ty * TILE_ROWS;
  };

  if (wg == 2) {                              // producer warp: one lane issues every load of the ring
    if (tid == NUM_THREADS) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap) : "memory");
      mbar_expect_tx(smem_u32(w_full), LAYER_W_BYTES);
      for (int t = 0; t < 9; ++t)
        bulk_load_1d(smem_u32(w_s + t * 8192u), p.wpk + ((size_t)t * p.Cout + n0) * 128, 8192u, smem_u32(w_full));
      for (int k = 0; k < my_tiles; ++k) {
        const int st = k % WS_STAGES;
        if (k >= WS_STAGES) mbar_wait(smem_u32(&empty[st]), (uint32_t)((k / WS_STAGES - 1) & 1));
        int n, y0, x0;
        tile_coords(k, n, y0, x0);
        const uint32_t bar = smem_u32(&full[st]);
        mbar_expect_tx(bar, HALO_BYTES);
        tma_load_4d(smem_u32(ring + (size_t)st * HALO_STAGE), &tmap, bar, 0, x0 - 1, y0 - 1, n);
      }
    }
    return;
  }

  // consumer warpgroup wg.  MODE 0: tiles wg, wg + 2, ... of the walk, whole.  MODE 1: rows 8 wg .. 8 wg + 7 of every
  // tile.  The MMAs are issued in turns over both warpgroups: MODE 0 issues tile k in turn k, MODE 1 warpgroup g's part
  // of tile k in turn 2 k + g.
  const int wq = (tid >> 5) & 3, lane = tid & 31;
  const bool leader = (tid & 127) == 0;       // issues this warpgroup's residual loads and output stores
  const int my_turn = 1 + wg, other_turn = 2 - wg;   // named barrier 1 + g: warpgroup g may issue its MMAs
  const int k_first = MODE == 0 ? wg : 0, k_step = MODE == 0 ? 2 : 1, turns = MODE == 0 ? my_tiles : 2 * my_tiles;
  auto load_res = [&](int k, int b) {         // staging tile b of this warpgroup <- the residual box of tile k
    int n, y0, x0;
    tile_coords(k, n, y0, x0);
    const uint32_t bar = smem_u32(&r_full[WS_OUT_BUFS * wg + b]);
    mbar_expect_tx(bar, WS_OUT_BYTES);
    tma_load_4d(smem_u32(outs + (WS_OUT_BUFS * wg + b) * WS_OUT_BYTES), &rmap, bar, n0, x0, y0, n);
  };
  const float bias_r[2] = {s_bias[16 * wq + (lane >> 2)], s_bias[16 * wq + 8 + (lane >> 2)]};   // MODE 0's channels
  uint32_t r_phase = 0;                       // bit b: parity of r_full[WS_OUT_BUFS wg + b]
  if (has_res && leader && k_first < my_tiles) load_res(k_first, 0);
  mbar_wait(smem_u32(w_full), 0);
  float acc[NACC][Cfg::NR];
  for (int k = k_first, m = 0; k < my_tiles; k += k_step, ++m) {
    const int st = k % WS_STAGES, sb = m % WS_OUT_BUFS, sb_next = sb + 1 == WS_OUT_BUFS ? 0 : sb + 1;
    const int turn = MODE == 0 ? k : 2 * k + wg;
    int n, y0, x0;
    tile_coords(k, n, y0, x0);
    const int oy0 = MODE == 0 ? y0 : y0 + 8 * wg;   // first input row of this warpgroup's box
    uint8_t* out_s = outs + (WS_OUT_BUFS * wg + sb) * (size_t)WS_OUT_BYTES;
    mbar_wait(smem_u32(&full[st]), (uint32_t)((k / WS_STAGES) & 1));
    if (turn > 0) named_bar_sync(my_turn, 2 * 128);
    const uint32_t halo_a = smem_u32(ring + (size_t)st * HALO_STAGE);
    if constexpr (MODE == 0) mma_issue_tile<KL>(acc[0], halo_a, smem_u32(w_s));
    else mma_issue<MODE, 64, NACC, true>(acc, halo_a, smem_u32(w_s), wg);
    if (turn + 1 < turns) named_bar_arrive(other_turn, 2 * 128);
    if (has_res && leader && k + k_step < my_tiles) {
      // staging tile sb_next was last used by this warpgroup's tile m + 1 - WS_OUT_BUFS; all of its later stores may still
      // be reading their own
      bulk_wait_read<(WS_OUT_BUFS >= 2 ? WS_OUT_BUFS - 2 : 0)>();
      load_res(k + k_step, sb_next);
    }
    wgmma_wait_all_fence(acc);
    if (lane == 0) mbar_arrive(smem_u32(&empty[st]));
    if (MODE == 1 && oy0 >= p.H) continue;    // MODE 1: this warpgroup's rows are all below the image

    if (has_res) {
      mbar_wait(smem_u32(&r_full[WS_OUT_BUFS * wg + sb]), (r_phase >> sb) & 1u);
      r_phase ^= 1u << sb;
    } else {
      if (leader) bulk_wait_read<WS_OUT_BUFS - 1>();   // the store that last used staging tile sb has read it
      named_bar_sync(3 + wg, 128);
    }
    const uint32_t out_a = smem_u32(out_s);
    if constexpr (POOL) {                     // the dispatch sends no residual with it
      switch (p.act) {
        case TECO_ACT_RELU: ws_epilogue_pool<TECO_ACT_RELU>(acc[0], bias_r, out_a, wq, lane); break;
        case TECO_ACT_LRELU02: ws_epilogue_pool<TECO_ACT_LRELU02>(acc[0], bias_r, out_a, wq, lane); break;
        case TECO_ACT_TANH24: ws_epilogue_pool<TECO_ACT_TANH24>(acc[0], bias_r, out_a, wq, lane); break;
        case TECO_ACT_SIGMOID: ws_epilogue_pool<TECO_ACT_SIGMOID>(acc[0], bias_r, out_a, wq, lane); break;
        default: ws_epilogue_pool<TECO_ACT_NONE>(acc[0], bias_r, out_a, wq, lane); break;
      }
    } else {
      switch (p.act) {                        // once per tile: the element loop is compiled per activation
        case TECO_ACT_RELU: ws_epilogue<TECO_ACT_RELU, MODE>(acc, s_bias, bias_r, out_a, has_res, wq, lane); break;
        case TECO_ACT_LRELU02: ws_epilogue<TECO_ACT_LRELU02, MODE>(acc, s_bias, bias_r, out_a, has_res, wq, lane); break;
        case TECO_ACT_TANH24: ws_epilogue<TECO_ACT_TANH24, MODE>(acc, s_bias, bias_r, out_a, has_res, wq, lane); break;
        case TECO_ACT_SIGMOID: ws_epilogue<TECO_ACT_SIGMOID, MODE>(acc, s_bias, bias_r, out_a, has_res, wq, lane); break;
        default: ws_epilogue<TECO_ACT_NONE, MODE>(acc, s_bias, bias_r, out_a, has_res, wq, lane); break;
      }
    }
    fence_async_smem();                       // the staging writes -> visible to the TMA store
    named_bar_sync(3 + wg, 128);
    if (leader) {
      // pooled: the 8 x 4 box at half the tile's coordinates on the [N, H / 2, W / 2] output (even x0, y0), clipped
      // where the odd last row or column of the input pools to nothing
      if constexpr (POOL) tma_store_4d(&ymap, out_a, n0, x0 / 2, y0 / 2, n);
      else tma_store_4d(&ymap, out_a, n0, S * x0, S * oy0, n);
      bulk_commit();
    }
  }
  if (leader) bulk_wait_all();
}

template <int MODE>
__global__ void __launch_bounds__(WS_THREADS, 1)
conv3x3_ws_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap ymap,
                  const __grid_constant__ CUtensorMap rmap, const TcParams p) {
  ws_layer<MODE, CB / 16, false>(tmap, ymap, rmap, p);
}

template <int KL, bool POOL>
__global__ void __launch_bounds__(WS_THREADS, 1)
conv3x3_ws_live_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap ymap,
                       const __grid_constant__ CUtensorMap rmap, const TcParams p) {
  ws_layer<0, KL, POOL>(tmap, ymap, rmap, p);
}

// ------------------------------------------------------------------ im2col-tiled layer (images smaller than a tile)
// Mode 0, 64-channel bf16 output slices, no residual, any Cin: FNet's 8 x 8 and 4 x 4 levels, where a 16 x 8 tile of one
// image would be one half or one eighth full.  The tile is IC_PIX = 128 output pixels in flat N*H*W order and spans as
// many images as it needs.
//   - Per (64-channel K block b, tap t) one im2col-mode TMA box brings the tile's 128 input pixels at the tap's offset,
//     64 channels each, as 128-byte SWIZZLE_128B rows: the map's bounding box (corners -1, -1) walks the output pixels in
//     flat order and each pixel is read at (x - 1 + kx, y - 1 + ky); the zero fill outside every image is the 'SAME'
//     padding, and past the last image it feeds pixels whose outputs are not stored.  Pixel row p of the box is row p of
//     the K-major B operand (8-row groups 1024 B apart).
//   - MMAs as conv3x3_ws_kernel<0>: M = the CTA's 64 output channels (blockIdx.y), A = the packed weight tap, N = the
//     tile's 128 pixels; taps in (K block, tap, K-step) order, scale-d = 0 first.  Per output element that is the order
//     of conv3x3_wgmma_kernel (nblk > 1) and of conv3x3_ws_kernel<0> (nblk = 1), so the results are bit-identical to the
//     layer's teco_conv3x3_tc launch.
//   - Cin up to 512 is 9 x 8 weight taps of 8 KB per Cout slice, too many to keep resident: one producer warp streams
//     (pixel box, weight tap) pairs through an IC_STAGES-deep ring; a stage is released once the MMAs that read it have
//     completed (one arrival per consumer warp, after wgmma.wait_group of the next step).
//   - Persistent CTAs; the two consumer warpgroups take alternate tiles of the CTA's walk and take turns to issue their
//     tiles' MMAs (named barriers 1 and 2, as in conv3x3_ws_kernel), so one warpgroup's epilogue overlaps the other's
//     MMAs.
//   - Epilogue: ws_epilogue<ACT, 0> (bias -> activation -> bf16, stmatrix) into the warpgroup's staging tile, whose pixel
//     p is row p as in the ws kernel; one TMA store of the [128 pixels, 64 channels] box on the flat [N*H*W, Cout] view,
//     clipped after the last pixel.
constexpr int IC_PIX = 128;                                  // output pixels per tile
constexpr uint32_t IC_BOX = IC_PIX * 128u;                   // one pixel box or staging tile: 16384
constexpr uint32_t IC_TAP = 64u * 128u;                      // one packed weight tap of a 64-channel Cout slice
constexpr uint32_t IC_STAGE = IC_BOX + IC_TAP;               // 24576: stages stay 1024-byte aligned
constexpr int IC_STAGES = 8;
constexpr size_t IC_SMEM = 1024 + IC_STAGES * (size_t)IC_STAGE + 2 * (size_t)IC_BOX + 2 * IC_STAGES * sizeof(uint64_t) +
                           64 * sizeof(float);
static_assert(IC_SMEM <= SMEM_MAX, "conv3x3_im2col_kernel: shared memory budget");

struct IcParams {
  int H, W, Cout, nblk, act, num_tiles;
  const uint8_t* wpk;
  const float* bias;
};

__global__ void __launch_bounds__(WS_THREADS, 1)
conv3x3_im2col_kernel(const __grid_constant__ CUtensorMap xmap, const __grid_constant__ CUtensorMap ymap, const IcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                                  // IC_STAGES x [pixel box | weight tap]
  uint8_t* outs = ring + IC_STAGES * (size_t)IC_STAGE;                   // [2] staging tiles
  uint64_t* full = reinterpret_cast<uint64_t*>(outs + 2 * (size_t)IC_BOX);   // [IC_STAGES]
  uint64_t* empty = full + IC_STAGES;                                    // [IC_STAGES]
  float* s_bias = reinterpret_cast<float*>(empty + IC_STAGES);           // [64]

  const int tid = threadIdx.x, wg = tid >> 7;
  const int n0 = blockIdx.y * 64;
  const int G = gridDim.x;
  const int my_tiles = (int)blockIdx.x < p.num_tiles ? (p.num_tiles - (int)blockIdx.x + G - 1) / G : 0;

  for (int c = tid; c < 64; c += WS_THREADS) s_bias[c] = p.bias ? p.bias[n0 + c] : 0.f;
  if (tid == 0) {
    for (int s = 0; s < IC_STAGES; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), 4);      // one arrival per warp of the consumer warpgroup reading the stage
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (my_tiles == 0) return;

  if (wg == 2) {                              // producer warp: one lane issues every load of the ring
    if (tid == NUM_THREADS) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
      const int HW = p.H * p.W;
      for (int k = 0, q = 0; k < my_tiles; ++k) {
        const int p0 = ((int)blockIdx.x + k * G) * IC_PIX;
        const int n = p0 / HW, r = p0 - n * HW, oy = r / p.W, ox = r - oy * p.W;
        for (int b = 0; b < p.nblk; ++b)
          for (int t = 0; t < 9; ++t, ++q) {
            const int st = q % IC_STAGES;
            if (q >= IC_STAGES) mbar_wait(smem_u32(&empty[st]), (uint32_t)((q / IC_STAGES - 1) & 1));
            const uint32_t base = smem_u32(ring + (size_t)st * IC_STAGE), bar = smem_u32(&full[st]);
            mbar_expect_tx(bar, IC_STAGE);
            tma_load_im2col_4d(base, &xmap, bar, b * CB, ox - 1, oy - 1, n, (uint16_t)(t % 3), (uint16_t)(t / 3));
            bulk_load_1d(base + IC_BOX, p.wpk + ((size_t)(b * 9 + t) * p.Cout + n0) * 128, IC_TAP, bar);
          }
      }
    }
    return;
  }

  // consumer warpgroup wg: tiles wg, wg + 2, ... of the walk; tile k issues its MMAs in turn k
  const int wq = (tid >> 5) & 3, lane = tid & 31;
  const bool leader = (tid & 127) == 0;       // issues this warpgroup's output stores
  const int my_turn = 1 + wg, other_turn = 2 - wg;
  const float bias_r[2] = {s_bias[16 * wq + (lane >> 2)], s_bias[16 * wq + 8 + (lane >> 2)]};
  const uint32_t ring_a = smem_u32(ring), out_a = smem_u32(outs + (size_t)wg * IC_BOX);
  const int steps = 9 * p.nblk;
  float acc[1][64];
  for (int k = wg; k < my_tiles; k += 2) {
    int q = k * steps;                        // ring steps of the tiles before this one
    if (k > 0) named_bar_sync(my_turn, 2 * 128);
    for (int b = 0; b < p.nblk; ++b) {
#pragma unroll
      for (int t = 0; t < 9; ++t, ++q) {
        const int st = q % IC_STAGES;
        mbar_wait(smem_u32(&full[st]), (uint32_t)((q / IC_STAGES) & 1));
        const uint32_t box_a = ring_a + (uint32_t)st * IC_STAGE, w_a = box_a + IC_BOX;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < CB / 16; ++kk)
          Wgmma<128, 0, 0>::run(acc[0], gmma_desc_sw128(w_a + 32u * kk, 16u, 1024u), gmma_desc_sw128(box_a + 32u * kk, 16u, 1024u),
                                b == 0 && t == 0 && kk == 0 ? 0u : 1u);
        wgmma_commit();
        if (b > 0 || t > 0) {
          wgmma_wait<1>();                    // the previous step's MMAs have completed: release its stage
          mbar_arrive_if(smem_u32(&empty[(q - 1) % IC_STAGES]), lane == 0);
        }
      }
    }
    if (k + 1 < my_tiles) named_bar_arrive(other_turn, 2 * 128);
    wgmma_wait_all_fence(acc);
    if (lane == 0) mbar_arrive(smem_u32(&empty[(q - 1) % IC_STAGES]));

    if (leader) bulk_wait_read<0>();          // this warpgroup's previous store has read the staging tile
    named_bar_sync(3 + wg, 128);
    switch (p.act) {                          // once per tile: the element loop is compiled per activation
      case TECO_ACT_RELU: ws_epilogue<TECO_ACT_RELU, 0>(acc, s_bias, bias_r, out_a, false, wq, lane); break;
      case TECO_ACT_LRELU02: ws_epilogue<TECO_ACT_LRELU02, 0>(acc, s_bias, bias_r, out_a, false, wq, lane); break;
      case TECO_ACT_TANH24: ws_epilogue<TECO_ACT_TANH24, 0>(acc, s_bias, bias_r, out_a, false, wq, lane); break;
      case TECO_ACT_SIGMOID: ws_epilogue<TECO_ACT_SIGMOID, 0>(acc, s_bias, bias_r, out_a, false, wq, lane); break;
      default: ws_epilogue<TECO_ACT_NONE, 0>(acc, s_bias, bias_r, out_a, false, wq, lane); break;
    }
    fence_async_smem();                       // the staging writes -> visible to the TMA store
    named_bar_sync(3 + wg, 128);
    if (leader) {
      tma_store_2d(&ymap, out_a, n0, ((int)blockIdx.x + k * G) * IC_PIX);
      bulk_commit();
    }
  }
  if (leader) bulk_wait_all();
}

// ------------------------------------------------------------------ fp32 output stage (64 -> 2 or 3 channels)
// Mode 0, Cin = 64, the 16-channel packed Cout slice, an fp32 output of C = 2 or 3 channels with an optional fp32
// residual and post scale / shift: the generator's output stage (64 -> 3, + bicubic, * 2 - 1) and FNet's flow head
// (64 -> 2, tanh * 24).  The products are those of conv3x3_wgmma_kernel<16>: per 64-pixel half of the 16 x 8 tile the
// unswapped m64n16k16 of mma_issue, the halo as A and the packed weights as B, taps 0..8 x K-steps 0..3 (scale-d = 0
// first); the epilogue runs epilogue()'s fp32 operations in its order, so the outputs are bit-identical to
// teco_conv3x3_tc's.  What differs is the pipeline, after conv3x3_ws_kernel<0>:
//   - one producer warp bulk-copies the 18 KB of weights once and TMA-loads the halo of each tile into an F32_STAGES-deep
//     ring;
//   - one consumer warpgroup owns a whole tile (both halves, 2 x 8 accumulator registers per thread); the two take
//     alternate tiles of the CTA's walk and take turns to issue their MMAs (named barriers 1 and 2), so one warpgroup's
//     epilogue overlaps the other's MMAs;
//   - two CTAs per SM, three halo stages each: four issuing warpgroups keep the tensor pipe fed better than one CTA with
//     an eight-stage ring (at 264 clips x 128 x 128 on an H100 at 700 W: 292 us against 350 us; three CTAs of two stages:
//     305 us);
//   - the residual and the output are boxes of 16 rows x 8 C floats on the [N, H, W C] fp32 view.  The residual box of
//     the warpgroup's next tile is TMA-loaded into its other staging box while this tile's MMAs run; the epilogue
//     overwrites the residual with the result and one TMA store writes the box out, clipped at the image edges.
constexpr int F32_STAGES = 3;
constexpr int F32_CTAS_PER_SM = 2;
constexpr int F32_BUFS = 2;                                                       // staging boxes per warpgroup
constexpr uint32_t F32_W_BYTES = 9u * 16u * 128u;                                 // 18432: 9 taps x 16 cout x 64 cin
constexpr uint32_t F32_BOX_BYTES = TILE_ROWS * TILE_COLS * 3 * sizeof(float);     // one box at C = 3: 1536
constexpr size_t F32_SMEM = 1024 + F32_STAGES * (size_t)HALO_STAGE + F32_W_BYTES + 2 * F32_BUFS * (size_t)F32_BOX_BYTES +
                            (2 * F32_STAGES + 1 + 2 * F32_BUFS) * sizeof(uint64_t) + 16 * sizeof(float);
static_assert(F32_CTAS_PER_SM * (F32_SMEM + 1024) <= 233472, "conv3x3_f32out_kernel: two CTAs per SM (228 KB, 1 KB reserved each)");

struct F32Params {
  int C, act, has_res, tiles_x, tiles_y, num_tiles;
  float post_scale, post_shift;
  const uint8_t* wpk;
  const float* bias;
};

// Epilogue of one tile into its staging box (pixel (row r, column x) at floats (8 r + x) C ..): this thread holds, per
// half h, pixels (row 8 h + 2 wq + i, column lane / 4) at channels 2 (lane % 4) + {0, 1} of the accumulator's first
// eight (C <= 3: only lanes with lane % 4 < 2 hold a stored channel).  bias -> activation -> (+ residual) -> * scale +
// shift, as epilogue() computes it.
template <int ACT>
__device__ __forceinline__ void f32_epilogue(const float (&acc)[2][1][8], const float* s_bias, float* box, const F32Params& p,
                                             int wq, int lane) {
  const int C = p.C, c = 2 * (lane & 3);
  if (c >= C) return;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* px = box + ((8 * h + 2 * wq + i) * TILE_COLS + (lane >> 2)) * C + c;
      const float v0 = teco_act(acc[h][0][2 * i] + s_bias[c], ACT);
      px[0] = (v0 + (p.has_res ? px[0] : 0.f)) * p.post_scale + p.post_shift;
      if (c + 1 < C) {
        const float v1 = teco_act(acc[h][0][2 * i + 1] + s_bias[c + 1], ACT);
        px[1] = (v1 + (p.has_res ? px[1] : 0.f)) * p.post_scale + p.post_shift;
      }
    }
}

// KL: K-steps per tap (mma_issue); 4 for the generator's output stage, 2 for FNet's flow head (32 live channels)
template <int KL>
__global__ void __launch_bounds__(WS_THREADS, F32_CTAS_PER_SM)
conv3x3_f32out_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap omap,
                      const __grid_constant__ CUtensorMap rmap, const F32Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* ring = smem;                                                     // F32_STAGES halo stages
  uint8_t* w_s = ring + F32_STAGES * (size_t)HALO_STAGE;                    // 9 taps x 16 x 64, resident
  uint8_t* boxes = w_s + F32_W_BYTES;                                       // [2][F32_BUFS] staging boxes
  uint64_t* full = reinterpret_cast<uint64_t*>(boxes + 2 * F32_BUFS * (size_t)F32_BOX_BYTES);   // [F32_STAGES]
  uint64_t* empty = full + F32_STAGES;                                      // [F32_STAGES]
  uint64_t* w_full = empty + F32_STAGES;
  uint64_t* r_full = w_full + 1;                                            // [2][F32_BUFS] residual arrived
  float* s_bias = reinterpret_cast<float*>(r_full + 2 * F32_BUFS);          // [16]

  const int tid = threadIdx.x, wg = tid >> 7;
  const int G = gridDim.x;
  const int my_tiles = (int)blockIdx.x < p.num_tiles ? (p.num_tiles - (int)blockIdx.x + G - 1) / G : 0;

  for (int c = tid; c < 16; c += WS_THREADS) s_bias[c] = p.bias ? p.bias[c] : 0.f;
  if (tid == 0) {
    for (int s = 0; s < F32_STAGES; ++s) {
      mbar_init(smem_u32(&full[s]), 1);
      mbar_init(smem_u32(&empty[s]), 4);      // one arrival per warp of the consumer warpgroup reading the stage
    }
    for (int i = 0; i < 1 + 2 * F32_BUFS; ++i) mbar_init(smem_u32(&w_full[i]), 1);   // w_full, r_full[]
    fence_mbar_init();
  }
  __syncthreads();
  if (my_tiles == 0) return;

  auto tile_coords = [&](int it, int& n, int& y0, int& x0) {
    int tile = (int)blockIdx.x + it * G;
    const int tx = tile % p.tiles_x;
    tile /= p.tiles_x;
    const int ty = tile % p.tiles_y;
    n = tile / p.tiles_y;
    x0 = tx * TILE_COLS;
    y0 = ty * TILE_ROWS;
  };

  if (wg == 2) {                              // producer warp: one lane issues every load of the ring
    if (tid == NUM_THREADS) {
      asm volatile("prefetch.tensormap [%0];" ::"l"(&tmap) : "memory");
      mbar_expect_tx(smem_u32(w_full), F32_W_BYTES);
      bulk_load_1d(smem_u32(w_s), p.wpk, F32_W_BYTES, smem_u32(w_full));
      for (int k = 0; k < my_tiles; ++k) {
        const int st = k % F32_STAGES;
        if (k >= F32_STAGES) mbar_wait(smem_u32(&empty[st]), (uint32_t)((k / F32_STAGES - 1) & 1));
        int n, y0, x0;
        tile_coords(k, n, y0, x0);
        const uint32_t bar = smem_u32(&full[st]);
        mbar_expect_tx(bar, HALO_BYTES);
        tma_load_4d(smem_u32(ring + (size_t)st * HALO_STAGE), &tmap, bar, 0, x0 - 1, y0 - 1, n);
      }
    }
    return;
  }

  // consumer warpgroup wg: tiles wg, wg + 2, ... of the walk; tile k issues its MMAs in turn k
  const int wq = (tid >> 5) & 3, lane = tid & 31;
  const bool leader = (tid & 127) == 0;       // issues this warpgroup's residual loads and output stores
  const int my_turn = 1 + wg, other_turn = 2 - wg;
  const uint32_t box_bytes = (uint32_t)(TILE_ROWS * TILE_COLS * p.C) * (uint32_t)sizeof(float);
  auto box_at = [&](int b) { return reinterpret_cast<float*>(boxes + (F32_BUFS * wg + b) * (size_t)F32_BOX_BYTES); };
  auto load_res = [&](int k, int b) {         // staging box b of this warpgroup <- the residual box of tile k
    int n, y0, x0;
    tile_coords(k, n, y0, x0);
    const uint32_t bar = smem_u32(&r_full[F32_BUFS * wg + b]);
    mbar_expect_tx(bar, box_bytes);
    tma_load_3d(smem_u32(box_at(b)), &rmap, bar, x0 * p.C, y0, n);
  };
  uint32_t r_phase = 0;                       // bit b: parity of r_full[F32_BUFS wg + b]
  if (p.has_res && leader && wg < my_tiles) load_res(wg, 0);
  mbar_wait(smem_u32(w_full), 0);
  const uint32_t w_a = smem_u32(w_s);
  float acc[2][1][8];
  for (int k = wg, m = 0; k < my_tiles; k += 2, ++m) {
    const int st = k % F32_STAGES, sb = m % F32_BUFS, sb_next = (m + 1) % F32_BUFS;
    int n, y0, x0;
    tile_coords(k, n, y0, x0);
    float* box = box_at(sb);
    mbar_wait(smem_u32(&full[st]), (uint32_t)((k / F32_STAGES) & 1));
    if (k > 0) named_bar_sync(my_turn, 2 * 128);
    const uint32_t halo_a = smem_u32(ring + (size_t)st * HALO_STAGE);
    mma_issue<0, 16, 1, true, KL>(acc[0], halo_a, w_a, 0);
    mma_issue<0, 16, 1, true, KL>(acc[1], halo_a, w_a, 1);
    if (k + 1 < my_tiles) named_bar_arrive(other_turn, 2 * 128);
    if (p.has_res && leader && k + 2 < my_tiles) {
      bulk_wait_read<F32_BUFS - 2>();         // the store of this warpgroup's previous tile has read box sb_next
      load_res(k + 2, sb_next);
    }
    wgmma_wait_all_fence(acc[0]);
    wgmma_wait_all_fence(acc[1]);
    if (lane == 0) mbar_arrive(smem_u32(&empty[st]));

    if (p.has_res) {
      mbar_wait(smem_u32(&r_full[F32_BUFS * wg + sb]), (r_phase >> sb) & 1u);
      r_phase ^= 1u << sb;
    } else {
      if (leader) bulk_wait_read<F32_BUFS - 1>();   // the store that last used box sb has read it
      named_bar_sync(3 + wg, 128);
    }
    switch (p.act) {                          // once per tile: the element loop is compiled per activation
      case TECO_ACT_RELU: f32_epilogue<TECO_ACT_RELU>(acc, s_bias, box, p, wq, lane); break;
      case TECO_ACT_LRELU02: f32_epilogue<TECO_ACT_LRELU02>(acc, s_bias, box, p, wq, lane); break;
      case TECO_ACT_TANH24: f32_epilogue<TECO_ACT_TANH24>(acc, s_bias, box, p, wq, lane); break;
      case TECO_ACT_SIGMOID: f32_epilogue<TECO_ACT_SIGMOID>(acc, s_bias, box, p, wq, lane); break;
      default: f32_epilogue<TECO_ACT_NONE>(acc, s_bias, box, p, wq, lane); break;
    }
    fence_async_smem();                       // the staging writes -> visible to the TMA store
    named_bar_sync(3 + wg, 128);
    if (leader) {
      tma_store_3d(&omap, smem_u32(box), x0 * p.C, y0, n);
      bulk_commit();
    }
  }
  if (leader) bulk_wait_all();
}

// ------------------------------------------------------------------ generator trunk in shared memory (32 x 32 images)
// A chain of 3x3 64 -> 64 layers on 32 x 32 images in one launch, the activations never leaving shared memory.  A cluster
// of two CTAs (one per SM, persistent) owns clips c, c + G, ... (G clusters); CTA r of the cluster owns image rows
// 16 r .. 16 r + 15 for every layer.
//   - Shared memory: the weight ring (9 taps x 8 KB, one whole layer), two activation slots and the mbarriers.  Each slot
//     is [18 rows][34 px][64 ch] bf16 in the SW128 image: the own rows, one halo row above and below, a zero column
//     either side.  Slot 0 holds the plan's buffer 0 (x_in, read by layer 0 only) and then buffer 2; slot 1 holds buffer
//     1.  Layer l reads slot l & 1 and writes the other.  x_in arrives as one 4-D TMA box {64, 34, 18} at
//     (0, -1, 16 r - 1, n), whose out-of-bounds zero fill is the padding; slot 1 is zeroed once, and rows and columns no
//     layer writes stay zero.
//   - The MMAs and the epilogue arithmetic are those of conv3x3_ws_kernel<0>, so the results are bit-identical to it: per
//     16 x 8 tile one m64n128k16 accumulator, the weight tap as A and the slot at the tap's offset as B (8-pixel groups one
//     34-pixel row apart), taps 0..8 x K-steps 0..3, scale-d = 0 first, one commit group per tap; bias -> activation ->
//     (+ bf16 residual) -> bf16.
//   - Strip s (0..3) is the 16 x 8 tile at columns 8 s .. 8 s + 7.  Consumer warpgroup 0 owns strips 0 and 1 and works on
//     them in that order, warpgroup 1 strips 3 and 2; write M(l, s) for the MMAs of strip s at layer l and E(l, s) for
//     its epilogue.  The warpgroups take turns to issue a whole strip (named barriers 1 and 2, as in conv3x3_ws_kernel):
//     W0 M(l, 0), W1 M(l, 3), W0 M(l, 1), W1 M(l, 2), W0 M(l + 1, 0), ...  A warpgroup waits for its first strip and
//     runs its epilogue under the other warpgroup's strip before it issues its second, and runs the epilogue of its
//     second strip under the other warpgroup's second one, so the tensor pipe has a strip queued across the layer
//     boundary as long as an epilogue takes less than a strip's 36 MMAs.
//   - Weights: one producer warp loads tap t of every layer into ring slot t.  A slot is released (8 arrivals, one per
//     consumer warp) once the warp has seen the tap complete in both of its warpgroup's strips: by wgmma.wait_group per
//     tap of its second strip, with no epilogue in between, so layer l + 1's tap t reloads while layer l's later taps
//     still run.
//   - The epilogue stmatrix-es the bf16 outputs straight into the other slot (an in-place residual is ldmatrix-ed from the
//     same place first); the 128-byte swizzle chunk is taken from the address, as the TMA and the MMAs apply it.  After a
//     generic -> async proxy fence and a barrier over the warpgroup, one of its threads bulk-copies the strip's 1 KB of
//     the CTA's boundary row into the partner's halo row of the same slot (16 x 4352 B and 1024 s are multiples of
//     1024: the swizzled bytes copy unchanged), completing on the partner's row_full[slot][s].
//   - After a clip's last layer the consumers copy the CTA's own 16 rows of each slot the plan wrote to global memory with
//     16-byte stores (un-swizzling the address); after a barrier one thread loads the next clip's x_in into slot 0.
// Dependencies (si = l & 1 is layer l's input slot, so = si ^ 1 its output slot).  M(l + 1, s) reads the columns of
// strips s - 1 .. s + 1 of slot so, in the own rows and in the partner's halo row.
//   - RAW, own rows: M(l + 1, s) follows E(l, s - 1 .. s + 1).  Within a warpgroup by program order; across the strip 1 |
//     strip 2 boundary through mid[g][so], on which every thread of warpgroup g arrives after E(l, 1 + g) and its
//     fence.proxy.async.  Each warpgroup runs its boundary epilogue before it next waits for the other one.
//   - RAW, partner rows: M(l + 1, s) waits on row_full[so][s - 1 .. s + 1].
//   - WAR, own rows: E(l + 1, s) overwrites in slot si what M(l, s - 1 .. s + 1) read.  The warpgroup waited for its own
//     M(l, .) before its epilogues, and the other warpgroup's boundary strip M(l, .) completed before that warpgroup's
//     E(l, .) arrived on mid[.][so], which M(l + 1, s) -- before E(l + 1, s) in program order -- waited for.
//   - WAR, the partner's halo row: this CTA sends row (l, s) after its M(l, s), which needed the partner's rows
//     (l - 1, s - 1 .. s + 1); the partner sent each after its E(l - 1, .), i.e. after its M(l - 1, .) that read the
//     halo columns of strip s in slot so had completed.  So the copy lands in columns the partner has finished reading.
//   - WAR, the source row: this CTA's row (l, s) in slot so is next rewritten by E(l + 2, s), after M(l + 2, s), which
//     needed the partner's row (l + 1, s), sent after the partner's M(l + 1, s), which waited for row (l, s) to land:
//     the copy has read its source.
//   - row_full[i][s] and mid[g][i] complete one phase per layer that writes slot i.  The next phase's bytes or arrivals
//     come from a layer two later, which needs the current phase's waiters to have moved on (the same chains as above),
//     and this CTA's expect_tx for a phase follows its wait for the previous one in program order.
//   - Clips: the first wait of a clip is on x_in in slot 0.  Before loading it, thread 0 has waited (a) for the
//     partner's last-layer rows (every consumer did) and (b) on peer_free, on which the partner arrives remotely once
//     it has waited for this CTA's last-layer rows.  So the next clip's TMA, epilogues and copies find every copy of the
//     previous clip landed and every source read.
constexpr int TR_COLS = LIN_W + 2;                                        // 34: a zero column either side
constexpr int TR_ROWS = 16 + 2;                                           // own rows + a halo row above and below
constexpr uint32_t TR_ROW_BYTES = TR_COLS * 128u;                         // 4352: wgmma SBO between tile rows
constexpr uint32_t TR_SLOT_BYTES = TR_ROWS * TR_ROW_BYTES;                // 78336
constexpr uint32_t TR_TAP = 64u * 128u;                                   // one packed tap [64 cout][64 cin]
constexpr uint32_t TR_SLOT0 = LAYER_W_BYTES;                              // 73728: after the nine-tap weight ring
constexpr uint32_t TR_SLOT1 = (TR_SLOT0 + TR_SLOT_BYTES + 1023u) & ~1023u;   // 152576: slots start on the swizzle period
constexpr uint32_t TR_BAR_OFF = TR_SLOT1 + TR_SLOT_BYTES;                 // 230912
constexpr uint32_t TR_STRIP_EDGE = TILE_COLS * 128u;                      // one strip's part of a boundary row: 1024
constexpr int TR_BARS = 9 + 9 + 2 * 4 + 2 * 2 + 2;                        // full, empty, row_full, mid, x_full, peer_free
constexpr size_t TR_SMEM = 1024 + TR_BAR_OFF + TR_BARS * sizeof(uint64_t);
static_assert(TR_SMEM <= SMEM_MAX, "conv3x3_trunk_cluster_kernel: shared memory budget");
static_assert(TR_SLOT0 % 1024 == 0 && TR_SLOT1 % 1024 == 0, "slots start on the swizzle period");
static_assert((16 * TR_ROW_BYTES) % 1024 == 0, "a boundary row and the partner's halo row share their swizzle phase");

struct TrunkParams {
  int N, L;
  uint64_t res_mask;                 // bit l: layer l adds its output buffer's previous value (in place)
  uint64_t relu_mask, lrelu_mask;    // bit l: layer l's activation (neither: none)
  const uint8_t* wpk;                // L packed layers back to back
  const float* bias;                 // [L][64]
  __nv_bfloat16* a;                  // buffer 1 (slot 1)
  __nv_bfloat16* b;                  // buffer 2 (slot 0 after layer 0)
};

// The CTA's own rows y0 .. y0 + 15 of image n in the slot at `slot` -> dst [N,32,32,64]: consecutive threads store
// consecutive 16-byte chunks of global memory, chunk q of slot pixel P read from chunk q ^ (P & 7).
__device__ __forceinline__ void trunk_store_rows(uint32_t slot, __nv_bfloat16* dst, int n, int y0, int tid) {
  uint4* out = reinterpret_cast<uint4*>(dst + ((size_t)n * LIN_W + y0) * LIN_W * 64);
#pragma unroll 4
  for (int c = tid; c < 16 * LIN_W * 8; c += NUM_THREADS) {
    const int px = c >> 3, q = c & 7;
    const int P = (1 + px / LIN_W) * TR_COLS + 1 + px % LIN_W;
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "r"(slot + (uint32_t)(P * 128 + ((q ^ (P & 7)) << 4))));
    out[c] = v;
  }
}

// Epilogue of one 16 x 8 tile at column x0 of the CTA's rows, into the slot at `slot`: ws_epilogue<ACT, 0> with the tile's
// pixel (row R, column C) at slot pixel P = (1 + R) * 34 + 1 + x0 + C, chunk q at q ^ (P & 7).
template <int ACT>
__device__ __forceinline__ void trunk_epilogue(const float (&acc)[64], const float (&b)[2], uint32_t slot, int x0, bool res,
                                               int wq, int lane) {
  const int q = 2 * wq + ((lane >> 3) & 1);
  const int p0 = (1 + (lane >> 4)) * TR_COLS + 1 + x0 + (lane & 7);
#pragma unroll
  for (int jj = 0; jj < TILE_ROWS / 2; ++jj) {
    const int px = p0 + 2 * jj * TR_COLS;
    const uint32_t a = slot + (uint32_t)(px * 128 + ((q ^ (px & 7)) << 4));
    uint32_t r[4];
    if (res) ldmatrix_x4_trans(r, a);
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int j = 2 * jj + (m >> 1), i = m & 1;
      float v0 = teco_act(acc[4 * j + 2 * i] + b[i], ACT);
      float v1 = teco_act(acc[4 * j + 2 * i + 1] + b[i], ACT);
      if (res) {
        const float2 rf = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&r[m]));
        v0 += rf.x;
        v1 += rf.y;
      }
      const __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
      r[m] = *reinterpret_cast<const uint32_t*>(&o);
    }
    stmatrix_x4_trans(a, r);
  }
}

// M(l, s): the 9 taps x 4 K-steps of one strip into acc, B from the input slot at the strip's column (b_a), tap t from
// ring slot t once full[t] shows it loaded (parity wpar); one commit group per tap.
__device__ __forceinline__ void trunk_issue_strip(float (&acc)[64], uint32_t wring_a, const uint64_t* full, uint32_t wpar,
                                                  uint32_t b_a) {
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    mbar_wait(smem_u32(&full[t]), wpar);
    wgmma_fence();
    const uint32_t a0 = wring_a + (uint32_t)t * TR_TAP;
    const uint32_t b0 = b_a + (uint32_t)(((t / 3) * TR_COLS + t % 3) * 128);
#pragma unroll
    for (int kk = 0; kk < CB / 16; ++kk)
      Wgmma<128, 0, 0>::run(acc, gmma_desc_sw128(a0 + 32u * kk, 16u, 1024u), gmma_desc_sw128(b0 + 32u * kk, 16u, TR_ROW_BYTES),
                            t == 0 && kk == 0 ? 0u : 1u);
    wgmma_commit();
  }
}

// With the second strip's 9 commit groups issued and the first strip's complete: release ring slot T, T + 1, .. 8 as the
// second strip's tap completes.  ptxas encodes a wait for at most 8 pending groups as one for at most 7, so slot 0 goes
// with slot 1.
template <int T>
__device__ __forceinline__ void trunk_release_taps(const uint64_t* empty, bool lane0) {
  wgmma_wait<8 - T>();
  mbar_arrive_if(smem_u32(&empty[T]), lane0);
  if constexpr (T < 8) trunk_release_taps<T + 1>(empty, lane0);
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(WS_THREADS, 1)
conv3x3_trunk_cluster_kernel(const __grid_constant__ CUtensorMap xmap, const TrunkParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + TR_BAR_OFF);   // [9]: tap t of the current layer is in ring slot t
  uint64_t* empty = full + 9;                    // [9]: every consumer warp is done with ring slot t
  uint64_t* row_full = empty + 9;                // [2][4]: strip s of the partner's boundary row has landed in slot i
  uint64_t* mid = row_full + 8;                  // [2][2]: warpgroup g's strip 1 + g is in slot i
  uint64_t* x_full = mid + 4;                    // x_in of the clip has landed in slot 0
  uint64_t* peer_free = x_full + 1;              // the partner has taken this CTA's last rows of the previous clip

  const int tid = threadIdx.x, wg = tid >> 7;
  const uint32_t rank = cluster_ctarank(), peer = rank ^ 1u;
  const int cl = (int)blockIdx.x >> 1, G = (int)gridDim.x >> 1;
  const int my_clips = cl < p.N ? (p.N - cl + G - 1) / G : 0;

  if (tid == 0) {
    for (int t = 0; t < 9; ++t) {
      mbar_init(smem_u32(&full[t]), 1);
      mbar_init(smem_u32(&empty[t]), 8);         // one arrival per consumer warp
    }
    for (int i = 0; i < 8; ++i) mbar_init(smem_u32(&row_full[i]), 1);
    for (int i = 0; i < 4; ++i) mbar_init(smem_u32(&mid[i]), 128);   // every thread of the warpgroup
    mbar_init(smem_u32(x_full), 1);
    mbar_init(smem_u32(peer_free), 1);
    fence_mbar_init();
  }
  for (uint32_t i = tid; i < TR_SLOT_BYTES / 16; i += WS_THREADS)   // slot 1 is never TMA-loaded: its padding is zeroed here
    asm volatile("st.shared.v4.u32 [%0], {%1, %1, %1, %1};" ::"r"(smem_u32(smem + TR_SLOT1) + 16 * i), "r"(0) : "memory");
  fence_async_smem();
  cluster_sync();                                // both CTAs' barriers are initialised before any remote access

  if (wg == 2) {                                 // producer warp: one lane loads every tap of every layer and clip
    if (tid == NUM_THREADS) {
      for (int u = 0; u < my_clips * p.L; ++u) {   // u: layers loaded so far; tap t of each goes to ring slot t
        const int l = u % p.L;
        for (int t = 0; t < 9; ++t) {
          if (u > 0) mbar_wait(smem_u32(&empty[t]), (uint32_t)(u - 1) & 1u);
          mbar_expect_tx(smem_u32(&full[t]), TR_TAP);
          bulk_load_1d(smem_u32(smem + t * TR_TAP), p.wpk + ((size_t)l * 9 + t) * TR_TAP, TR_TAP, smem_u32(&full[t]));
        }
      }
    }
    __syncwarp();
    cluster_sync();
    return;
  }

  const int wq = (tid >> 5) & 3, lane = tid & 31;
  const bool leader = (tid & 127) == 0;          // issues this warpgroup's boundary-row copies
  const uint32_t wring_a = smem_u32(smem);
  auto slot_a = [&](uint32_t i) { return wring_a + (i ? TR_SLOT1 : TR_SLOT0); };
  const int y0 = 16 * (int)rank;                 // first image row of this CTA
  // this CTA's boundary row (buffer row 16 for r = 0, 1 for r = 1) -> the partner's halo row (0, resp. 17); column 1 on
  const uint32_t edge_src = (rank == 0 ? 16u : 1u) * TR_ROW_BYTES + 128u;
  const uint32_t edge_dst = (rank == 0 ? 0u : 17u) * TR_ROW_BYTES + 128u;
  const int sa = wg == 0 ? 0 : 3, sb = wg == 0 ? 1 : 2;   // this warpgroup's first and second strip
  const int my_turn = 1 + wg, other_turn = 2 - wg;        // named barrier 1 + g: warpgroup g may issue a strip
  auto load_x = [&](int n) {
    mbar_expect_tx(smem_u32(x_full), TR_SLOT_BYTES);
    tma_load_4d(slot_a(0), &xmap, smem_u32(x_full), 0, -1, y0 - 1, n);
  };
  // wait for the partner's rows of strips s - 1 .. s + 1 in slot i
  auto wait_rows = [&](uint32_t i, int s, uint32_t par) {
    for (int x = s > 0 ? s - 1 : 0; x <= (s < 3 ? s + 1 : 3); ++x) mbar_wait(smem_u32(&row_full[4 * i + x]), par);
  };
  if (tid == 0 && my_clips > 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&xmap) : "memory");
    load_x(cl);
  }

  float acc0[64], acc1[64];                      // strips sa and sb
  uint32_t ph = 0;                               // bit i: parity of the next phase of row_full[i][.] and mid[.][i]
  for (int k = 0; k < my_clips; ++k) {
    const int n = cl + k * G;
    for (int l = 0; l < p.L; ++l) {
      const uint32_t si = (uint32_t)l & 1u, so = si ^ 1u, par = (ph >> si) & 1u;
      const uint32_t wpar = (uint32_t)(k * p.L + l) & 1u;   // parity of full[.] for this layer's taps
      const uint32_t in_a = slot_a(si), out_a = slot_a(so);
      const bool last_turn = k + 1 == my_clips && l + 1 == p.L;

      if (l == 0) mbar_wait(smem_u32(x_full), (uint32_t)k & 1u);
      else wait_rows(si, sa, par);
      if (wg == 1 || k > 0 || l > 0) named_bar_sync(my_turn, 2 * 128);
      trunk_issue_strip(acc0, wring_a, full, wpar, in_a + (uint32_t)(TILE_COLS * sa) * 128u);
      named_bar_arrive(other_turn, 2 * 128);

      const float* bl = p.bias + 64 * l;
      const float b[2] = {bl[16 * wq + (lane >> 2)], bl[16 * wq + 8 + (lane >> 2)]};
      const bool res = (p.res_mask >> l) & 1u;
      auto epilogue = [&](const float (&acc)[64], int s) {   // E(l, s), then its boundary-row copy
        // once per strip: the element loop is compiled per activation
        if ((p.relu_mask >> l) & 1u) trunk_epilogue<TECO_ACT_RELU>(acc, b, out_a, TILE_COLS * s, res, wq, lane);
        else if ((p.lrelu_mask >> l) & 1u) trunk_epilogue<TECO_ACT_LRELU02>(acc, b, out_a, TILE_COLS * s, res, wq, lane);
        else trunk_epilogue<TECO_ACT_NONE>(acc, b, out_a, TILE_COLS * s, res, wq, lane);
        fence_async_smem();                      // the stmatrix writes -> visible to the MMAs and the bulk copy
        if (s == sb) mbar_arrive(smem_u32(&mid[2 * wg + so]));
        named_bar_sync(3 + wg, 128);
        if (leader) {
          const uint32_t e = (uint32_t)s * TR_STRIP_EDGE, bar = smem_u32(&row_full[4 * so + s]);
          mbar_expect_tx(bar, TR_STRIP_EDGE);    // the partner's row of this strip and layer
          bulk_copy_to_peer(mapa_shared(out_a + edge_dst + e, peer), out_a + edge_src + e, TR_STRIP_EDGE, mapa_shared(bar, peer));
        }
      };
      wgmma_wait_all_fence(acc0);                // the first strip has completed: its epilogue runs under the other
      epilogue(acc0, sa);                        // warpgroup's strip

      if (l > 0) {
        wait_rows(si, sb, par);
        mbar_wait(smem_u32(&mid[2 * (wg ^ 1) + si]), par);   // the other warpgroup's E(l - 1, 2 - wg)
        ph ^= 1u << si;
      }
      named_bar_sync(my_turn, 2 * 128);
      trunk_issue_strip(acc1, wring_a, full, wpar, in_a + (uint32_t)(TILE_COLS * sb) * 128u);
      if (!(wg == 1 && last_turn)) named_bar_arrive(other_turn, 2 * 128);
      trunk_release_taps<0>(empty, lane == 0);   // ring slot t as the second strip's tap t completes
      wgmma_wait_all_fence(acc1);
      epilogue(acc1, sb);
    }
    // the partner's rows of the last layer: no layer reads them, but their copies must have landed before the slot is
    // reused
    const uint32_t sf = (uint32_t)((p.L - 1) & 1) ^ 1u;
    for (int x = 0; x < 4; ++x) mbar_wait(smem_u32(&row_full[4 * sf + x]), (ph >> sf) & 1u);
    ph ^= 1u << sf;
    named_bar_sync(5, NUM_THREADS);              // both warpgroups' last epilogues are in place
    trunk_store_rows(slot_a(1), p.a, n, y0, tid);
    if (p.L > 1) trunk_store_rows(slot_a(0), p.b, n, y0, tid);
    fence_async_smem();                          // these generic reads before the next clip's TMA and bulk-copy writes
    named_bar_sync(5, NUM_THREADS);
    if (tid == 0 && k + 1 < my_clips) {
      mbar_arrive_peer(mapa_shared(smem_u32(peer_free), peer));
      mbar_wait(smem_u32(peer_free), (uint32_t)k & 1u);   // the partner has this CTA's last rows: their sources are free
      load_x(n + G);
    }
  }
  cluster_sync();                                // no CTA leaves while its partner may still address its shared memory
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

// The 4x4 stride-2 SAME convolution w[4,4,cin,cout] as a 3x3 one on its space-to-depth-2 input (teco_conv4x4s2_tc):
// W'[ty][tx][(py*2 + px)*cin + ci][co] = w[2ty + py - 1][2tx + px - 1][ci][co], zero where a kernel index falls outside
// 0..3.  dgrad == 0 packs W' in pack_conv3x3_kernel's image ([4cin/64][9][cout][64]); dgrad == 1 packs the input-gradient
// convolution of W', taps flipped and channels swapped ([cout/64][9][4cin][64]).
__global__ void pack_conv4x4s2_kernel(const float* __restrict__ w, int cin, int cout, int dgrad, __nv_bfloat16* __restrict__ out) {
  const int kdim = dgrad ? cout : 4 * cin, ndim = dgrad ? 4 * cin : cout;
  const long long total = 9LL * kdim * ndim;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i & 7);
    const int jpos = (int)((i >> 3) & 7);
    long long t = i >> 6;
    const int n = (int)(t % ndim);
    t /= ndim;
    const int tap = (int)(t % 9);
    const int k = (int)(t / 9) * 64 + (jpos ^ (n & 7)) * 8 + e;
    const int s = dgrad ? 8 - tap : tap;         // tap of W'
    const int sc = dgrad ? n : k;                // space-to-depth channel (phase, ci)
    const int co = dgrad ? k : n;
    const int ph = sc / cin, ci = sc - ph * cin;
    const int ky = 2 * (s / 3) + (ph >> 1) - 1, kx = 2 * (s % 3) + (ph & 1) - 1;
    float v = 0.f;
    if (ky >= 0 && ky < 4 && kx >= 0 && kx < 4) v = w[((long long)(ky * 4 + kx) * cin + ci) * cout + co];
    out[i] = __float2bfloat16_rn(v);
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                     CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                     CUtensorMapFloatOOBfill);

void* driver_entry(const char* name) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
    return p;
  return nullptr;
}

PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) fn = (PFN_encodeTiled)driver_entry("cuTensorMapEncodeTiled");
  return fn;
}

PFN_encodeIm2col get_encode_im2col() {
  static PFN_encodeIm2col fn = nullptr;
  if (!fn) fn = (PFN_encodeIm2col)driver_entry("cuTensorMapEncodeIm2col");
  return fn;
}

// NHWC bf16 activations [N,H,W,C] as a 4-D map whose box is box_h rows x box_w pixels x 64 channels (SWIZZLE_128B, zero
// fill): by default one tile's halo
int encode_halo_map(CUtensorMap* map, const void* x, int N, int H, int W, int C, const char* who, int box_w = HALO_COLS,
                    int box_h = HALO_ROWS) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    teco_set_error("%s: cuTensorMapEncodeTiled is unavailable (no CUDA driver?)", who);
    return TECO_E_CUDA;
  }
  const cuuint64_t gdim[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t gstr[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)CB, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
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

// conv3x3_im2col_kernel's maps: x [N,H,W,Cin] in im2col mode, IC_PIX pixels x 64 channels per load with the 3 x 3 'SAME'
// bounding box (corners -1, -1: output pixel (y, x) starts at input (y - 1, x - 1)); y as a 2-D [N*H*W, Cout] view
// stored in boxes of IC_PIX pixels x 64 channels.  Both SWIZZLE_128B.
int encode_im2col_maps(CUtensorMap* xmap, CUtensorMap* ymap, const void* x, const void* y, int N, int H, int W, int Cin,
                       int Cout) {
  const char* who = "teco_conv3x3_im2col_tc";
  PFN_encodeIm2col enc = get_encode_im2col();
  if (!enc || !get_encode()) {
    teco_set_error("%s: cuTensorMapEncodeIm2col is unavailable (no CUDA driver?)", who);
    return TECO_E_CUDA;
  }
  const cuuint64_t gdim[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t gstr[3] = {(cuuint64_t)Cin * 2, (cuuint64_t)W * Cin * 2, (cuuint64_t)H * W * Cin * 2};
  const int lower[2] = {-1, -1}, upper[2] = {-1, -1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult cr = enc(xmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), gdim, gstr, lower, upper, CB, IC_PIX,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    teco_set_error("%s: cuTensorMapEncodeIm2col failed with CUresult %d (N=%d H=%d W=%d C=%d)", who, (int)cr, N, H, W, Cin);
    return TECO_E_CUDA;
  }
  const cuuint64_t ydim[2] = {(cuuint64_t)Cout, (cuuint64_t)N * H * W};
  const cuuint64_t ystr[1] = {(cuuint64_t)Cout * 2};
  const cuuint32_t ybox[2] = {(cuuint32_t)CB, (cuuint32_t)IC_PIX};
  cr = get_encode()(ymap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(y), ydim, ystr, ybox, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    teco_set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d (output N*H*W=%lld C=%d)", who, (int)cr,
                   (long long)N * H * W, Cout);
    return TECO_E_CUDA;
  }
  return TECO_OK;
}

using KernelT = void (*)(const CUtensorMap, const TcParams);

// The mode-0 launches that conv3x3_ws_kernel does not take (Cin > 64, Cout not a multiple of 64 or an fp32 output), NT
// output channels per CTA
KernelT pick_kernel(int nt) {
  if (nt == 64) return conv3x3_wgmma_kernel<64>;
  if (nt == 32) return conv3x3_wgmma_kernel<32>;
  return conv3x3_wgmma_kernel<16>;
}

using WsKernelT = void (*)(const CUtensorMap, const CUtensorMap, const CUtensorMap, const TcParams);

// Mode 0 on the warp-specialised kernel: the full K without a pool on conv3x3_ws_kernel<0>, every other (k_live, pool) on
// its conv3x3_ws_live_kernel instance
WsKernelT pick_ws_kernel(int k_live, int pool) {
  if (k_live == 1) return pool ? conv3x3_ws_live_kernel<1, true> : conv3x3_ws_live_kernel<1, false>;
  if (k_live == 2) return pool ? conv3x3_ws_live_kernel<2, true> : conv3x3_ws_live_kernel<2, false>;
  return pool ? conv3x3_ws_live_kernel<CB / 16, true> : conv3x3_ws_kernel<0>;
}

// CTAs of `kern` resident per SM at `smem` bytes of dynamic shared memory; the opt-in shared-memory attribute is set on
// first use and the answer cached per (kernel, size), so a launch costs no extra driver calls.
int resident_ctas(const void* kern, size_t smem, int* per_sm, int threads = NUM_THREADS) {
  struct Entry { const void* kern; size_t smem; int per_sm; };
  static Entry cache[32];
  static int used = 0;
  for (int i = 0; i < used; ++i)
    if (cache[i].kern == kern && cache[i].smem == smem) { *per_sm = cache[i].per_sm; return TECO_OK; }
  bool attr_set = false;
  for (int i = 0; i < used; ++i) attr_set |= cache[i].kern == kern;
  if (!attr_set) TECO_CUDA_CALL(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX));
  int n = 0;
  TECO_CUDA_CALL(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, threads, smem));
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
  const int nt = d->Cout % 64 == 0 ? 64 : (d->Cout % 32 == 0 ? 32 : 16);   // output channels per CTA
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
  int per_sm = 0;
  // one K block and 64-channel bf16 output slices, as every mode-1 launch has: the warp-specialised kernel
  const bool ws = p.nblk == 1 && d->Cout % 64 == 0 && !out_f32;
  TECO_CHECK_ARG(!d->pool || (ws && d->mode == 0 && !res && d->H >= 2 && d->W >= 2),
                 "teco_conv3x3_tc: pool needs mode 0, Cin 64, Cout a multiple of 64, H, W >= 2 and no residual or fp32 output");
  if (ws) {
    // output and residual: one warpgroup's box of 16 rows x 8 pixels (a whole tile; 16 x 16 of the 2H x 2W output in
    // mode 1) x 64 channels; pooled, 8 rows x 4 pixels of the H / 2 x W / 2 output
    const int s = d->mode == 1 ? 2 : 1;
    CUtensorMap ymap, rmap;
    int rc_map = d->pool ? encode_halo_map(&ymap, y, d->N, d->H / 2, d->W / 2, d->Cout, "teco_conv3x3_tc", TILE_COLS / 2, TILE_ROWS / 2)
                         : encode_halo_map(&ymap, y, d->N, s * d->H, s * d->W, d->Cout, "teco_conv3x3_tc", s * TILE_COLS, TILE_ROWS);
    if (rc_map != TECO_OK) return rc_map;
    rmap = ymap;
    if (res && res != y) {
      rc_map = encode_halo_map(&rmap, res, d->N, d->H, d->W, d->Cout, "teco_conv3x3_tc", TILE_COLS, TILE_ROWS);
      if (rc_map != TECO_OK) return rc_map;
    }
    const WsKernelT kern = d->mode == 1 ? conv3x3_ws_kernel<1> : pick_ws_kernel(d->k_live, d->pool);
    const size_t ws_smem = d->mode == 1 ? WsCfg<1>::SMEM : WsCfg<0>::SMEM;
    const int rc_occ = resident_ctas((const void*)kern, ws_smem, &per_sm, WS_THREADS);
    if (rc_occ != TECO_OK) return rc_occ;
    const int nsplit_ws = d->Cout / 64;
    const long long slots = ((long long)per_sm * teco_sm_count() + nsplit_ws - 1) / nsplit_ws;
    const unsigned gx = (unsigned)(tiles < slots ? tiles : slots);
    kern<<<dim3(gx, (unsigned)nsplit_ws), WS_THREADS, ws_smem, stream>>>(tmap, ymap, rmap, p);
    TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_tc");
    return TECO_OK;
  }
  const KernelT kern = pick_kernel(nt);
  const int rc_occ = resident_ctas((const void*)kern, smem, &per_sm);
  if (rc_occ != TECO_OK) return rc_occ;
  // persistent: as many CTAs as are resident at once, spread over the Cout splits
  const long long slots = ((long long)per_sm * teco_sm_count() + nsplit - 1) / nsplit;
  const unsigned gx = (unsigned)(tiles < slots ? tiles : slots);
  kern<<<dim3(gx, (unsigned)nsplit), NUM_THREADS, smem, stream>>>(tmap, p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_tc");
  return TECO_OK;
}

int launch_conv3x3_im2col(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, void* y,
                          cudaStream_t stream) {
  IcParams p;
  p.H = d->H; p.W = d->W; p.Cout = d->Cout; p.nblk = d->Cin / CB; p.act = d->act;
  p.wpk = (const uint8_t*)wpk; p.bias = bias;
  const long long tiles = ((long long)d->N * d->H * d->W + IC_PIX - 1) / IC_PIX;
  TECO_CHECK_ARG(tiles * IC_PIX < (1LL << 31), "teco_conv3x3_im2col_tc: too many pixels");
  p.num_tiles = (int)tiles;
  CUtensorMap xmap, ymap;
  const int rc_map = encode_im2col_maps(&xmap, &ymap, x, y, d->N, d->H, d->W, d->Cin, d->Cout);
  if (rc_map != TECO_OK) return rc_map;
  int per_sm = 0;
  const int rc_occ = resident_ctas((const void*)conv3x3_im2col_kernel, IC_SMEM, &per_sm, WS_THREADS);
  if (rc_occ != TECO_OK) return rc_occ;
  // persistent: as many CTAs as are resident at once, spread over the Cout slices
  const int nsplit = d->Cout / 64;
  const long long slots = ((long long)per_sm * teco_sm_count() + nsplit - 1) / nsplit;
  const unsigned gx = (unsigned)(tiles < slots ? tiles : slots);
  conv3x3_im2col_kernel<<<dim3(gx, (unsigned)nsplit), WS_THREADS, IC_SMEM, stream>>>(xmap, ymap, p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_im2col_tc");
  return TECO_OK;
}

// conv3x3_f32out_kernel's fp32 residual / output [N,H,W,C] as a 3-D [N, H, W*C] view stored in boxes of 16 rows x 8 C
// floats (no swizzle, zero fill).  The row stride W*C*4 must be a multiple of 16 bytes (the caller checks).
int encode_f32_box_map(CUtensorMap* map, const float* t, int N, int H, int W, int C) {
  const char* who = "teco_conv3x3_f32out_tc";
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    teco_set_error("%s: cuTensorMapEncodeTiled is unavailable (no CUDA driver?)", who);
    return TECO_E_CUDA;
  }
  const cuuint64_t gdim[3] = {(cuuint64_t)W * C, (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t gstr[2] = {(cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
  const cuuint32_t box[3] = {(cuuint32_t)(TILE_COLS * C), (cuuint32_t)TILE_ROWS, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult cr = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(t), gdim, gstr, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    teco_set_error("%s: cuTensorMapEncodeTiled failed with CUresult %d (N=%d H=%d W=%d C=%d)", who, (int)cr, N, H, W, C);
    return TECO_E_CUDA;
  }
  return TECO_OK;
}

int launch_conv3x3_f32out(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, const float* res_f32,
                          float* out_f32, cudaStream_t stream) {
  F32Params p;
  p.C = d->out_f32_c; p.act = d->act; p.has_res = res_f32 != nullptr;
  p.post_scale = d->post_scale; p.post_shift = d->post_shift;
  p.wpk = (const uint8_t*)wpk; p.bias = bias;
  p.tiles_x = teco_ceil_div(d->W, TILE_COLS);
  p.tiles_y = teco_ceil_div(d->H, TILE_ROWS);
  const long long tiles = (long long)d->N * p.tiles_x * p.tiles_y;
  TECO_CHECK_ARG(tiles < (1LL << 31), "teco_conv3x3_f32out_tc: too many tiles");
  p.num_tiles = (int)tiles;
  CUtensorMap tmap, omap, rmap;
  int rc = encode_halo_map(&tmap, x, d->N, d->H, d->W, d->Cin, "teco_conv3x3_f32out_tc");
  if (rc != TECO_OK) return rc;
  rc = encode_f32_box_map(&omap, out_f32, d->N, d->H, d->W, p.C);
  if (rc != TECO_OK) return rc;
  rmap = omap;
  if (res_f32) {
    rc = encode_f32_box_map(&rmap, res_f32, d->N, d->H, d->W, p.C);
    if (rc != TECO_OK) return rc;
  }
  int per_sm = 0;
  const auto kern = d->k_live == 1 ? conv3x3_f32out_kernel<1> : d->k_live == 2 ? conv3x3_f32out_kernel<2> : conv3x3_f32out_kernel<4>;
  rc = resident_ctas((const void*)kern, F32_SMEM, &per_sm, WS_THREADS);
  if (rc != TECO_OK) return rc;
  const long long slots = (long long)per_sm * teco_sm_count();   // persistent: as many CTAs as are resident at once
  const unsigned gx = (unsigned)(tiles < slots ? tiles : slots);
  kern<<<gx, WS_THREADS, F32_SMEM, stream>>>(tmap, omap, rmap, p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_f32out_tc");
  return TECO_OK;
}

// The plans conv3x3_trunk_cluster_kernel runs: 32 x 32 images; layer 0 reads x_in (buffer 0) into buffer 1 without a
// residual; every later layer reads the previous layer's output and writes the other one of buffers 1 and 2, with no
// residual or an in-place one on a buffer an earlier layer wrote.  So layer l writes buffer 1 (slot 1) for even l and
// buffer 2 (slot 0) for odd l, and no layer reads a buffer's contents from before the launch except x_in.
bool trunk_plan_fits(int H, int W, int L, const int32_t* plan) {
  if (H != LIN_W || W != LIN_W || L < 1 || L > LIN_MAX_LAYERS) return false;
  for (int l = 0; l < L; ++l) {
    const int32_t* pl = plan + 4 * l;
    const int in = l == 0 ? 0 : (l & 1 ? 1 : 2), out = l & 1 ? 2 : 1;
    if (pl[0] != in || pl[1] != out || pl[3] < 0 || pl[3] >= TECO_ACT_TANH24) return false;
    if (pl[2] != -1 && !(pl[2] == out && (out == 1 ? l >= 2 : l >= 3))) return false;
  }
  return true;
}

// Clusters of conv3x3_trunk_cluster_kernel resident at once on this device (cached).
int trunk_clusters(int* G) {
  static int cached = 0;
  if (!cached) {
    TECO_CUDA_CALL(cudaFuncSetAttribute(conv3x3_trunk_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TR_SMEM));
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(2 * (unsigned)teco_sm_count());
    cfg.blockDim = dim3(WS_THREADS);
    cfg.dynamicSmemBytes = TR_SMEM;
    int n = 0;
    TECO_CUDA_CALL(cudaOccupancyMaxActiveClusters(&n, conv3x3_trunk_cluster_kernel, &cfg));
    if (n < 1) {
      teco_set_error("conv3x3_trunk_cluster_kernel: no cluster of two CTAs with %zu bytes of shared memory each fits", TR_SMEM);
      return TECO_E_CUDA;
    }
    cached = n;
  }
  *G = cached;
  return TECO_OK;
}

int launch_trunk(int N, int L, const void* x_in, void* buf_a, void* buf_b, const void* wpk_all, const float* bias_all,
                 const int32_t* plan, cudaStream_t stream) {
  TrunkParams p = {};
  p.N = N; p.L = L;
  for (int l = 0; l < L; ++l) {
    if (plan[4 * l + 3] == TECO_ACT_RELU) p.relu_mask |= 1ull << l;
    if (plan[4 * l + 3] == TECO_ACT_LRELU02) p.lrelu_mask |= 1ull << l;
    if (plan[4 * l + 2] >= 0) p.res_mask |= 1ull << l;
  }
  p.wpk = (const uint8_t*)wpk_all; p.bias = bias_all;
  p.a = (__nv_bfloat16*)buf_a; p.b = (__nv_bfloat16*)buf_b;
  CUtensorMap xmap;                 // one CTA's slot: 18 rows x 34 pixels x 64 channels
  const int rc_map = encode_halo_map(&xmap, x_in, N, LIN_W, LIN_W, 64, "teco_conv3x3_lin_tc", TR_COLS, TR_ROWS);
  if (rc_map != TECO_OK) return rc_map;
  int G = 0;
  const int rc = trunk_clusters(&G);
  if (rc != TECO_OK) return rc;
  const unsigned grid = 2u * (unsigned)(N < G ? N : G);
  conv3x3_trunk_cluster_kernel<<<grid, WS_THREADS, TR_SMEM, stream>>>(xmap, p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_lin_tc");
  return TECO_OK;
}

// k_live 0 is every K-step; 1, 2 or 4 steps of 16 channels per tap only make sense with one 64-channel K block
bool k_live_ok(const teco_tc_desc* d) {
  return d->k_live == 0 || (d->Cin == CB && (d->k_live == 1 || d->k_live == 2 || d->k_live == 4));
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
  // mode 1 runs on conv3x3_ws_kernel<1> only
  TECO_CHECK_ARG(d->mode == 0 || d->Cin == 64, "teco_conv3x3_tc: mode 1 needs Cin 64 (got %d)", d->Cin);
  TECO_CHECK_ARG(d->mode == 0 || d->Cout % 64 == 0, "teco_conv3x3_tc: mode 1 needs Cout a multiple of 64 (got %d)", d->Cout);
  TECO_CHECK_ARG(d->mode == 0 || !res, "teco_conv3x3_tc: mode 1 takes no residual");
  TECO_CHECK_ARG(d->mode == 0 || !out_f32, "teco_conv3x3_tc: mode 1 takes no fp32 output, only a bf16 y");
  TECO_CHECK_ARG(d->act >= 0 && d->act <= TECO_ACT_SIGMOID, "teco_conv3x3_tc: unknown activation %d", d->act);
  TECO_CHECK_ARG(!out_f32 || (d->out_f32_c > 0 && d->out_f32_c <= d->Cout), "teco_conv3x3_tc: bad out_f32_c");
  TECO_CHECK_ARG((((uintptr_t)x) & 15) == 0 && (((uintptr_t)wpk) & 15) == 0 && (((uintptr_t)y) & 15) == 0 &&
                     (((uintptr_t)res) & 15) == 0,
                 "teco_conv3x3_tc: tensors must be 16-byte aligned");
  TECO_CHECK_ARG(k_live_ok(d), "teco_conv3x3_tc: k_live must be 0, or 1, 2 or 4 with Cin 64 (got %d, Cin %d)", d->k_live, d->Cin);
  TECO_CHECK_ARG(d->pool == 0 || d->pool == 1, "teco_conv3x3_tc: pool must be 0 or 1 (got %d)", d->pool);
  return launch_conv3x3(d, x, wpk, bias, res, y, res_f32, out_f32, (cudaStream_t)stream);
}

extern "C" int teco_conv3x3_im2col_tc(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, void* y,
                                      void* stream) {
  TECO_CHECK_ARG(d && x && wpk && y, "teco_conv3x3_im2col_tc: NULL argument");
  TECO_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0, "teco_conv3x3_im2col_tc: bad shape N=%d H=%d W=%d", d->N, d->H, d->W);
  TECO_CHECK_ARG(d->Cin >= 64 && d->Cin % 64 == 0 && d->Cin <= 512,
                 "teco_conv3x3_im2col_tc: Cin must be a multiple of 64 in [64,512] (got %d)", d->Cin);
  TECO_CHECK_ARG(d->Cout >= 64 && d->Cout % 64 == 0 && d->Cout <= 512,
                 "teco_conv3x3_im2col_tc: Cout must be a multiple of 64 in [64,512] (got %d)", d->Cout);
  TECO_CHECK_ARG(d->mode == 0 && d->out_f32_c == 0 && d->k_live == 0 && d->pool == 0,
                 "teco_conv3x3_im2col_tc: mode 0 with a bf16 output only (k_live and pool 0)");
  TECO_CHECK_ARG(d->act >= 0 && d->act <= TECO_ACT_SIGMOID, "teco_conv3x3_im2col_tc: unknown activation %d", d->act);
  TECO_CHECK_ARG((((uintptr_t)x) & 15) == 0 && (((uintptr_t)wpk) & 15) == 0 && (((uintptr_t)y) & 15) == 0,
                 "teco_conv3x3_im2col_tc: tensors must be 16-byte aligned");
  return launch_conv3x3_im2col(d, x, wpk, bias, y, (cudaStream_t)stream);
}

extern "C" int teco_conv3x3_f32out_tc(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, const void* res,
                                      void* y, const float* res_f32, float* out_f32, void* stream) {
  TECO_CHECK_ARG(d && x && wpk && out_f32, "teco_conv3x3_f32out_tc: NULL argument");
  TECO_CHECK_ARG(!res && !y, "teco_conv3x3_f32out_tc: fp32 output only (no bf16 output or residual)");
  TECO_CHECK_ARG(d->N > 0 && d->H > 0 && d->W > 0, "teco_conv3x3_f32out_tc: bad shape N=%d H=%d W=%d", d->N, d->H, d->W);
  TECO_CHECK_ARG(d->Cin == 64 && d->Cout == 16 && d->mode == 0,
                 "teco_conv3x3_f32out_tc: mode 0 with Cin 64 and Cout 16 only (got mode %d, Cin %d, Cout %d)", d->mode, d->Cin,
                 d->Cout);
  TECO_CHECK_ARG(d->act >= 0 && d->act <= TECO_ACT_SIGMOID, "teco_conv3x3_f32out_tc: unknown activation %d", d->act);
  TECO_CHECK_ARG(d->out_f32_c == 2 || d->out_f32_c == 3, "teco_conv3x3_f32out_tc: out_f32_c must be 2 or 3 (got %d)",
                 d->out_f32_c);
  TECO_CHECK_ARG(k_live_ok(d) && d->pool == 0, "teco_conv3x3_f32out_tc: k_live must be 0, 1, 2 or 4 and pool 0 (got %d, %d)",
                 d->k_live, d->pool);
  TECO_CHECK_ARG(((long long)d->W * d->out_f32_c * 4) % 16 == 0,
                 "teco_conv3x3_f32out_tc: an fp32 row (W*out_f32_c*4 = %lld bytes) must be a multiple of 16 bytes",
                 (long long)d->W * d->out_f32_c * 4);
  TECO_CHECK_ARG((((uintptr_t)x) & 15) == 0 && (((uintptr_t)wpk) & 15) == 0 && (((uintptr_t)res_f32) & 15) == 0 &&
                     (((uintptr_t)out_f32) & 15) == 0,
                 "teco_conv3x3_f32out_tc: tensors must be 16-byte aligned");
  return launch_conv3x3_f32out(d, x, wpk, bias, res_f32, out_f32, (cudaStream_t)stream);
}

// Shapes of the 4x4 stride-2 convolution on its space-to-depth-2 form: even H, W; Cin a multiple of 64 with 4 * Cin <= 512
// (the input of the forward 3x3 and the output of its input gradient); Cout a multiple of 64 in [64,512].
static int conv4x4s2_check(int N, int H, int W, int Cin, int Cout, const char* who) {
  TECO_CHECK_ARG(N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0, "%s: H and W must be even (got N=%d H=%d W=%d)", who, N, H, W);
  TECO_CHECK_ARG(Cin >= 64 && Cin % 64 == 0 && Cin <= 128, "%s: Cin must be 64 or 128 (got %d)", who, Cin);
  TECO_CHECK_ARG(Cout >= 64 && Cout % 64 == 0 && Cout <= 512, "%s: Cout must be a multiple of 64 in [64,512] (got %d)", who, Cout);
  return TECO_OK;
}

// The 3x3 launch on the half-resolution grid: 128-pixel tiles across images below conv3x3_tc's 16 x 8 tile, as FNet's
// small levels do.
static int launch_conv3x3_s2d(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, void* y,
                              cudaStream_t stream) {
  if (d->H < TILE_ROWS || d->W < TILE_COLS) return launch_conv3x3_im2col(d, x, wpk, bias, y, stream);
  return launch_conv3x3(d, x, wpk, bias, nullptr, y, nullptr, nullptr, stream);
}

extern "C" int teco_pack_conv4x4s2_bf16(const float* w, int32_t cin, int32_t cout, int32_t dgrad, void* wpk, void* stream) {
  TECO_CHECK_ARG(w && wpk, "teco_pack_conv4x4s2_bf16: NULL tensor");
  TECO_CHECK_ARG(dgrad == 0 || dgrad == 1, "teco_pack_conv4x4s2_bf16: dgrad must be 0 or 1 (got %d)", dgrad);
  const int rc = conv4x4s2_check(1, 2, 2, cin, cout, "teco_pack_conv4x4s2_bf16");
  if (rc != TECO_OK) return rc;
  const long long total = 36LL * cin * cout;
  int blocks = teco_ceil_div(total, 256);
  if (blocks > 4096) blocks = 4096;
  pack_conv4x4s2_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(w, cin, cout, dgrad, (__nv_bfloat16*)wpk);
  TECO_CUDA_LAUNCH_CHECK("teco_pack_conv4x4s2_bf16");
  return TECO_OK;
}

extern "C" int teco_conv4x4s2_tc(int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t act, const void* xs,
                                 const void* wpk, const float* bias, void* y, void* stream) {
  TECO_CHECK_ARG(xs && wpk && y, "teco_conv4x4s2_tc: NULL argument");
  const int rc = conv4x4s2_check(N, H, W, Cin, Cout, "teco_conv4x4s2_tc");
  if (rc != TECO_OK) return rc;
  TECO_CHECK_ARG(act >= 0 && act <= TECO_ACT_SIGMOID, "teco_conv4x4s2_tc: unknown activation %d", act);
  TECO_CHECK_ARG((((uintptr_t)xs) & 15) == 0 && (((uintptr_t)wpk) & 15) == 0 && (((uintptr_t)y) & 15) == 0,
                 "teco_conv4x4s2_tc: tensors must be 16-byte aligned");
  const teco_tc_desc d = {N, H / 2, W / 2, 4 * Cin, Cout, act, 0, 0, 1.f, 0.f};
  return launch_conv3x3_s2d(&d, xs, wpk, bias, y, (cudaStream_t)stream);
}

extern "C" int teco_conv4x4s2_dgrad_tc(int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, const void* dz,
                                       const void* wpk_t, void* dxs, void* stream) {
  TECO_CHECK_ARG(dz && wpk_t && dxs, "teco_conv4x4s2_dgrad_tc: NULL argument");
  const int rc = conv4x4s2_check(N, H, W, Cin, Cout, "teco_conv4x4s2_dgrad_tc");
  if (rc != TECO_OK) return rc;
  TECO_CHECK_ARG((((uintptr_t)dz) & 15) == 0 && (((uintptr_t)wpk_t) & 15) == 0 && (((uintptr_t)dxs) & 15) == 0,
                 "teco_conv4x4s2_dgrad_tc: tensors must be 16-byte aligned");
  const teco_tc_desc d = {N, H / 2, W / 2, Cout, 4 * Cin, TECO_ACT_NONE, 0, 0, 1.f, 0.f};
  return launch_conv3x3_s2d(&d, dz, wpk_t, nullptr, dxs, (cudaStream_t)stream);
}

extern "C" int teco_conv3x3_lin_in_smem(int32_t N, int32_t H, int32_t W, int32_t num_layers, const int32_t* plan_host) {
  return N > 0 && plan_host && trunk_plan_fits(H, W, num_layers, plan_host) ? 1 : 0;
}

extern "C" int teco_conv3x3_lin_tc(int32_t N, int32_t H, int32_t W, int32_t num_layers, const void* x_in, void* buf_a, void* buf_b,
                                   const void* wpk_all, const float* bias_all, const int32_t* plan_host, void* stream) {
  TECO_CHECK_ARG(teco_conv3x3_lin_in_smem(N, H, W, num_layers, plan_host),
                 "teco_conv3x3_lin_tc: needs N > 0, 32x32 images and a generator-trunk-shaped plan of 1..%d layers "
                 "(teco_conv3x3_lin_in_smem; got N=%d H=%d W=%d L=%d)", LIN_MAX_LAYERS, N, H, W, num_layers);
  TECO_CHECK_ARG(x_in && buf_a && buf_b && wpk_all && bias_all, "teco_conv3x3_lin_tc: NULL argument");
  TECO_CHECK_ARG((((uintptr_t)x_in) & 15) == 0 && (((uintptr_t)buf_a) & 15) == 0 && (((uintptr_t)buf_b) & 15) == 0 &&
                     (((uintptr_t)wpk_all) & 15) == 0,
                 "teco_conv3x3_lin_tc: tensors must be 16-byte aligned");
  return launch_trunk(N, num_layers, x_in, buf_a, buf_b, wpk_all, bias_all, plan_host, (cudaStream_t)stream);
}

extern "C" int teco_conv3x3_lin_clusters(void) {
  int G = 0;
  const int rc = trunk_clusters(&G);
  return rc == TECO_OK ? G : rc;
}
