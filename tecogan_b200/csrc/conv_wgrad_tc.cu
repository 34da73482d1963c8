// Weight gradient of the 3x3 stride-1 SAME convolution on the Hopper tensor cores (sm_90a, wgmma).
//
// Replaces the gradient TensorFlow computes for slim.conv2d (reference lib/ops.py:47-56) inside
// tf.train.AdamOptimizer.compute_gradients (reference lib/Teco.py:426,446-447):
//     dW[ky][kx][ci][co] += sum over pixels p of  X[p + (ky-1, kx-1)][ci] * dZ[p][co]
// i.e. one GEMM per tap with the PIXELS as the contraction dimension.  Both operands are NHWC bf16 with 64 channels per
// 128-byte row, so as wgmma operands they are "MN-major" (the M / N index -- the channel -- is the contiguous one, K = the
// pixel steps from row to row): exactly the SWIZZLE_128B image a TMA box leaves in shared memory, no transposition.
//   * CTA = one 8x16-pixel tile of one image and one (64 input channel, 64 output channel) block pair.
//   * A K-step is one image row of the tile = 16 consecutive pixels = two 8-row swizzle atoms (SBO = 1024 B).
//   * Three warpgroups, one per kernel row ky; each keeps the three taps of its row as three M = 64 x N = 64 register
//     accumulators.  Tap (ky, kx) of K-step r is the descriptor start address of halo row r + ky, pixel kx.
//   * Epilogue: (ci, co) fragments from registers -> 8-byte fp32 atomics (co, co + 1) into dW[3,3,Cin,Cout] (TF layout).
#include <cuda.h>
#include "teco_common.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace tcptx;

constexpr int WG_ROWS = 8, WG_COLS = 16;
constexpr int WG_HALO_BYTES = (WG_ROWS + 2) * (WG_COLS + 2) * 128;   // 23040
constexpr int WG_DZ_BYTES = WG_ROWS * WG_COLS * 128;                 // 16384
constexpr int WG_THREADS = 384;

struct WgParams {
  int N, H, W, Cin, Cout;      // real channel counts of dW
  int cob, tiles_x, tiles_y;   // 64-channel output blocks, tiles per image
  float* dw;
};

__global__ void __launch_bounds__(WG_THREADS)
conv3x3_wgrad_wgmma_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_dz, const WgParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* halo = smem;                                   // [10 rows][18 px][128 B]
  uint8_t* dzt = smem + ((WG_HALO_BYTES + 1023) & ~1023); // [8 rows][16 px][128 B]
  uint64_t* bar = reinterpret_cast<uint64_t*>(dzt + WG_DZ_BYTES);
  const int tid = threadIdx.x, ky = tid >> 7, wq = (tid >> 5) & 3, lane = tid & 31;

  int tile = blockIdx.x;
  const int tx = tile % p.tiles_x; tile /= p.tiles_x;
  const int ty = tile % p.tiles_y;
  const int n = tile / p.tiles_y;
  const int cb = blockIdx.y / p.cob, ob = blockIdx.y - cb * p.cob;
  const int x0 = tx * WG_COLS, y0 = ty * WG_ROWS;

  if (tid == 0) {
    mbar_init(smem_u32(bar), 1);
    fence_mbar_init();
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(smem_u32(bar), (uint32_t)(WG_HALO_BYTES + WG_DZ_BYTES));
    tma_load_4d(smem_u32(halo), &tmap_x, smem_u32(bar), cb * 64, x0 - 1, y0 - 1, n);   // zero fill = SAME padding
    tma_load_4d(smem_u32(dzt), &tmap_dz, smem_u32(bar), ob * 64, x0, y0, n);
  }
  float acc[3][32];   // written first by the r == 0 MMAs (scale-d 0)
  mbar_wait(smem_u32(bar), 0);
  const uint32_t halo_a = smem_u32(halo), dz_a = smem_u32(dzt);
  wgmma_fence();
#pragma unroll
  for (int r = 0; r < WG_ROWS; ++r) {
    const uint64_t b_desc = gmma_desc_sw128(dz_a + (uint32_t)(r * WG_COLS * 128), 8192u, 1024u);
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const uint32_t a0 = halo_a + (uint32_t)(((r + ky) * (WG_COLS + 2) + kx) * 128);
      Wgmma<64, 1, 1>::run(acc[kx], gmma_desc_sw128(a0, 8192u, 1024u), b_desc, r > 0 ? 1u : 0u);
    }
  }
  wgmma_commit();
  wgmma_wait_all();

  // ---- epilogue: register 4 j + 2 i + c of accumulator kx = (ci = 16 wq + lane / 4 + 8 i, co = 8 j + 2 (lane % 4) + c)
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int ci = cb * 64 + 16 * wq + (lane >> 2) + 8 * i;
    if (ci >= p.Cin) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      float* dst = p.dw + ((size_t)(3 * ky + kx) * p.Cin + ci) * p.Cout;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int co = ob * 64 + 8 * j + 2 * (lane & 3);
        if (co < p.Cout)   // Cout % 4 == 0: co and co + 1 are both in range, dst + co is 8-byte aligned
          atomicAdd(reinterpret_cast<float2*>(dst + co), make_float2(acc[kx][4 * j + 2 * i], acc[kx][4 * j + 2 * i + 1]));
      }
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled wg_get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
      fn = (PFN_encodeTiled)p;
  }
  return fn;
}

}  // namespace

extern "C" int teco_conv3x3_wgrad_tc(int32_t N, int32_t H, int32_t W, int32_t cin_pad, int32_t cout_pad, int32_t cin, int32_t cout,
                                     const void* x, const void* dz, float* dw, int32_t accumulate, void* stream) {
  TECO_CHECK_ARG(x && dz && dw, "teco_conv3x3_wgrad_tc: NULL tensor");
  TECO_CHECK_ARG(N > 0 && H > 0 && W > 0, "teco_conv3x3_wgrad_tc: bad shape N=%d H=%d W=%d", N, H, W);
  TECO_CHECK_ARG(cin_pad % 64 == 0 && cout_pad % 64 == 0 && cin > 0 && cout > 0 && cin <= cin_pad && cout <= cout_pad,
                 "teco_conv3x3_wgrad_tc: x / dz must carry multiples of 64 channels (got %d, %d for %d -> %d)", cin_pad, cout_pad, cin, cout);
  TECO_CHECK_ARG(cout % 4 == 0, "teco_conv3x3_wgrad_tc: Cout must be a multiple of 4 (channel pairs of the fragment), got %d", cout);
  TECO_CHECK_ARG((((uintptr_t)x) & 15) == 0 && (((uintptr_t)dz) & 15) == 0 && (((uintptr_t)dw) & 15) == 0,
                 "teco_conv3x3_wgrad_tc: tensors must be 16-byte aligned");
  cudaStream_t s = (cudaStream_t)stream;
  if (!accumulate) TECO_CUDA_CALL(cudaMemsetAsync(dw, 0, sizeof(float) * (size_t)9 * cin * cout, s));
  PFN_encodeTiled enc = wg_get_encode();
  if (!enc) {
    teco_set_error("teco_conv3x3_wgrad_tc: cuTensorMapEncodeTiled is unavailable (no CUDA driver?)");
    return TECO_E_CUDA;
  }
  CUtensorMap tx, tz;
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  {
    const cuuint64_t gdim[4] = {(cuuint64_t)cin_pad, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t gstr[3] = {(cuuint64_t)cin_pad * 2, (cuuint64_t)W * cin_pad * 2, (cuuint64_t)H * W * cin_pad * 2};
    const cuuint32_t box[4] = {64, WG_COLS + 2, WG_ROWS + 2, 1};
    CUresult cr = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(x), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { teco_set_error("teco_conv3x3_wgrad_tc: cuTensorMapEncodeTiled(x) failed with CUresult %d", (int)cr); return TECO_E_CUDA; }
  }
  {
    const cuuint64_t gdim[4] = {(cuuint64_t)cout_pad, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t gstr[3] = {(cuuint64_t)cout_pad * 2, (cuuint64_t)W * cout_pad * 2, (cuuint64_t)H * W * cout_pad * 2};
    const cuuint32_t box[4] = {64, WG_COLS, WG_ROWS, 1};
    CUresult cr = enc(&tz, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(dz), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (cr != CUDA_SUCCESS) { teco_set_error("teco_conv3x3_wgrad_tc: cuTensorMapEncodeTiled(dz) failed with CUresult %d", (int)cr); return TECO_E_CUDA; }
  }
  WgParams p;
  p.N = N; p.H = H; p.W = W; p.Cin = cin; p.Cout = cout;
  p.cob = teco_ceil_div(cout, 64);
  p.tiles_x = teco_ceil_div(W, WG_COLS);
  p.tiles_y = teco_ceil_div(H, WG_ROWS);
  p.dw = dw;
  const long long tiles = (long long)N * p.tiles_x * p.tiles_y;
  TECO_CHECK_ARG(tiles < (1LL << 31), "teco_conv3x3_wgrad_tc: too many tiles");
  const int cib = teco_ceil_div(cin, 64);
  const size_t smem = 1024 + ((WG_HALO_BYTES + 1023) & ~1023) + WG_DZ_BYTES + 64;
  static bool attr = false;
  if (!attr) {
    TECO_CUDA_CALL(cudaFuncSetAttribute(conv3x3_wgrad_wgmma_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  conv3x3_wgrad_wgmma_kernel<<<dim3((unsigned)tiles, (unsigned)(cib * p.cob)), WG_THREADS, smem, s>>>(tx, tz, p);
  TECO_CUDA_LAUNCH_CHECK("teco_conv3x3_wgrad_tc");
  return TECO_OK;
}
