// lpips.cu -- the parts of LPIPS-AlexNet (v0.1) that the convolution kernels do not cover: the network's input scaling,
// the 3x3 / 2 max-pool between its convolutions, and the LPIPS head (channel normalisation, squared difference, learned
// per-channel weights, mean over pixels).  Reference: metrics.py:183-202 (the LPIPS / tLP100 terms of the evaluation loop),
// LPIPSmodels/util.py:142-144 (im2tensor), networks_basic.py:111-112,131-177 (scaling layer and PNetLin head, v0.1),
// util.py:72-75 (normalize_tensor), pretrained_networks.py:67-76 (torchvision alexnet().features sliced after each ReLU).
// The five convolutions run through teco_conv2d_f32 with a fused ReLU.  Everything is fp32 on the CUDA cores; the head
// accumulates in float64 because tLP100 is 100 x the difference of two small distances.
#include "teco_common.cuh"

namespace {
constexpr int TPB = 256;
constexpr int HEAD_MAXV = 12;                   // channels per lane: C <= 32 * 12 = 384 (AlexNet's widest layer)
constexpr int HEAD_MAXP = 256;                  // pairs per head launch (indices travel in the kernel parameters)

// im2tensor then the v0.1 scaling layer, bit for bit: x = float32(u8 / 127.5 - 1) with the arithmetic in float64 (numpy),
// then (x - shift[c]) / scale[c] as an fp32 subtract and a correctly rounded fp32 divide (torch).
__global__ void __launch_bounds__(TPB) lpips_input_kernel(const uint8_t* __restrict__ img, int H, int W, int y0, int x0,
                                                          int h, int w, long long total, float* __restrict__ x) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int c = (int)(i % 3);
    long long t = i / 3;
    const int col = (int)(t % w);
    t /= w;
    const int row = (int)(t % h);
    const long long n = t / h;
    const uint8_t u = img[((n * H + y0 + row) * W + x0 + col) * 3 + c];
    const float v = (float)__dsub_rn(__ddiv_rn((double)u, 127.5), 1.0);
    const float shift = c == 0 ? -.030f : (c == 1 ? -.088f : -.188f);
    const float scale = c == 0 ? .458f : (c == 1 ? .448f : .450f);
    x[i] = __fdiv_rn(__fsub_rn(v, shift), scale);
  }
}

// torch MaxPool2d(3, 2): no padding, floor.  NaN wins, as in torch's CPU and CUDA kernels.
__global__ void __launch_bounds__(TPB) maxpool3s2_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W,
                                                         int C, int OH, int OW, long long total) {
  for (long long i = blockIdx.x * (long long)TPB + threadIdx.x; i < total; i += (long long)gridDim.x * TPB) {
    const int c = (int)(i % C);
    long long t = i / C;
    const int ox = (int)(t % OW);
    t /= OW;
    const int oy = (int)(t % OH);
    const long long n = t / OH;
    const float* p = x + ((n * H + 2 * oy) * W + 2 * ox) * C + c;
    float m = p[0];
#pragma unroll
    for (int dy = 0; dy < 3; ++dy)
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const float v = p[((long long)dy * W + dx) * C];
        if (v > m || isnan(v)) m = v;
      }
    y[i] = m;
  }
}

struct HeadPairs {
  int32_t a[HEAD_MAXP], b[HEAD_MAXP];
};

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per pixel: lane l holds channels l, l+32, ... of both feature vectors in registers, so the norms and the
// weighted normalised difference come from one read of each map.  Per-pixel terms are summed in float64 per lane, then per
// CTA, and each CTA adds its share of the pixel mean into out[pair] (blockIdx.y = pair).
__global__ void __launch_bounds__(TPB) lpips_head_kernel(const float* __restrict__ fa, const float* __restrict__ fb,
                                                         const HeadPairs pr, int HW, int C, const float* __restrict__ lin,
                                                         double* __restrict__ out, double inv_hw) {
  const int p = blockIdx.y;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const float* A = fa + (size_t)pr.a[p] * HW * C;
  const float* B = fb + (size_t)pr.b[p] * HW * C;
  double wl[HEAD_MAXV];
#pragma unroll
  for (int k = 0; k < HEAD_MAXV; ++k) wl[k] = (lane + 32 * k < C) ? (double)lin[lane + 32 * k] : 0.0;
  double acc = 0.0;
  for (int pix = blockIdx.x * (TPB / 32) + wid; pix < HW; pix += gridDim.x * (TPB / 32)) {
    const float* a = A + (size_t)pix * C;
    const float* b = B + (size_t)pix * C;
    double va[HEAD_MAXV], vb[HEAD_MAXV], sa = 0.0, sb = 0.0;
#pragma unroll
    for (int k = 0; k < HEAD_MAXV; ++k) {
      const int c = lane + 32 * k;
      va[k] = c < C ? (double)a[c] : 0.0;
      vb[k] = c < C ? (double)b[c] : 0.0;
      sa += va[k] * va[k];
      sb += vb[k] * vb[k];
    }
    sa = warp_sum_f64(sa);
    sb = warp_sum_f64(sb);
    const double ra = 1.0 / (sqrt(sa) + 1e-10), rb = 1.0 / (sqrt(sb) + 1e-10);   // normalize_tensor, eps 1e-10
#pragma unroll
    for (int k = 0; k < HEAD_MAXV; ++k) {
      // both products rounded (no FMA contraction of one of them), so that identical features give exactly 0
      const double d = __dmul_rn(va[k], ra) - __dmul_rn(vb[k], rb);
      acc += wl[k] * (d * d);
    }
  }
  acc = warp_sum_f64(acc);
  __shared__ double red[TPB / 32];
  if (lane == 0) red[wid] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < TPB / 32; ++k) acc += red[k];
    atomicAdd(out + p, acc * inv_hw);
  }
}

int grid_for(long long total) {
  return (int)max(1LL, min((total + TPB - 1) / TPB, (long long)(8 * teco_sm_count())));
}
}  // namespace

extern "C" {

int teco_lpips_input_u8(const uint8_t* img, int32_t N, int32_t H, int32_t W, int32_t y0, int32_t x0, int32_t h, int32_t w,
                        float* x, void* stream) {
  TECO_CHECK_ARG(img && x, "teco_lpips_input_u8: NULL tensor");
  TECO_CHECK_ARG(N > 0 && H > 0 && W > 0 && h > 0 && w > 0, "teco_lpips_input_u8: bad size N=%d %dx%d window %dx%d", N, H, W,
                 h, w);
  TECO_CHECK_ARG(y0 >= 0 && x0 >= 0 && y0 + h <= H && x0 + w <= W,
                 "teco_lpips_input_u8: window %d+%d x %d+%d does not fit a %dx%d frame", y0, h, x0, w, H, W);
  const long long total = (long long)N * h * w * 3;
  lpips_input_kernel<<<grid_for(total), TPB, 0, (cudaStream_t)stream>>>(img, H, W, y0, x0, h, w, total, x);
  TECO_CUDA_LAUNCH_CHECK("teco_lpips_input_u8");
  return TECO_OK;
}

int teco_maxpool3s2_f32(const float* x, float* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream) {
  TECO_CHECK_ARG(x && y, "teco_maxpool3s2_f32: NULL tensor");
  TECO_CHECK_ARG(N > 0 && C > 0 && H >= 3 && W >= 3, "teco_maxpool3s2_f32: a %dx%d input (N=%d C=%d) is smaller than the 3x3 window",
                 H, W, N, C);
  const int OH = (H - 3) / 2 + 1, OW = (W - 3) / 2 + 1;
  const long long total = (long long)N * OH * OW * C;
  maxpool3s2_kernel<<<grid_for(total), TPB, 0, (cudaStream_t)stream>>>(x, y, H, W, C, OH, OW, total);
  TECO_CUDA_LAUNCH_CHECK("teco_maxpool3s2_f32");
  return TECO_OK;
}

int teco_lpips_head_f32(const float* fa, int32_t Na, const float* fb, int32_t Nb, const int32_t* ia_host,
                        const int32_t* ib_host, int32_t P, int32_t H, int32_t W, int32_t C, const float* lin, double* out,
                        void* stream) {
  TECO_CHECK_ARG(fa && fb && lin && out && ia_host && ib_host, "teco_lpips_head_f32: NULL argument");
  TECO_CHECK_ARG(P > 0 && P <= HEAD_MAXP, "teco_lpips_head_f32: %d pairs (1..%d per launch)", P, HEAD_MAXP);
  TECO_CHECK_ARG(Na > 0 && Nb > 0 && H > 0 && W > 0 && C > 0 && C <= 32 * HEAD_MAXV,
                 "teco_lpips_head_f32: bad feature shape Na=%d Nb=%d %dx%d C=%d (C <= %d)", Na, Nb, H, W, C, 32 * HEAD_MAXV);
  HeadPairs pr;
  for (int p = 0; p < P; ++p) {
    TECO_CHECK_ARG(ia_host[p] >= 0 && ia_host[p] < Na && ib_host[p] >= 0 && ib_host[p] < Nb,
                   "teco_lpips_head_f32: pair %d = (%d, %d) outside %d x %d frames", p, ia_host[p], ib_host[p], Na, Nb);
    pr.a[p] = ia_host[p];
    pr.b[p] = ib_host[p];
  }
  const int HW = H * W;
  const int want = (HW + 8 * (TPB / 32) - 1) / (8 * (TPB / 32));          // about 8 pixels per warp
  const int bx = max(1, min(want, max(1, 4 * teco_sm_count() / P)));
  lpips_head_kernel<<<dim3(bx, P), TPB, 0, (cudaStream_t)stream>>>(fa, fb, pr, HW, C, lin, out, 1.0 / (double)HW);
  TECO_CUDA_LAUNCH_CHECK("teco_lpips_head_f32");
  return TECO_OK;
}

}  // extern "C"
