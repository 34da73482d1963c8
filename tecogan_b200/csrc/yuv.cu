// `main.py --input_y4m / --output_y4m`: the 4:2:0 colour conversions of YUV4MPEG2 streams, byte for byte with cv2 4.13's
// cvtColor(COLOR_RGB2YUV_I420) and cvtColor(COLOR_YUV2RGB_I420) (DESIGN.md section 4.12; tests/golden/yuv_oracle.py
// restates both).  BT.601 limited range in 20-bit fixed point, integer arithmetic throughout:
//   RGB -> I420  Y = (269484 R + 528482 G + 102760 B + HALF + (16 << 20)) >> 20 per pixel; U and V from the top-left pixel
//                of each 2 x 2 block (cv2 does not average the block).
//   I420 -> RGB  y = max(0, Y - 16) * 1220542, u = U - 128, v = V - 128 of the pixel's block;
//                R = sat8((y + HALF + 1673527 v) >> 20), G = sat8((y + HALF - 852492 v - 409993 u) >> 20),
//                B = sat8((y + HALF + 2116026 u) >> 20).
// An I420 frame is [3H/2, W] uint8: the Y plane, then U (H/2 x W/2), then V, each packed -- a Y4M frame's payload.
//
// Both kernels give each thread a strip of two rows by kStrip = 8 columns (one row of 2 x 2 chroma blocks, four wide), so
// the chroma of a block comes from pixels the thread already holds.  When W % 8 == 0 and the buffers are aligned, the
// strip is moved with 4- and 8-byte loads and stores; otherwise byte by byte.  The strips are taken grid-stride.
#include "teco_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kStrip = 8;                // columns per thread: 8 Y bytes per row, 4 U and 4 V bytes
constexpr int kS = 20;
constexpr int kHalf = 1 << (kS - 1);
constexpr int kMaxSide = 65534;

__device__ __forceinline__ int sat8(int v) { return v < 0 ? 0 : (v > 255 ? 255 : v); }

__device__ __forceinline__ uint32_t luma(int r, int g, int b) {
  return (uint32_t)((269484 * r + 528482 * g + 102760 * b + kHalf + (16 << kS)) >> kS);
}
__device__ __forceinline__ uint32_t chroma_u(int r, int g, int b) {
  return (uint32_t)((-155188 * r - 305135 * g + 460324 * b + kHalf + (128 << kS)) >> kS);
}
__device__ __forceinline__ uint32_t chroma_v(int r, int g, int b) {
  return (uint32_t)((460324 * r - 385875 * g - 74448 * b + kHalf + (128 << kS)) >> kS);
}

// src [H, W, 3] RGB rows every `pitch` bytes -> dst [3H/2, W] I420.  Item i is strip i % strips of row pair i / strips.
// kVec: W % 8 == 0, src and pitch 4-byte aligned, dst 8-byte aligned -- every strip is full and its moves are vectors.
template <bool kVec>
__global__ void __launch_bounds__(kThreads) rgb_to_i420_kernel(const uint8_t* __restrict__ src, int64_t pitch, int H,
                                                               int W, uint8_t* __restrict__ dst, int strips,
                                                               int64_t total) {
  const int64_t plane = (int64_t)H * W;
  const int cw = W >> 1;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total; i += (int64_t)gridDim.x * kThreads) {
    const int yp = (int)(i / strips), x0 = (int)(i - (int64_t)yp * strips) * kStrip;
    const int nx = kVec ? kStrip : min(kStrip, W - x0);
    const uint8_t* row = src + (int64_t)(2 * yp) * pitch + 3 * (int64_t)x0;
    uint8_t* yout = dst + (int64_t)(2 * yp) * W + x0;
    uint8_t* uout = dst + plane + (int64_t)yp * cw + (x0 >> 1);
    uint8_t* vout = uout + (plane >> 2);
    uint32_t U = 0, V = 0;
#pragma unroll
    for (int r = 0; r < 2; ++r, row += pitch, yout += W) {
      uint32_t px[6];                                      // the strip's 24 bytes of this row, little-endian words
      if (kVec) {
#pragma unroll
        for (int k = 0; k < 6; ++k) px[k] = __ldg(reinterpret_cast<const uint32_t*>(row) + k);
      } else {
#pragma unroll
        for (int k = 0; k < 6; ++k) px[k] = 0;
#pragma unroll
        for (int k = 0; k < 3 * kStrip; ++k)
          if (k < 3 * nx) px[k >> 2] |= (uint32_t)__ldg(row + k) << (8 * (k & 3));
      }
      uint32_t Y[2] = {0, 0};
#pragma unroll
      for (int p = 0; p < kStrip; ++p) {
        const int R = (px[(3 * p) >> 2] >> (8 * ((3 * p) & 3))) & 0xff;
        const int G = (px[(3 * p + 1) >> 2] >> (8 * ((3 * p + 1) & 3))) & 0xff;
        const int B = (px[(3 * p + 2) >> 2] >> (8 * ((3 * p + 2) & 3))) & 0xff;
        Y[p >> 2] |= luma(R, G, B) << (8 * (p & 3));
        if (r == 0 && (p & 1) == 0) {
          U |= chroma_u(R, G, B) << (8 * (p >> 1));
          V |= chroma_v(R, G, B) << (8 * (p >> 1));
        }
      }
      if (kVec) {
        *reinterpret_cast<uint2*>(yout) = make_uint2(Y[0], Y[1]);
      } else {
#pragma unroll
        for (int p = 0; p < kStrip; ++p)
          if (p < nx) yout[p] = (uint8_t)(Y[p >> 2] >> (8 * (p & 3)));
      }
    }
    if (kVec) {
      *reinterpret_cast<uint32_t*>(uout) = U;
      *reinterpret_cast<uint32_t*>(vout) = V;
    } else {
#pragma unroll
      for (int b = 0; b < kStrip / 2; ++b)
        if (2 * b < nx) {
          uout[b] = (uint8_t)(U >> (8 * b));
          vout[b] = (uint8_t)(V >> (8 * b));
        }
    }
  }
}

// src N packed I420 frames [N, 3H/2, W] -> dst [N, H, W, 3] RGB.  Item i is strip i % strips of row pair
// (i / strips) % (H / 2) of frame i / (strips * H / 2).  kVec: W % 8 == 0, src and dst 8-byte aligned.
template <bool kVec>
__global__ void __launch_bounds__(kThreads) i420_to_rgb_kernel(const uint8_t* __restrict__ src, int H, int W,
                                                               uint8_t* __restrict__ dst, int strips, int64_t total) {
  const int64_t plane = (int64_t)H * W;
  const int cw = W >> 1, pairs = H >> 1;
  for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < total; i += (int64_t)gridDim.x * kThreads) {
    const int64_t rp = i / strips;                         // row pair over all frames
    const int x0 = (int)(i - rp * strips) * kStrip;
    const int64_t n = rp / pairs;
    const int yp = (int)(rp - n * pairs);
    const int nx = kVec ? kStrip : min(kStrip, W - x0);
    const uint8_t* frame = src + n * (plane + (plane >> 1));
    const uint8_t* yin = frame + (int64_t)(2 * yp) * W + x0;
    const uint8_t* uin = frame + plane + (int64_t)yp * cw + (x0 >> 1);
    const uint8_t* vin = uin + (plane >> 2);
    uint8_t* out = dst + ((n * H + 2 * yp) * W + x0) * 3;
    uint32_t U = 0, V = 0;
    if (kVec) {
      U = __ldg(reinterpret_cast<const uint32_t*>(uin));
      V = __ldg(reinterpret_cast<const uint32_t*>(vin));
    } else {
#pragma unroll
      for (int b = 0; b < kStrip / 2; ++b)
        if (2 * b < nx) {
          U |= (uint32_t)__ldg(uin + b) << (8 * b);
          V |= (uint32_t)__ldg(vin + b) << (8 * b);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r, yin += W, out += 3 * (int64_t)W) {
      uint32_t Y[2] = {0, 0};
      if (kVec) {
        const uint2 y2 = __ldg(reinterpret_cast<const uint2*>(yin));
        Y[0] = y2.x;
        Y[1] = y2.y;
      } else {
#pragma unroll
        for (int p = 0; p < kStrip; ++p)
          if (p < nx) Y[p >> 2] |= (uint32_t)__ldg(yin + p) << (8 * (p & 3));
      }
      uint32_t px[6] = {0, 0, 0, 0, 0, 0};
#pragma unroll
      for (int p = 0; p < kStrip; ++p) {
        const int yv = (int)((Y[p >> 2] >> (8 * (p & 3))) & 0xff) - 16;
        const int y = (yv < 0 ? 0 : yv) * 1220542 + kHalf;
        const int u = (int)((U >> (8 * (p >> 1))) & 0xff) - 128, v = (int)((V >> (8 * (p >> 1))) & 0xff) - 128;
        const uint32_t R = sat8((y + 1673527 * v) >> kS);
        const uint32_t G = sat8((y - 852492 * v - 409993 * u) >> kS);
        const uint32_t B = sat8((y + 2116026 * u) >> kS);
        px[(3 * p) >> 2] |= R << (8 * ((3 * p) & 3));
        px[(3 * p + 1) >> 2] |= G << (8 * ((3 * p + 1) & 3));
        px[(3 * p + 2) >> 2] |= B << (8 * ((3 * p + 2) & 3));
      }
      if (kVec) {
#pragma unroll
        for (int k = 0; k < 3; ++k) reinterpret_cast<uint2*>(out)[k] = make_uint2(px[2 * k], px[2 * k + 1]);
      } else {
#pragma unroll
        for (int k = 0; k < 3 * kStrip; ++k)
          if (k < 3 * nx) out[k] = (uint8_t)(px[k >> 2] >> (8 * (k & 3)));
      }
    }
  }
}

bool aligned(const void* p, int64_t a) { return ((uintptr_t)p % (uintptr_t)a) == 0; }

// Persistent grid: as many CTAs as fit on the device at once, fewer for a small frame.
template <typename Kernel>
int grid_for(Kernel kernel, int64_t total, int* per_sm) {
  if (*per_sm == 0 && cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kernel, kThreads, 0) != cudaSuccess)
    *per_sm = 1;
  const int64_t need = (total + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)(*per_sm > 0 ? *per_sm : 1) * teco_sm_count();
  return (int)(need < cap ? need : cap);
}

}  // namespace

extern "C" int teco_rgb_to_i420_u8(const uint8_t* src, int64_t src_pitch, int32_t H, int32_t W, uint8_t* dst,
                                   void* stream) {
  TECO_CHECK_ARG(src && dst, "teco_rgb_to_i420_u8: NULL pointer");
  TECO_CHECK_ARG(H >= 2 && W >= 2 && H <= kMaxSide && W <= kMaxSide && H % 2 == 0 && W % 2 == 0,
                 "teco_rgb_to_i420_u8: sides must be even and 2..65534 (got %dx%d)", H, W);
  TECO_CHECK_ARG(src_pitch >= 3 * (int64_t)W, "teco_rgb_to_i420_u8: row pitch %lld below 3 * width %d",
                 (long long)src_pitch, W);
  const int strips = teco_ceil_div(W, kStrip);
  const int64_t total = (int64_t)(H / 2) * strips;
  const bool vec = W % kStrip == 0 && aligned(src, 4) && src_pitch % 4 == 0 && aligned(dst, 8);
  static int per_sm[2] = {0, 0};
  cudaStream_t s = (cudaStream_t)stream;
  if (vec) {
    rgb_to_i420_kernel<true><<<grid_for(rgb_to_i420_kernel<true>, total, &per_sm[1]), kThreads, 0, s>>>(
        src, src_pitch, H, W, dst, strips, total);
  } else {
    rgb_to_i420_kernel<false><<<grid_for(rgb_to_i420_kernel<false>, total, &per_sm[0]), kThreads, 0, s>>>(
        src, src_pitch, H, W, dst, strips, total);
  }
  TECO_CUDA_LAUNCH_CHECK("teco_rgb_to_i420_u8");
  return TECO_OK;
}

extern "C" int teco_i420_to_rgb_u8(const uint8_t* src, int32_t N, int32_t H, int32_t W, uint8_t* dst, void* stream) {
  TECO_CHECK_ARG(src && dst, "teco_i420_to_rgb_u8: NULL pointer");
  TECO_CHECK_ARG(N >= 1, "teco_i420_to_rgb_u8: need N >= 1 frames (got %d)", N);
  TECO_CHECK_ARG(H >= 2 && W >= 2 && H <= kMaxSide && W <= kMaxSide && H % 2 == 0 && W % 2 == 0,
                 "teco_i420_to_rgb_u8: sides must be even and 2..65534 (got %dx%d)", H, W);
  const int strips = teco_ceil_div(W, kStrip);
  const int64_t total = (int64_t)N * (H / 2) * strips;
  const bool vec = W % kStrip == 0 && aligned(src, 8) && aligned(dst, 8);
  static int per_sm[2] = {0, 0};
  cudaStream_t s = (cudaStream_t)stream;
  if (vec) {
    i420_to_rgb_kernel<true><<<grid_for(i420_to_rgb_kernel<true>, total, &per_sm[1]), kThreads, 0, s>>>(
        src, H, W, dst, strips, total);
  } else {
    i420_to_rgb_kernel<false><<<grid_for(i420_to_rgb_kernel<false>, total, &per_sm[0]), kThreads, 0, s>>>(
        src, H, W, dst, strips, total);
  }
  TECO_CUDA_LAUNCH_CHECK("teco_i420_to_rgb_u8");
  return TECO_OK;
}
