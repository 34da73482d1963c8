// `main.py --scene_threshold`: the frame difference behind the scene-cut score (DESIGN.md section 4.13).
//   teco_frame_sad_q8: *out = sum over the n values of |q(a[i]) - q(b[i])|, q(x) = clamp(rint(255 x), 0, 255)
// with 255 x a float32 product rounded half-even to an integer: for a frame decoded from 8-bit pixels (u / 255f) q gives
// the byte back exactly; 16-bit sources divided by 255 may exceed 1, hence the clamp.  The sum is an integer, summed in
// 64 bits: exact, and the same for every grid and launch.
//
// A grid-stride pass over the frame pair: float4 loads when both pointers are 16-byte aligned (the n % 4 tail element by
// element), single floats otherwise.  Each thread sums its elements, each CTA reduces its threads with shuffles and one
// shared-memory step, and one thread per CTA adds the CTA's sum to *out with a 64-bit integer atomicAdd.
//
// `dataPrepare.py --scene_threshold`: the same difference on the 8-bit frames themselves (DESIGN.md section 4.14).
//   teco_frame_sads_u8: out[i] = sum over the frame_bytes bytes of |f_i[j] - f_{i-1}[j]| for n packed frames, f_{-1} =
// prev (out[0] = 0 without it).  For 8-bit frames q(u / 255) = u, so out[i] is teco_frame_sad_q8 of the same frames.
// One launch covers a staging window: blockIdx.y walks the pairs, blockIdx.x strides through a pair's bytes, 16 at a
// time with __vsadu4 when every frame is 16-byte aligned, byte by byte otherwise; one atomicAdd per CTA per pair.
#include "teco_common.cuh"

namespace {

constexpr int kThreads = 256;

// The CTA's sum of every thread's acc, valid in warp 0 (lane 0 is the one that uses it).  `part` is read after the
// __syncthreads here: a caller that calls again must __syncthreads before that.
__device__ __forceinline__ unsigned long long block_sum(unsigned long long acc, unsigned long long* part) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) part[wid] = acc;
  __syncthreads();
  if (wid == 0) {
    acc = lane < kThreads / 32 ? part[lane] : 0ull;
#pragma unroll
    for (int o = kThreads / 64; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  }
  return acc;
}

__device__ __forceinline__ int q8(float x) {
  const int v = __float2int_rn(__fmul_rn(x, 255.0f));    // no contraction: the product is rounded to float32 first
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

__device__ __forceinline__ unsigned int absdiff(float a, float b) {
  const int d = q8(a) - q8(b);
  return (unsigned int)(d < 0 ? -d : d);
}

template <bool kVec>
__global__ void __launch_bounds__(kThreads) frame_sad_q8_kernel(const float* __restrict__ a,
                                                                const float* __restrict__ b, int64_t n,
                                                                unsigned long long* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int64_t first = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  unsigned long long acc = 0;
  int64_t tail = 0;
  if (kVec) {
    const int64_t n4 = n >> 2;
    const float4* a4 = reinterpret_cast<const float4*>(a);
    const float4* b4 = reinterpret_cast<const float4*>(b);
    for (int64_t i = first; i < n4; i += stride) {
      const float4 x = __ldg(a4 + i), y = __ldg(b4 + i);
      acc += absdiff(x.x, y.x) + absdiff(x.y, y.y) + absdiff(x.z, y.z) + absdiff(x.w, y.w);
    }
    tail = n4 << 2;
  }
  for (int64_t i = tail + first; i < n; i += stride) acc += absdiff(__ldg(a + i), __ldg(b + i));

  __shared__ unsigned long long part[kThreads / 32];
  acc = block_sum(acc, part);
  if (threadIdx.x == 0 && acc != 0) atomicAdd(out, acc);
}

// Pair p = blockIdx.y, blockIdx.y + gridDim.y, ...: frames p - 1 (prev for p = 0) and p.  A pair without a first frame
// (p = 0, prev NULL) is skipped by the whole CTA, so every thread reaches block_sum's barrier.
template <bool kVec>
__global__ void __launch_bounds__(kThreads) frame_sads_u8_kernel(const uint8_t* __restrict__ frames, int64_t frame_bytes,
                                                                 int32_t n, const uint8_t* __restrict__ prev,
                                                                 unsigned long long* __restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * kThreads;
  const int64_t first = (int64_t)blockIdx.x * kThreads + threadIdx.x;
  __shared__ unsigned long long part[kThreads / 32];
  for (int32_t p = blockIdx.y; p < n; p += gridDim.y) {
    const uint8_t* b = frames + (int64_t)p * frame_bytes;
    const uint8_t* a = p > 0 ? b - frame_bytes : prev;
    if (a == nullptr) continue;
    unsigned long long acc = 0;
    if (kVec) {
      const uint4* a4 = reinterpret_cast<const uint4*>(a);
      const uint4* b4 = reinterpret_cast<const uint4*>(b);
      for (int64_t i = first; i < (frame_bytes >> 4); i += stride) {
        const uint4 x = __ldg(a4 + i), y = __ldg(b4 + i);
        acc += __vsadu4(x.x, y.x) + __vsadu4(x.y, y.y) + __vsadu4(x.z, y.z) + __vsadu4(x.w, y.w);
      }
    } else {
      for (int64_t i = first; i < frame_bytes; i += stride) {
        const int d = (int)__ldg(a + i) - (int)__ldg(b + i);
        acc += (unsigned int)(d < 0 ? -d : d);
      }
    }
    acc = block_sum(acc, part);
    if (threadIdx.x == 0 && acc != 0) atomicAdd(out + p, acc);
    __syncthreads();                                     // part is written again by the next pair
  }
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

int resident_ctas(const void* kernel, int* per_sm) {
  if (*per_sm == 0 && cudaOccupancyMaxActiveBlocksPerMultiprocessor(per_sm, kernel, kThreads, 0) != cudaSuccess)
    *per_sm = 1;
  return (*per_sm > 0 ? *per_sm : 1) * teco_sm_count();
}

// Persistent grid: as many CTAs as fit on the device at once, fewer for a small frame.
template <typename Kernel>
int grid_for(Kernel kernel, int64_t items, int* per_sm) {
  const int64_t need = (items + kThreads - 1) / kThreads;
  const int64_t cap = resident_ctas((const void*)kernel, per_sm);
  return (int)(need < cap ? need : cap);
}

// The window's grid: one row of CTAs per pair (up to 65 535 rows, looped beyond), each row as wide as its share of the
// resident CTAs, at least one and no wider than one pair needs.
template <typename Kernel>
dim3 window_grid(Kernel kernel, int64_t items, int32_t n, int* per_sm) {
  const int rows = n < 65535 ? n : 65535;
  const int64_t need = (items + kThreads - 1) / kThreads;
  int64_t cols = (resident_ctas((const void*)kernel, per_sm) + rows - 1) / rows;
  if (cols > need) cols = need;
  return dim3((unsigned)(cols > 0 ? cols : 1), (unsigned)rows);
}

}  // namespace

extern "C" int teco_frame_sad_q8(const float* a, const float* b, int64_t n, uint64_t* out, void* stream) {
  TECO_CHECK_ARG(a && b && out, "teco_frame_sad_q8: NULL pointer");
  TECO_CHECK_ARG(n >= 0, "teco_frame_sad_q8: n must be >= 0 (got %lld)", (long long)n);
  cudaStream_t s = (cudaStream_t)stream;
  TECO_CUDA_CALL(cudaMemsetAsync(out, 0, sizeof(uint64_t), s));     // this entry zeroes *out: the caller need not
  if (n == 0) return TECO_OK;
  unsigned long long* sum = reinterpret_cast<unsigned long long*>(out);
  static int per_sm[2] = {0, 0};
  if (aligned16(a) && aligned16(b)) {
    const int grid = grid_for(frame_sad_q8_kernel<true>, (n + 3) >> 2, &per_sm[1]);
    frame_sad_q8_kernel<true><<<grid, kThreads, 0, s>>>(a, b, n, sum);
  } else {
    const int grid = grid_for(frame_sad_q8_kernel<false>, n, &per_sm[0]);
    frame_sad_q8_kernel<false><<<grid, kThreads, 0, s>>>(a, b, n, sum);
  }
  TECO_CUDA_LAUNCH_CHECK("teco_frame_sad_q8");
  return TECO_OK;
}

extern "C" int teco_frame_sads_u8(const uint8_t* frames, int64_t frame_bytes, int32_t n, const uint8_t* prev,
                                  uint64_t* out, void* stream) {
  TECO_CHECK_ARG(frames && out, "teco_frame_sads_u8: NULL pointer");
  TECO_CHECK_ARG(n >= 1, "teco_frame_sads_u8: n must be >= 1 (got %d)", n);
  TECO_CHECK_ARG(frame_bytes >= 1 && frame_bytes <= INT64_MAX / n,
                 "teco_frame_sads_u8: frame_bytes must be >= 1 and n * frame_bytes fit in 64 bits (got %lld x %d)",
                 (long long)frame_bytes, n);
  cudaStream_t s = (cudaStream_t)stream;
  TECO_CUDA_CALL(cudaMemsetAsync(out, 0, (size_t)n * sizeof(uint64_t), s));    // this entry zeroes out[0..n) itself
  if (n == 1 && prev == nullptr) return TECO_OK;
  unsigned long long* sums = reinterpret_cast<unsigned long long*>(out);
  static int per_sm[2] = {0, 0};
  if (aligned16(frames) && (prev == nullptr || aligned16(prev)) && frame_bytes % 16 == 0) {
    const dim3 grid = window_grid(frame_sads_u8_kernel<true>, frame_bytes >> 4, n, &per_sm[1]);
    frame_sads_u8_kernel<true><<<grid, kThreads, 0, s>>>(frames, frame_bytes, n, prev, sums);
  } else {
    const dim3 grid = window_grid(frame_sads_u8_kernel<false>, frame_bytes, n, &per_sm[0]);
    frame_sads_u8_kernel<false><<<grid, kThreads, 0, s>>>(frames, frame_bytes, n, prev, sums);
  }
  TECO_CUDA_LAUNCH_CHECK("teco_frame_sads_u8");
  return TECO_OK;
}
