// Shared helpers for libteco.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/teco.h"

void teco_set_error(const char* fmt, ...);

#define TECO_CHECK_ARG(cond, ...)                 \
  do {                                            \
    if (!(cond)) {                                \
      teco_set_error(__VA_ARGS__);                \
      return TECO_E_INVALID;                      \
    }                                             \
  } while (0)

#define TECO_CUDA_LAUNCH_CHECK(name)                                              \
  do {                                                                            \
    cudaError_t e__ = cudaGetLastError();                                         \
    if (e__ != cudaSuccess) {                                                     \
      teco_set_error("%s: CUDA launch failed: %s", name, cudaGetErrorString(e__)); \
      return TECO_E_CUDA;                                                         \
    }                                                                             \
  } while (0)

#define TECO_CUDA_CALL(expr)                                                       \
  do {                                                                             \
    cudaError_t e__ = (expr);                                                      \
    if (e__ != cudaSuccess) {                                                      \
      teco_set_error("%s failed: %s", #expr, cudaGetErrorString(e__));             \
      return TECO_E_CUDA;                                                          \
    }                                                                              \
  } while (0)

static inline int teco_ceil_div(long long a, long long b) { return (int)((a + b - 1) / b); }

__device__ __forceinline__ float teco_act(float v, int act) {
  switch (act) {
    case TECO_ACT_RELU: return fmaxf(v, 0.f);
    case TECO_ACT_LRELU02: return v >= 0.f ? v : 0.2f * v;
    case TECO_ACT_TANH24: return tanhf(v) * 24.0f;
    case TECO_ACT_SIGMOID: return 1.0f / (1.0f + expf(-v));
    default: return v;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum for blockDim.x <= 1024 (multiple of 32); result valid in thread 0.
__device__ __forceinline__ float block_sum(float v, float* smem32) {
  v = warp_sum(v);
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) smem32[wid] = v;
  __syncthreads();
  float r = 0.f;
  if (wid == 0) {
    int nw = (blockDim.x + 31) >> 5;
    r = lane < nw ? smem32[lane] : 0.f;
    r = warp_sum(r);
  }
  __syncthreads();
  return r;
}

// Exclusive scan of one int per thread over a CTA of NT threads (multiple of 32); returns the prefix, *total the sum.
// Every thread of the CTA must call it.
template <int NT>
__device__ __forceinline__ int cta_exclusive_scan(int v, int* sm /* NT/32 + 1 ints */, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) sm[wid] = x;
  __syncthreads();
  if (wid == 0) {
    int w = lane < NT / 32 ? sm[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      int y = __shfl_up_sync(0xffffffffu, w, d);
      if (lane >= d) w += y;
    }
    if (lane < NT / 32) sm[lane] = w;
  }
  __syncthreads();
  const int before = (wid > 0 ? sm[wid - 1] : 0) + x - v;
  *total = sm[NT / 32 - 1];
  __syncthreads();
  return before;
}

int teco_sm_count();
// out[e] (+)= part[0][e] + ... + part[S-1][e] for e < E, summed in split order (eltwise.cu).  S >= 1.
int teco_reduce_splits(const float* part, int S, long long E, float* out, int accumulate, cudaStream_t stream);
