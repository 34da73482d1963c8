// Training clips cut from the device-resident frame store (tecogan_b200/lib/dataloader.py::FrameStore): the pixel half of
// HRClipLoader.sample() -- crop, left-right flip, convert_image_dtype -- on the GPU.  The draws (which frames, where, whether
// flipped) are made on the host and arrive as one table row per output frame.
#include "teco_common.cuh"

namespace {

// One block per (output row, output frame).  Row y of output frame n reads S pixels of one source row, mirrored when
// flip != 0, and writes them as 3*S contiguous floats.  __fdiv_rn: the correctly rounded quotient, which is what numpy's
// float32 division of the host path computes, whatever -use_fast_math or -prec-div say.
__global__ void gather_clips_u8_kernel(const uint8_t* __restrict__ store, const int64_t* __restrict__ table, int S,
                                       float* __restrict__ out) {
  const int y = blockIdx.x, n = blockIdx.y;
  const int64_t src0 = table[3 * n + 0], pitch = table[3 * n + 1];
  const bool flip = table[3 * n + 2] != 0;
  const uint8_t* row = store + src0 + (int64_t)y * pitch;
  float* dst = out + ((int64_t)n * S + y) * (int64_t)S * 3;
  for (int e = threadIdx.x; e < 3 * S; e += blockDim.x) {
    const int x = e / 3, c = e - 3 * x;
    const int sx = flip ? S - 1 - x : x;
    dst[e] = __fdiv_rn((float)row[3 * sx + c], 255.0f);
  }
}

}  // namespace

extern "C" int teco_gather_clips_u8(const uint8_t* store, const int64_t* table, int32_t n, int32_t S, float* out,
                                    void* stream) {
  TECO_CHECK_ARG(store && table && out, "teco_gather_clips_u8: NULL pointer");
  TECO_CHECK_ARG(n > 0 && n <= 65535 && S > 0, "teco_gather_clips_u8: need 0 < n <= 65535 and S > 0 (got n=%d, S=%d)", n, S);
  gather_clips_u8_kernel<<<dim3((unsigned)S, (unsigned)n), 128, 0, (cudaStream_t)stream>>>(store, table, S, out);
  TECO_CUDA_LAUNCH_CHECK("teco_gather_clips_u8");
  return TECO_OK;
}
