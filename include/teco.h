/*
 * teco.h -- C ABI of libteco.so: hand-written sm_90a kernels for the TecoGAN recurrent
 * video-SR hot path (SURVEY.md section 8).  Plain pointers and sizes only; no torch types.
 *
 * The reference (thunil/TecoGAN) has no FFI layer: its "operator API" is Python functions
 * that build TensorFlow graph ops.  Each entry point below names the reference call site
 * (file:line in the reference repository) whose TensorFlow/cuDNN arithmetic it replaces; the Python
 * mirror in tecogan_b200/lib/{ops,frvsr,Teco}.py keeps the reference's function names and
 * binds these symbols through ctypes (see INTEGRATION.md).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless the name ends in _host;
 *  - activations are NHWC, contiguous, with an explicit channel pitch where stated;
 *  - weights use the TensorFlow layouts (conv: [kh,kw,Cin,Cout]; conv_transpose: [kh,kw,Cout,Cin]);
 *  - `stream` is a cudaStream_t passed as void*; all work is stream-ordered, nothing allocates;
 *  - return 0 on success, a negative TECO_E_* code on failure; teco_last_error() gives the
 *    thread-local message.  No exceptions cross the ABI.  There is no CPU fallback.
 */
#ifndef TECO_H_
#define TECO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TECO_OK 0
#define TECO_E_INVALID (-1)   /* bad shape / argument            -> Python ValueError   */
#define TECO_E_CUDA (-2)      /* CUDA runtime / driver error     -> Python RuntimeError */
#define TECO_E_UNSUPPORTED (-3)

/* epilogue activations (reference: tf.nn.relu lib/frvsr.py:53; lrelu lib/ops.py:84-85 with
 * alpha 0.2 lib/frvsr.py:8; tanh*24 lib/frvsr.py:39; sigmoid lib/Teco.py:72) */
enum { TECO_ACT_NONE = 0, TECO_ACT_RELU = 1, TECO_ACT_LRELU02 = 2, TECO_ACT_TANH24 = 3, TECO_ACT_SIGMOID = 4 };

const char* teco_last_error(void);
int teco_version(void);
/* Fills props[0..7] = {sm_count, cc_major, cc_minor, max_smem_optin, l2_bytes, 0,0,0}. */
int teco_device_props(int device, int64_t* props);
/* Host utility: CRC32C (Castagnoli) of n bytes continuing from crc (0 to start); returns the CRC in [0, 2^32) or a negative
   TECO_E_* code.  Used by tecogan_b200/tf_bundle.py to verify TensorFlow checkpoint blocks and tensors (the reference gets
   this from tf.train.Saver, main.py:224,245,307). */
int64_t teco_crc32c(const void* data, int64_t n, int64_t crc);

/* ---------------------------------------------------------------------------------------
 * fp32 direct convolution (exact-parity path; also dgrad via flipped weights).
 * Replaces slim.conv2d behind conv2() lib/ops.py:47-56 and, phase by phase, slim.conv2d_transpose
 * behind conv2_tran() lib/ops.py:35-44.
 *   y[n, oy*out_sy+out_oy, ox*out_sx+out_ox, co] =
 *       post_scale * ( act( bias[co] + sum_{ky,kx,ci} x[n, oy*stride-pad_t+ky, ox*stride-pad_l+kx, ci]
 *                                                    * w[ky,kx,ci,co] ) + res[same position] ) + post_shift
 * out-of-range taps read zero (TF 'SAME').  bias / res may be NULL.
 * ------------------------------------------------------------------------------------- */
typedef struct teco_conv_desc {
  int32_t N, H, W, Cin;          /* input tensor; in_cpitch >= Cin is its channel pitch      */
  int32_t OH, OW, Cout;          /* logical output grid computed by this launch               */
  int32_t KH, KW, stride, pad_t, pad_l;
  int32_t out_H, out_W;          /* physical output tensor (y and res) spatial dims           */
  int32_t out_sy, out_oy, out_sx, out_ox;
  int32_t in_cpitch, out_cpitch; /* channel pitch (elements) of x and of y/res                */
  int32_t act;
  float post_scale, post_shift;
} teco_conv_desc;

int teco_conv2d_f32(const teco_conv_desc* d, const float* x, const float* w, const float* bias,
                    const float* res, float* y, void* stream);

/* Weight gradient of the same convolution: dw[ky,kx,ci,co] (+)= sum x(...) * dy(...), and
 * optionally db[co] (+)= sum dy.  dy is addressed like y above.  accumulate!=0 adds into dw/db. */
int teco_conv2d_wgrad_f32(const teco_conv_desc* d, const float* x, const float* dy, float* dw, float* db,
                          int accumulate, void* stream);

/* ---------------------------------------------------------------------------------------
 * bf16 tensor-core convolution (wgmma m64nNk16, fp32 accumulation in registers).
 * 3x3, stride 1, SAME: the generator / FNet layers (lib/frvsr.py:5-41, 50-63, 79-80).
 * x: NHWC bf16 with Cin (multiple of 16); y: NHWC bf16 with Cout channels.
 * wpk: weights pre-packed by teco_pack_conv3x3_bf16 (K-major SWIZZLE_128B core matrices).
 * res (bf16, optional) is added after the activation; out_f32 (optional, [N,H,W,out_f32_c])
 * receives post_scale*(value + res_f32) + post_shift for the first out_f32_c channels
 * (used by the generator's output stage: + bicubic, *2-1  lib/frvsr.py:85-87).
 * mode 1 (the transposed convolution, y [N,2H,2W,Cout]) takes Cin 64, Cout a multiple of 64 and a bf16 y, with no res
 * and no out_f32; any other mode-1 launch returns TECO_E_INVALID.
 * ------------------------------------------------------------------------------------- */
typedef struct teco_tc_desc {
  int32_t N, H, W, Cin, Cout;    /* Cin, Cout: padded channel counts (multiples of 16)       */
  int32_t act;
  int32_t mode;                  /* 0: conv3x3 s1 SAME; 1: conv_transpose 3x3 s2 SAME (4 phases) */
  int32_t out_f32_c;             /* >0: also/only write fp32 output with this many channels  */
  float post_scale, post_shift;
  int32_t k_live;                /* 1, 2, 4 (Cin 64): input channels from 16*k_live on are zero, their K-steps may be
                                    skipped (same outputs); 0: all                              */
  int32_t pool;                  /* 1: y is [N,H/2,W/2,Cout], the 2x2 max of the bf16 outputs (teco_maxpool2_bf16's
                                    result; mode 0, Cin 64, Cout % 64 == 0, no residual / fp32 output) */
} teco_tc_desc;

/* transpose_layout bit 0: w is [3,3,cout,cin] (conv_transpose layout); bit 1: taps flipped (ky,kx) -> (2-ky,2-kx).
 * Value 3 with (cin, cout) = (Cout, Cin) of a forward conv packs its input-gradient convolution. */
int teco_pack_conv3x3_bf16(const float* w, int32_t cin, int32_t cout, int32_t cin_pad, int32_t cout_pad,
                           int32_t transpose_layout, const int32_t* cin_perm, void* wpk, void* stream);
int64_t teco_packed_weight_bytes(int32_t cin_pad, int32_t cout_pad);
int teco_conv3x3_tc(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias,
                    const void* res, void* y, const float* res_f32, float* out_f32, void* stream);
/* The same 3x3 SAME convolution (mode 0, bf16 output, no residual) tiled over 128 output pixels in flat N*H*W order, so a
 * tile spans several images: for images smaller than teco_conv3x3_tc's 16 x 8 tile (FNet's 8x8 and 4x4 levels).
 * Cin and Cout multiples of 64 in [64,512]; d->mode and d->out_f32_c must be 0.  Bit-identical to teco_conv3x3_tc. */
int teco_conv3x3_im2col_tc(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias, void* y, void* stream);
/* The fp32 output stage of teco_conv3x3_tc (the generator's 64 -> 3 output conv, FNet's 64 -> 2 flow head) on a pipelined
 * kernel: the same arguments, the same MMAs and epilogue, bit-identical outputs.  Takes mode 0, Cin 64, Cout 16 (the
 * packed slice), out_f32_c 2 or 3 with W*out_f32_c*4 a multiple of 16 bytes, optional res_f32, any activation and post
 * transform; res and y must be NULL, and out_f32 / res_f32 16-byte aligned.  Anything else -> TECO_E_INVALID. */
int teco_conv3x3_f32out_tc(const teco_tc_desc* d, const void* x, const void* wpk, const float* bias,
                           const void* res, void* y, const float* res_f32, float* out_f32, void* stream);

/* conv2() 4x4 stride 2 SAME (discriminator_F's disblocks, reference lib/Teco.py:35-41,54-67) on the tensor cores, through
 * its space-to-depth-2 form.  On even H, W TF pads one row / column before, so with xs = space-to-depth-2 of x
 * [N,H/2,W/2,4*Cin], channel (py*2 + px)*Cin + ci = x[2i + py, 2j + px, ci], the convolution is the 3x3 stride-1 SAME one
 *   y = conv3x3(xs, W'),  W'[ty][tx][(py*2 + px)*Cin + ci][co] = w[2ty + py - 1][2tx + px - 1][ci][co]
 * (zero where a kernel index leaves 0..3: 16 of the 36 (tap, phase) slots are live).  Its input gradient is
 * dxs = conv3x3(dz, W'') with W'' the flipped-tap transpose of W', and dx = depth-to-space-2(dxs); its weight gradient is
 * teco_conv3x3_wgrad_tc(xs, dz) at the 16 live slots.  H and W even, Cin 64 or 128, Cout a multiple of 64 in [64,512];
 * anything else -> TECO_E_INVALID.  Maps smaller than a 16 x 8 tile run on teco_conv3x3_im2col_tc's kernel.
 * teco_pack_conv4x4s2_bf16: w [4,4,Cin,Cout] fp32 -> W' packed as teco_pack_conv3x3_bf16 packs a [3,3,4Cin,Cout] weight
 *   (dgrad 0, 36*Cin*Cout bf16), or W'' as its flag 3 packs W' (dgrad 1, same size).
 * teco_conv4x4s2_tc: xs bf16 [N,H/2,W/2,4Cin] -> y bf16 [N,H/2,W/2,Cout] = act(conv(x, w) + bias); bias may be NULL.
 * teco_conv4x4s2_dgrad_tc: dz bf16 [N,H/2,W/2,Cout] -> dxs bf16 [N,H/2,W/2,4Cin].  H, W: the full-resolution input size. */
int teco_pack_conv4x4s2_bf16(const float* w, int32_t cin, int32_t cout, int32_t dgrad, void* wpk, void* stream);
int teco_conv4x4s2_tc(int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, int32_t act, const void* xs,
                      const void* wpk, const float* bias, void* y, void* stream);
int teco_conv4x4s2_dgrad_tc(int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t Cout, const void* dz, const void* wpk_t,
                            void* dxs, void* stream);
/* The conversions around it: x fp32 [N,H,W,C] -> xs bf16 [N,H/2,W/2,4C] (space-to-depth-2 as above), and
 * dxs bf16 [N,H/2,W/2,4C] -> dx fp32 [N,H,W,C] (its inverse).  H, W even, C % 4 == 0, 16-byte aligned tensors. */
int teco_f32_to_bf16_s2d2(const float* x, void* xs, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
int teco_bf16_d2s2_to_f32(const void* dxs, float* dx, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);

/* Bias gradient of conv2() (slim.conv2d biases, reference lib/ops.py:47-56): db[c] (+)= sum over npix pixels of dy[pixel*cpitch + c]. */
int teco_bias_grad_f32(const float* dy, float* db, int64_t npix, int32_t C, int32_t cpitch, int32_t accumulate, void* stream);

/* Weight gradient of conv2() 3x3 stride 1 SAME on the tensor cores (the gradient tf.train.AdamOptimizer.compute_gradients takes
 * through slim.conv2d: reference lib/ops.py:47-56, lib/Teco.py:426,446-447):
 *   dw[ky][kx][ci][co] (+)= sum_p x[p + (ky-1,kx-1)][ci] * dz[p][co],  dw fp32 in TF layout [3,3,cin,cout].
 * x [N,H,W,cin_pad], dz [N,H,W,cout_pad]: NHWC bf16, channel counts padded to multiples of 64; cout % 4 == 0.
 * accumulate == 0 zeroes dw first (pixel tiles are summed with fp32 atomics). */
int teco_conv3x3_wgrad_tc(int32_t N, int32_t H, int32_t W, int32_t cin_pad, int32_t cout_pad, int32_t cin, int32_t cout,
                          const void* x, const void* dz, float* dw, int32_t accumulate, void* stream);

/* Multi-layer 3x3 64->64 chain on 32x32 images (the metric configuration's LR clips) in ONE launch whose activations
 * stay in shared memory: a cluster of two CTAs owns each image through all layers.  The plan has the shape of
 * generator_F's input conv + residual blocks (reference lib/frvsr.py:59-70): conv2(3x3, 64->64) + bias + ReLU /
 * LeakyReLU / none + optional in-place residual per layer.  The results are bit-identical to one teco_conv3x3_tc launch
 * per layer.
 * x_in / buf_a / buf_b: NHWC bf16 [N,32,32,64] (buffer ids 0 / 1 / 2; x_in is never written).
 * plan_host: HOST array [num_layers][4] = {input buffer id, output buffer id, residual buffer id or -1, TECO_ACT_*}.
 * wpk_all: num_layers packed layers back to back (teco_pack_conv3x3_bf16, 64x64 -> 73728 bytes each); bias_all [num_layers][64].
 * teco_conv3x3_lin_in_smem: 1 for exactly the shapes and plans teco_conv3x3_lin_tc takes -- N > 0; H == W == 32; 1..40
 *   layers; layer 0 is {0, 1, -1, act}; layer l >= 1 reads layer l-1's output and writes the other of buffers 1 and 2,
 *   with no residual or an in-place one on a buffer an earlier layer wrote; act is none, ReLU or LeakyReLU.  Host-only,
 *   needs no device.  teco_conv3x3_lin_tc returns TECO_E_INVALID for anything else. */
int teco_conv3x3_lin_tc(int32_t N, int32_t H, int32_t W, int32_t num_layers, const void* x_in, void* buf_a, void* buf_b,
                        const void* wpk_all, const float* bias_all, const int32_t* plan_host, void* stream);
int teco_conv3x3_lin_in_smem(int32_t N, int32_t H, int32_t W, int32_t num_layers, const int32_t* plan_host);
/* Clusters of the one-launch kernel resident at once on the current device (its persistent grid), or a TECO_E_* error. */
int teco_conv3x3_lin_clusters(void);

/* ---------------------------------------------------------------------------------------
 * Warp / resample family (HBM-bound).
 * ------------------------------------------------------------------------------------- */
/* tf.contrib.image.dense_image_warp (lib/Teco.py:120,140,224,254; main.py:215):
 * out[n,y,x,c] = bilinear(img[n], (y - flow[n,y,x,0], x - flow[n,y,x,1])), border clamped. */
int teco_warp_f32(const float* img, const float* flow, float* out, int32_t N, int32_t H, int32_t W, int32_t C,
                  void* stream);
/* gradients of the above: dimg (+)= scatter, dflow = d/dflow (zero where alpha is clipped). */
int teco_warp_bwd_f32(const float* img, const float* flow, const float* dout, float* dimg, float* dflow,
                      int32_t N, int32_t H, int32_t W, int32_t C, void* stream);

/* Fused previous-HR feedback of the recurrence (main.py:201,209-216; lib/Teco.py:113,138-150):
 *   flow_hr = upscale_four(4 * pad_symmetric(flow_lr))        lib/ops.py:126-163, main.py:212-213
 *   warped  = dense_image_warp(pre_gen, flow_hr)              main.py:215
 *   dst[n,y,x, ch_off + (dy*4+dx)*3 + c] = warped[n,4y+dy,4x+dx,c] * in_scale + in_shift   (space-to-depth 4)
 * pre_gen: [N,4h,4w,3] fp32.  flow_lr: [N,fh,fw,2] fp32 with fh<=h, fw<=w (symmetric-padded to h,w).
 * dst: [N,h,w,dst_cpitch] fp32 (dst_bf16==0) or bf16 (dst_bf16!=0).  warped_out (optional): fp32 [N,4h,4w,3].
 * A bf16 dst needs ch_off and dst_cpitch multiples of 8, a 16-byte-aligned dst and no warped_out (else TECO_E_INVALID). */
int teco_warp_s2d_fused(const float* pre_gen, const float* flow_lr, void* dst, float* warped_out,
                        int32_t N, int32_t h, int32_t w, int32_t fh, int32_t fw, int32_t dst_cpitch,
                        int32_t ch_off, int32_t dst_bf16, float in_scale, float in_shift, void* stream);

/* upscale_four lib/ops.py:126-163 (legacy bilinear x4), `scale` multiplies the input (4.0 for flow). */
int teco_upscale4_f32(const float* x, float* y, int32_t N, int32_t h, int32_t w, int32_t C, float scale, void* stream);
/* bicubic_four lib/ops.py:166-212.  x read with channel pitch in_cpitch (first C channels). */
int teco_bicubic4_f32(const float* x, float* y, int32_t N, int32_t h, int32_t w, int32_t C, int32_t in_cpitch,
                      void* stream);
/* tf.image.resize_images legacy bilinear to (oh,ow): lib/frvsr.py:21-22, lib/Teco.py:244. */
int teco_resize_bilinear_f32(const float* x, float* y, int32_t N, int32_t h, int32_t w, int32_t C,
                             int32_t oh, int32_t ow, void* stream);
int teco_resize_bilinear_bwd_f32(const float* dy, float* dx, int32_t N, int32_t h, int32_t w, int32_t C,
                                 int32_t oh, int32_t ow, void* stream);
/* slim.max_pool2d 2x2 s2 VALID, lib/ops.py:92-93 (+ its gradient, routed to the first max). */
int teco_maxpool2_f32(const float* x, float* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
int teco_maxpool2_bwd_f32(const float* x, const float* dy, float* dx, int32_t N, int32_t H, int32_t W, int32_t C,
                          void* stream);
/* bf16 NHWC variants used between tensor-core layers of FNet */
int teco_maxpool2_bf16(const void* x, void* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
int teco_resize2x_bf16(const void* x, void* y, int32_t N, int32_t h, int32_t w, int32_t C, void* stream);
/* tf.space_to_depth(x,4) main.py:201 / lib/Teco.py:145-148 and its inverse (gradient). */
int teco_space_to_depth4_f32(const float* x, float* y, int32_t N, int32_t h, int32_t w, int32_t C,
                             int32_t out_cpitch, int32_t ch_off, void* stream);
int teco_depth_to_space4_f32(const float* y, float* x, int32_t N, int32_t h, int32_t w, int32_t C,
                             int32_t in_cpitch, int32_t ch_off, void* stream);
/* tf_data_gaussDownby4 lib/ops.py:347-367: 9x9 sigma-1.5 Gaussian, stride 4, VALID, per channel. */
int teco_gauss_down4_f32(const float* hr, float* lr, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);

/* Training clips from the device-resident frame store (the pixel half of loadHR, lib/dataloader.py:206-258:
 * random crop, left-right flip, tf.image.convert_image_dtype).  store: uint8 RGB frames back to back.
 * table: n rows of int64 {byte offset of the crop's top-left pixel, row pitch in bytes, flip}.
 *   out[i, y, x, c] = store[table[i][0] + y * table[i][1] + 3 * (flip ? S-1-x : x) + c] / 255   (fp32, correctly rounded)
 * out: [n, S, S, 3] fp32.  The caller keeps every crop inside its frame; 0 < n <= 65535. */
int teco_gather_clips_u8(const uint8_t* store, const int64_t* table, int32_t n, int32_t S, float* out, void* stream);
/* The same output from a store in host memory mapped into the device's address space: store_dev_addr is the device
 * address teco_host_register gave for it.  Each source row is read as the 16-byte-aligned span covering its 3*S bytes,
 * so the mapping must be readable from each row's start rounded down to 16 bytes to its end rounded up (a store in a
 * page-aligned mapping whose size is a multiple of 16 is).  Same table, same limits, bit for bit the same out. */
int teco_gather_clips_host_u8(uint64_t store_dev_addr, const int64_t* table, int32_t n, int32_t S, float* out,
                              void* stream);
/* Host memory for the host-placed frame store: teco_host_register page-locks `bytes` at `host` in place and maps them
 * into every device's address space (cudaHostRegister Mapped | Portable); *dev is the current device's address of
 * `host` (cudaHostGetDevicePointer).  teco_host_unregister undoes it; call it before the memory is unmapped, once no
 * device work reads it any more.  A failure of either leaves no CUDA error behind for later calls to report. */
int teco_host_register(void* host, size_t bytes, void** dev);
int teco_host_unregister(void* host);

/* Inference input (reference lib/dataloader.py:38-43).  frames: device int64 [N], the device address of each of N
 * packed [H, W, 3] RGB frames of uint8 (bits 8) or uint16 (bits 16); 0 < N <= 65535.
 * teco_frames_to_f32:    out [N, H, W, 3] fp32 = frame / 255 (correctly rounded), the LR input.
 * teco_gauss_blur_down4: out [N, ceil(H/4), ceil(W/4), 3] fp32 = cv2.GaussianBlur(frame, (0, 0), sigmaX=1.5)[::4, ::4]
 *   / 255, bit for bit with cv2 4.13's float32 filter (13 taps, BORDER_REFLECT_101; DESIGN.md section 4.9), the LR
 *   input made from HR frames.  2 <= H, W <= 65535: a 1-pixel side -> TECO_E_INVALID. */
int teco_frames_to_f32(const int64_t* frames, int32_t bits, int32_t N, int32_t H, int32_t W, float* out, void* stream);
int teco_gauss_blur_down4(const int64_t* frames, int32_t bits, int32_t N, int32_t H, int32_t W, float* out,
                          void* stream);
/* Training-data preparation (reference dataPrepare.py, lib/data/video.py:168-173).  frames: device int64 [N], the device
 * address of each of N packed [H, W, 3] uint8 frames; 0 < N <= 65535, 2 <= H, W <= 65535 (else TECO_E_INVALID).
 * teco_area_half_u8: out [N, cvRound(H/2), cvRound(W/2), 3] uint8 = cv2.resize(frame, (0, 0), fx=0.5, fy=0.5,
 *   interpolation=INTER_AREA), bit for bit with cv2 4.13 (halves of the sizes round to even; DESIGN.md section 4.10);
 *   swap_rb != 0 stores the channels reversed (BGR in, RGB out). */
int teco_area_half_u8(const int64_t* frames, int32_t N, int32_t H, int32_t W, uint8_t* out, int32_t swap_rb,
                      void* stream);
/* Output resize of `main.py --outscale` (DESIGN.md section 4.11).  dst [H_out, W_out, 3] uint8 = cv2.resize(src,
 * (W_out, H_out), interpolation=INTER_LANCZOS4), bit for bit with cv2 4.13's fixed-point path, for a uint8 RGB src
 * [H_in, W_in, 3].  Rows start every src_pitch / dst_pitch bytes (>= 3 * width).  xtab int32 [W_out, 9] and ytab int32
 * [H_out, 9] are the host-computed axis tables of tecogan_b200/resize.py: base source index, then the eight int16
 * weights.  1 <= sides <= 65535 and at most a 4x down-scale per axis (H_in <= 4 H_out, W_in <= 4 W_out), else
 * TECO_E_INVALID. */
int teco_resize_lanczos4_u8(const uint8_t* src, int64_t src_pitch, int32_t H_in, int32_t W_in, uint8_t* dst,
                            int64_t dst_pitch, int32_t H_out, int32_t W_out, const int32_t* xtab, const int32_t* ytab,
                            void* stream);
/* Colour conversions of `main.py --input_y4m / --output_y4m` (DESIGN.md section 4.12), bit for bit with cv2 4.13's
 * BT.601 limited-range fixed-point cvtColor.  An I420 frame is [3H/2, W] uint8: the Y plane, then U and V at
 * (H/2) x (W/2), each packed.  Sides are even and 2..65534, else TECO_E_INVALID (nothing is launched).
 * teco_rgb_to_i420_u8: dst = cvtColor(src, COLOR_RGB2YUV_I420) for a uint8 RGB src [H, W, 3] whose rows start every
 *   src_pitch (>= 3 * W) bytes; U and V come from the top-left pixel of each 2 x 2 block, as in cv2.
 * teco_i420_to_rgb_u8: dst [N, H, W, 3] uint8 RGB = cvtColor(frame, COLOR_YUV2RGB_I420) of N >= 1 packed I420 frames
 *   src [N, 3H/2, W]. */
int teco_rgb_to_i420_u8(const uint8_t* src, int64_t src_pitch, int32_t H, int32_t W, uint8_t* dst, void* stream);
int teco_i420_to_rgb_u8(const uint8_t* src, int32_t N, int32_t H, int32_t W, uint8_t* dst, void* stream);
/* Frame difference of `main.py --scene_threshold` (DESIGN.md section 4.13): *out = sum over i < n of
 * |q(a[i]) - q(b[i])|, q(x) = clamp(rint(255 x), 0, 255) with 255 x rounded to float32 and then half-even to an integer.
 * Exact 64-bit integer sum, independent of the launch.  The entry zeroes *out on `stream` itself, then adds to it;
 * n == 0 gives 0.  a, b: n float32 values each, any 4-byte alignment (float4 loads when both are 16-byte aligned).
 * NULL pointers or n < 0: TECO_E_INVALID, nothing is enqueued. */
int teco_frame_sad_q8(const float* a, const float* b, int64_t n, uint64_t* out, void* stream);
/* Frame differences of `dataPrepare.py --scene_threshold` (DESIGN.md section 4.14): out[i] = sum over j < frame_bytes of
 * |f_i[j] - f_{i-1}[j]| for the n packed uint8 frames f_i = frames + i * frame_bytes, f_{-1} = prev; out[0] = 0 when
 * prev is NULL.  Exact 64-bit integer sums, independent of the launch, in one launch for all n.  The entry zeroes
 * out[0..n) on `stream` itself, then adds to it.  Any alignment (16-byte loads when frames, prev and frame_bytes are
 * 16-byte aligned).  NULL frames or out, n < 1, frame_bytes < 1 or n * frame_bytes past 64 bits: TECO_E_INVALID,
 * nothing is enqueued. */
int teco_frame_sads_u8(const uint8_t* frames, int64_t frame_bytes, int32_t n, const uint8_t* prev, uint64_t* out,
                       void* stream);

/* generic elementwise y = f(a*x + b) with f in TECO_ACT_*; n elements. preprocess/deprocess lib/ops.py:13-22 */
int teco_affine_act_f32(const float* x, float* y, int64_t n, float a, float b, int32_t act, void* stream);
/* dx = dy * act'(pre) expressed on the activation OUTPUT y (relu/lrelu/tanh24/sigmoid are invertible enough). */
int teco_act_bwd_f32(const float* y, const float* dy, float* dx, int64_t n, int32_t act, void* stream);
/* fp32 <-> bf16 channel-padded copies: dst[n, c_off + c] = src[n, c] for c < C, pixel count npix. */
int teco_f32_to_bf16_pad(const float* src, void* dst, int64_t npix, int32_t C, int32_t src_cpitch,
                         int32_t dst_cpitch, int32_t c_off, float scale, float shift, void* stream);
int teco_bf16_to_f32(const void* src, float* dst, int64_t npix, int32_t C, int32_t src_cpitch, int32_t dst_cpitch,
                     void* stream);
/* dst[p, c] = float(src[p, c]) + (add ? add[p, c] : 0) for c < C; dst/add pitch = dst_cpitch */
int teco_bf16_to_f32_add(const void* src, const float* add, float* dst, int64_t npix, int32_t C, int32_t src_cpitch,
                         int32_t dst_cpitch, void* stream);
/* dst[p, c] = bf16(src[p, c]) for c < C, 0 for C <= c < dst_cpitch (whole padded row written) */
int teco_f32_to_bf16_rowpad(const float* src, void* dst, int64_t npix, int32_t C, int32_t src_cpitch, int32_t dst_cpitch,
                            void* stream);
/* save_img quantisation lib/ops.py:521-523: clip(x*255,0,255) -> uint8 (truncation), RGB order kept. */
int teco_to_u8(const float* x, uint8_t* y, int64_t n, void* stream);
/* deprocess + save_img in one pass (reference lib/ops.py:17-22 and 521-523): y01 = (x + 1) / 2 and y8 = u8(clip(255 * y01)).
   Bit-identical to teco_affine_act_f32(0.5, 0.5) followed by teco_to_u8.  y01 may be NULL (uint8 frame only). */
int teco_deprocess_u8(const float* x, float* y01, uint8_t* y8, int64_t n, void* stream);

/* ---------------------------------------------------------------------------------------
 * Batch-norm of the discriminator (lib/ops.py:88-90; lib/Teco.py:38): batch stats, no gamma, eps 1e-3.
 * stats[0..C) = mean, stats[C..2C) = biased variance (outputs).  lrelu02!=0 fuses LeakyReLU(0.2).
 * ------------------------------------------------------------------------------------- */
int teco_bn_train_f32(const float* x, const float* beta, float* y, float* stats, int64_t npix, int32_t C,
                      float eps, int32_t lrelu02, void* stream);
int teco_bn_train_bwd_f32(const float* x, const float* y, const float* dy, const float* stats, float* dx,
                          float* dbeta, int64_t npix, int32_t C, float eps, int32_t lrelu02, void* stream);

/* ---------------------------------------------------------------------------------------
 * Fixed-order (deterministic) training reductions (main.py --deterministic; DESIGN.md section 4.3).
 * Each *_det call computes what the entry point of the same name without _det computes, but every floating-point sum
 * runs in an order fixed by the call's shapes alone (never by the device, occupancy, stream or timing): reductions split
 * into a partition declared from the shapes, each part stores its partial into the caller's workspace `ws`, and one
 * pass sums the partials in part order.  `ws` is caller-owned, 16-byte aligned and at least the bytes the matching
 * *_plan_bytes call (host only, no device) writes to *ws_bytes_host; a smaller or NULL workspace -> TECO_E_INVALID.
 * accumulate != 0 adds the fixed-order sum to the output's previous value (out + sum), else stores it.
 *  teco_conv3x3_wgrad_tc_det: as teco_conv3x3_wgrad_tc; CTA x runs a fixed run of 8x16 tiles into one accumulator set and
 *    stores it to ws[x][3,3,cin,cout] (fp32); dw = ws[0] + ws[1] + ... in split order.
 *  teco_conv2d_wgrad_f32_det: as teco_conv2d_wgrad_f32 (db may be NULL); pixel splits stored to ws, then db's blocks.
 *  teco_bias_grad_f32_det, teco_bn_train_f32_det, teco_bn_train_bwd_f32_det, teco_loss_*_f32_det: per-block partials,
 *    then one fixed-order sum.  The loss workspace of teco_loss_det_plan_bytes serves all four losses for (npix, C)
 *    (teco_loss_gan_f32_det: npix = n, C = 1).
 *  teco_warp_bwd_f32_det: dimg is STORED (not added to): dimg[q] = sum of q's contributions in ascending source pixel
 *    order (a counting sort of the contributions in ws); dflow as teco_warp_bwd_f32.  4 N H W < 2^31.
 *  teco_resize_bilinear_bwd_f32_det: a gather, no workspace: input pixel (y, x) sums the outputs that read it in
 *    ascending output row, column, then corner order.
 *  teco_sum_ranks_f32: dst[e] = src[0][e] + src[1][e] + ... + src[R-1][e] in rank order (src: [R, n] fp32, gathered
 *    per-rank buckets), so every rank that runs it on the same gather holds the same bits.
 * ------------------------------------------------------------------------------------- */
int teco_conv3x3_wgrad_tc_det_plan_bytes(int32_t N, int32_t H, int32_t W, int32_t cin, int32_t cout, int64_t* ws_bytes_host);
int teco_conv3x3_wgrad_tc_det(int32_t N, int32_t H, int32_t W, int32_t cin_pad, int32_t cout_pad, int32_t cin, int32_t cout,
                              const void* x, const void* dz, float* dw, int32_t accumulate, void* ws, int64_t ws_bytes,
                              void* stream);
int teco_conv2d_wgrad_f32_det_plan_bytes(const teco_conv_desc* d, int32_t with_bias, int64_t* ws_bytes_host);
int teco_conv2d_wgrad_f32_det(const teco_conv_desc* d, const float* x, const float* dy, float* dw, float* db,
                              int32_t accumulate, void* ws, int64_t ws_bytes, void* stream);
int teco_bias_grad_f32_det_plan_bytes(int64_t npix, int32_t C, int64_t* ws_bytes_host);
int teco_bias_grad_f32_det(const float* dy, float* db, int64_t npix, int32_t C, int32_t cpitch, int32_t accumulate,
                           void* ws, int64_t ws_bytes, void* stream);
int teco_bn_det_plan_bytes(int64_t npix, int32_t C, int64_t* ws_bytes_host);
int teco_bn_train_f32_det(const float* x, const float* beta, float* y, float* stats, int64_t npix, int32_t C, float eps,
                          int32_t lrelu02, void* ws, int64_t ws_bytes, void* stream);
int teco_bn_train_bwd_f32_det(const float* x, const float* y, const float* dy, const float* stats, float* dx, float* dbeta,
                              int64_t npix, int32_t C, float eps, int32_t lrelu02, void* ws, int64_t ws_bytes, void* stream);
int teco_loss_det_plan_bytes(int64_t npix, int32_t C, int64_t* ws_bytes_host);
int teco_loss_l2_f32_det(const float* a, const float* b, float* out, float* da, int64_t npix, int32_t C, float gscale,
                         void* ws, int64_t ws_bytes, void* stream);
int teco_loss_l1_f32_det(const float* a, const float* b, float* out, float* da, float* db, int64_t npix, int32_t C,
                         int32_t per_pixel, float gscale, void* ws, int64_t ws_bytes, void* stream);
int teco_loss_cosine_f32_det(const float* f, const float* g, float* out, float* df, int64_t npix, int32_t C, float gscale,
                             void* ws, int64_t ws_bytes, void* stream);
int teco_loss_gan_f32_det(const float* d_fake, const float* d_real, float* out, float* g_adv, float* g_dis_f,
                          float* g_dis_r, int64_t n, float eps, float s_adv, float s_dis, void* ws, int64_t ws_bytes,
                          void* stream);
int teco_warp_bwd_f32_det_plan_bytes(int32_t N, int32_t H, int32_t W, int64_t* ws_bytes_host);
int teco_warp_bwd_f32_det(const float* img, const float* flow, const float* dout, float* dimg, float* dflow, int32_t N,
                          int32_t H, int32_t W, int32_t C, void* ws, int64_t ws_bytes, void* stream);
int teco_resize_bilinear_bwd_f32_det(const float* dy, float* dx, int32_t N, int32_t h, int32_t w, int32_t C, int32_t oh,
                                     int32_t ow, void* stream);
int teco_sum_ranks_f32(const float* src, int32_t R, int64_t n, float* dst, void* stream);

/* ---------------------------------------------------------------------------------------
 * Fused loss reductions (lib/Teco.py:316-413).  Each writes its scalar (fp32) to out[0] and, when the
 * gradient pointer is non-NULL, d(loss*gscale)/d(a) elementwise (same shape as a).
 * ------------------------------------------------------------------------------------- */
/* mean over pixels of sum_c (a-b)^2 : content loss :320-322, warp loss :329-331 */
int teco_loss_l2_f32(const float* a, const float* b, float* out, float* da, int64_t npix, int32_t C, float gscale,
                     void* stream);
/* mean |a-b| over all elements: ping-pong :364-367; mean over pixels of sum_c|a-b| when per_pixel!=0: layer loss :295-296 */
int teco_loss_l1_f32(const float* a, const float* b, float* out, float* da, float* db, int64_t npix, int32_t C,
                     int32_t per_pixel, float gscale, void* stream);
/* VGG cosine term :346-349 on raw features f,g [npix,C]: 1 - mean_pix( <f,g> / (|f|_eps |g|_eps) ) */
int teco_loss_cosine_f32(const float* f, const float* g, float* out, float* df, int64_t npix, int32_t C, float gscale,
                         void* stream);
/* per-pixel channel L2 normalisation of VGG features, lib/Teco.py:19-21: y = f / sqrt(sum_c f^2 + 1e-12) */
int teco_l2norm_channels_f32(const float* f, float* y, int64_t npix, int32_t C, void* stream);
/* GAN terms :376,394-399 on sigmoid outputs.  out[0]=mean -log(df+eps)  out[1]=mean -(log(1-df+eps)+log(dr+eps))
 * out[2]=mean log(dr+eps)  out[3]=mean dr  out[4]=mean df.  Gradients w.r.t. the sigmoid OUTPUTS:
 * g_adv = d(out0*s_adv)/d df ; g_dis_f, g_dis_r = d(out1*s_dis)/d(df,dr). */
int teco_loss_gan_f32(const float* d_fake, const float* d_real, float* out, float* g_adv, float* g_dis_f,
                      float* g_dis_r, int64_t n, float eps, float s_adv, float s_dis, void* stream);

/* tf.train.AdamOptimizer (lib/Teco.py:425,439-440), multi-tensor over one flat buffer of n floats.
 * lr_t = lr*sqrt(1-b2^t)/(1-b1^t) is computed by the caller.  gscale multiplies g (1/world after allreduce). */
int teco_adam_f32(float* p, float* m, float* v, const float* g, int64_t n, float lr_t, float b1, float b2, float eps,
                  float gscale, void* stream);

/* ---------------------------------------------------------------------------------------
 * Evaluation metrics on the device (SURVEY 8f-3; reference metrics.py).  tgt / out: uint8 RGB frames
 * [N,tH,tW,3] / [N,oH,oW,3] (the decoded PNGs; to_uint8(x,0,255) metrics.py:57-61 is the identity on them).
 * (y0,x0,h,w) is the crop_8x8 window of metrics.py:77-92, the same offsets in both frames (the reference
 * first cuts the output to the target size, metrics.py:134-135, which a window inside both frames covers).
 * acc: N x 4 doubles {sum (Yt-Yp)^2, ~bits(min Yp), bits(max Yp), sum of SSIM map} -- 8-byte slots, the
 * min / max of Y_pred held as (complemented) bit patterns so that zero is neutral for every slot.
 * Y = 16 + 0.2568 R + 0.5041 G + 0.0979 B in float64, metrics.py:37-55 (_rgb2ycbcr, maxVal 255).
 * ------------------------------------------------------------------------------------- */
/* psnr() metrics.py:63-70: zeroes acc, then fills slots 0..2.  PSNR_n = 20 log10(255 / sqrt(acc[n][0] / (h*w))). */
int teco_metrics_psnr_y_u8(const uint8_t* tgt, int32_t tH, int32_t tW, const uint8_t* out, int32_t oH, int32_t oW,
                           int32_t N, int32_t y0, int32_t x0, int32_t h, int32_t w, double* acc, void* stream);
/* ssim() metrics.py:72-75 = skimage compare_ssim(Y_true, Y_pred, data_range = max Yp - min Yp): 7x7 uniform
 * window, sample covariance, K1 0.01, K2 0.03, mean over the (h-6) x (w-6) positions whose window lies inside.
 * Needs slots 1..2 from teco_metrics_psnr_y_u8 on the same stream; adds into slot 3.
 * SSIM_n = acc[n][3] / ((h-6)*(w-6)).  h or w below 7 -> TECO_E_INVALID (skimage raises ValueError). */
int teco_metrics_ssim_y_u8(const uint8_t* tgt, int32_t tH, int32_t tW, const uint8_t* out, int32_t oH, int32_t oW,
                           int32_t N, int32_t y0, int32_t x0, int32_t h, int32_t w, double* acc, void* stream);

/* ---------------------------------------------------------------------------------------
 * LPIPS-AlexNet v0.1 and tLP100 (reference metrics.py:183-202, LPIPSmodels/).  The five convolutions of
 * torchvision alexnet().features[0:12] run through teco_conv2d_f32 with TECO_ACT_RELU; these three entry points
 * are the rest of the network and the distance.  All fp32 except the head's float64 accumulation.
 * ------------------------------------------------------------------------------------- */
/* util.py:142-144 im2tensor + networks_basic.py:131-132 scaling layer, bit for bit: uint8 RGB [N,H,W,3] read
 * through the window (y0,x0,h,w) -> x [N,h,w,3] fp32 = (float32(u8/127.5 - 1) - shift[c]) / scale[c] with the
 * first part in float64, shift = (-.030,-.088,-.188), scale = (.458,.448,.450). */
int teco_lpips_input_u8(const uint8_t* img, int32_t N, int32_t H, int32_t W, int32_t y0, int32_t x0, int32_t h,
                        int32_t w, float* x, void* stream);
/* torch MaxPool2d(3, stride 2), no padding, floor (alexnet().features[2] and [5], pretrained_networks.py:67-76):
 * x [N,H,W,C] -> y [N,(H-3)/2+1,(W-3)/2+1,C].  H or W below 3 -> TECO_E_INVALID. */
int teco_maxpool3s2_f32(const float* x, float* y, int32_t N, int32_t H, int32_t W, int32_t C, void* stream);
/* PNetLin head of one layer (networks_basic.py:150-177, util.py:72-75).  For pair p, with a = fa[ia_host[p]] and
 * b = fb[ib_host[p]] (feature maps [Na|Nb,H,W,C]) and f^ = f / (sqrt(sum_c f^2) + 1e-10):
 *   out[p] += mean over the H*W pixels of sum_c lin[c] * (a^ - b^)^2     (float64 accumulation, double out[P])
 * ia_host / ib_host: HOST arrays of P frame indices, 1 <= P <= 256; C <= 384. */
int teco_lpips_head_f32(const float* fa, int32_t Na, const float* fb, int32_t Nb, const int32_t* ia_host,
                        const int32_t* ib_host, int32_t P, int32_t H, int32_t W, int32_t C, const float* lin, double* out,
                        void* stream);

/* ---------------------------------------------------------------------------------------
 * tOF (reference metrics.py:143-169): cv2.cvtColor(RGB2GRAY) and cv2.calcOpticalFlowFarneback(prev, next, None,
 * 0.5, 3, 15, 3, 5, 1.2, 0) in stages, each batched over frames or frame pairs, then the per-pair tOF.  Only these
 * parameters exist.  Level k of an H x W frame is round_half_even(H / 2^k) x round_half_even(W / 2^k); levels
 * whose sides would fall below 32 are dropped (tecogan_b200/tof.py: pyramid_sizes).  DESIGN.md section 4.4.
 * ------------------------------------------------------------------------------------- */
/* uint8 RGB [N,H,W,3] read through the window (y0,x0,h,w) -> grey [N,h,w] uint8,
 * (9798 R + 19235 G + 3735 B + 16384) >> 15 (cv2's COLOR_RGB2GRAY on uint8, bit for bit). */
int teco_tof_grey_u8(const uint8_t* img, int32_t N, int32_t H, int32_t W, int32_t y0, int32_t x0, int32_t h, int32_t w,
                     uint8_t* grey, void* stream);
/* Pyramid level 0..3 of full-resolution grey frames [N,H,W] -> out [N,lh,lw] fp32: Gaussian blur (reflect-101;
 * sigma (2^level - 1) / 2, ksize max(cvRound(5 sigma) | 1, 3); level 0: the fixed 1/4 1/2 1/4) of the FULL frame,
 * then INTER_LINEAR to lh x lw (an exact halving is the 2x2 mean).  (lh, lw) must be the level's size. */
int teco_farneback_pyramid_u8(const uint8_t* grey, int32_t N, int32_t H, int32_t W, int32_t level, int32_t lh, int32_t lw,
                              float* out, void* stream);
/* Polynomial expansion (poly_n 5, sigma 1.2) of fp32 images [N,h,w] -> R [N,h,w,5] fp32, channels = coefficients
 * of (y, x, yy, xx, xy); borders replicated.  One R per frame and level serves every pair that uses the frame. */
int teco_farneback_polyexp_f32(const float* img, int32_t N, int32_t h, int32_t w, float* R, void* stream);
/* One update iteration of P pairs: pair p = (R[i0_host[p]], R[i1_host[p]]) of R [Nf,h,w,5], flow_in [P,h,w,2]
 * (NULL: zero flow) -> flow_out [P,h,w,2] (must not alias flow_in).  Per-pixel field from R0, R1 sampled at
 * x + flow and the border weights, 15x15 box mean (float64), (g11 g22 - g12^2 + 1e-3)-regularised solve.
 * i0_host / i1_host: HOST arrays, 1 <= P <= 256. */
int teco_farneback_iterate_f32(const float* R, int32_t Nf, int32_t h, int32_t w, const int32_t* i0_host,
                               const int32_t* i1_host, int32_t P, const float* flow_in, float* flow_out, void* stream);
/* Flow of the coarser level [P,sh,sw,2] -> INTER_LINEAR to [P,h,w,2], times 2 (1 / pyr_scale). */
int teco_farneback_flow_up_f32(const float* flow_in, int32_t P, int32_t sh, int32_t sw, float* flow_out, int32_t h,
                               int32_t w, void* stream);
/* tOF of P flow pairs [P,H,W,2] over the window (y0,x0,h,w) (crop_8x8): out[p] = mean of
 * sqrt(|a-b|_x^2 + |a-b|_y^2) (fp32 per pixel as numpy, float64 sum; no atomics: deterministic).
 * partial: scratch of P * 32 doubles. */
int teco_tof_reduce_f32(const float* flow_a, const float* flow_b, int32_t P, int32_t H, int32_t W, int32_t y0, int32_t x0,
                        int32_t h, int32_t w, double* partial, double* out, void* stream);

/* ---------------------------------------------------------------------------------------
 * PNG encoding of one RGB uint8 frame, byte-identical to cv2.imwrite(path.png, bgr) (libpng: filter Sub, zlib level 1,
 * Z_RLE, 8 192-byte IDAT chunks), the file save_img writes (reference lib/ops.py:521-523).  DESIGN.md section 4.5.
 * ------------------------------------------------------------------------------------- */
/* Host-only size query for an H x W frame: the workspace (device, 256-byte aligned) and the output capacity in bytes.
 * H, W >= 1 and H * (3W + 1) <= 2^30, else TECO_E_INVALID. */
int teco_png_plan_bytes(int32_t H, int32_t W, int64_t* workspace_bytes_host, int64_t* out_capacity_host);
/* rgb [H,W,3] uint8 -> out: the complete PNG file; *out_len (device int64) receives its length.  Buffers smaller than
 * teco_png_plan_bytes gives -> TECO_E_INVALID.  Nothing allocates; every stage runs on `stream`. */
int teco_png_encode_rgb8(const uint8_t* rgb, int32_t H, int32_t W, void* workspace, int64_t workspace_bytes, uint8_t* out,
                         int64_t out_capacity, int64_t* out_len, void* stream);

/* ---------------------------------------------------------------------------------------
 * PNG decoding of a batch of files to RGB uint8, byte-identical to cv2.imread(path, IMREAD_COLOR)[..., ::-1] on the
 * subset the device takes (non-interlaced; grey 1/2/4/8 bits, RGB 8, palette 1/2/4/8, grey + alpha 8, RGBA 8;
 * 1 <= H, W <= 65500).  The caller walks the chunks and checks the CRCs; the device reports per file whether its zlib
 * stream decoded exactly.  DESIGN.md section 4.7.
 * ------------------------------------------------------------------------------------- */
/* Host-only size query: the workspace bytes one file of this size and format needs (its filtered rows, rounded up to
 * 256).  Sizes or formats outside the subset -> TECO_E_INVALID. */
int teco_png_decode_plan_bytes(int32_t H, int32_t W, int32_t colour_type, int32_t bit_depth, int64_t* workspace_bytes_host);
/* desc: device int64 [nfiles, 11], one row per file:
 *   0 stream offset in src, 1 stream length (the IDAT data, concatenated), 2 H, 3 W, 4 colour type, 5 bit depth,
 *   6 palette offset in src, 7 palette entries (colour type 3; else unused), 8 destination offset in dst,
 *   9 destination row pitch in bytes (>= 3W), 10 workspace offset (rows of the sizes teco_png_decode_plan_bytes gives,
 *   not overlapping one another or dst).
 * status: device int32 [nfiles], written for every file: 0 the RGB frame is at dst; otherwise nothing is promised about
 * the file's destination rows and the caller decodes it another way.  1 zlib header, 2 block type or stored length,
 * 3 Huffman code or code lengths, 4 symbol outside the code, 5 distance before the start or beyond the window,
 * 6 stream ends early, 7 more bytes than H * (rowbytes + 1), 8 fewer, 9 Adler-32, 10 bytes after the Adler-32,
 * 11 filter type above 4, 12 palette index beyond the palette, 13 descriptor outside the buffers or the subset.
 * No file reads or writes outside its own ranges.  Nothing allocates; every stage runs on `stream`. */
int teco_png_decode_rgb8(const uint8_t* src, int64_t src_bytes, const int64_t* desc, int32_t nfiles, void* workspace,
                         int64_t workspace_bytes, uint8_t* dst, int64_t dst_bytes, int32_t* status, void* stream);

/* ---------------------------------------------------------------------------------------
 * JPEG encoding of one RGB uint8 frame, byte-identical to cv2.imwrite(path.jpg, bgr) with cv2's defaults (baseline,
 * quality 95, 4:2:0, islow FDCT, the Annex K Huffman tables), the file save_img writes by default (reference
 * lib/ops.py:521-523, main.py --output_ext jpg).  DESIGN.md section 4.6.
 * ------------------------------------------------------------------------------------- */
/* Host-only size query for an H x W frame: the workspace (device, 256-byte aligned) and the output capacity in bytes.
 * 1 <= H, W <= 65500 (JPEG's limit), else TECO_E_INVALID. */
int teco_jpeg_plan_bytes(int32_t H, int32_t W, int64_t* workspace_bytes_host, int64_t* out_capacity_host);
/* rgb [H,W,3] uint8 -> out: the complete JPEG file; *out_len (device int64) receives its length.  Buffers smaller than
 * teco_jpeg_plan_bytes gives -> TECO_E_INVALID.  Nothing allocates; every stage runs on `stream`. */
int teco_jpeg_encode_rgb8(const uint8_t* rgb, int32_t H, int32_t W, void* workspace, int64_t workspace_bytes, uint8_t* out,
                          int64_t out_capacity, int64_t* out_len, void* stream);

/* ---------------------------------------------------------------------------------------
 * GIF89a encoding of a batch of RGB uint8 animations, the TensorBoard image summaries of training (reference
 * lib/Teco.py:498-503, lib/ops.py:399-431): per animation one median-cut palette of up to 256 colours over all of its
 * frames, Sierra-2-4A error diffusion per frame, LZW at minimum code size 8, 33 cs per frame, looping.  DESIGN.md
 * section 4.8 specifies every rule; an animation of at most 256 distinct colours is stored exactly.
 * ------------------------------------------------------------------------------------- */
/* tf.image.convert_image_dtype(x, uint8, saturate=True) in float32: y = trunc(clamp(x * 255.5, 0, 255)), NaN -> 0;
   deprocess = 1 first maps x to (x + 1) / 2 (reference lib/ops.py:17-22).  n elements, any layout. */
int teco_convert_image_u8(const float* x, uint8_t* y, int64_t n, int32_t deprocess, void* stream);
/* Host-only size query for N animations of T frames of H x W: the workspace (device, 256-byte aligned) and the output
 * capacity in bytes.  N, T >= 1, 1 <= H, W <= 65535 and T * H * W <= 2^28, else TECO_E_INVALID. */
int teco_gif_plan_bytes(int32_t N, int32_t T, int32_t H, int32_t W, int64_t* workspace_bytes_host,
                        int64_t* out_capacity_host);
/* rgb [N,T,H,W,3] uint8 -> out: the N GIF files back to back; out_len (device int64 [N]) receives each file's length,
 * so file i starts at the sum of the lengths before it.  Buffers smaller than teco_gif_plan_bytes gives ->
 * TECO_E_INVALID.  Nothing allocates; every stage runs on `stream`. */
int teco_gif_encode_rgb8(const uint8_t* rgb, int32_t N, int32_t T, int32_t H, int32_t W, void* workspace,
                         int64_t workspace_bytes, uint8_t* out, int64_t out_capacity, int64_t* out_len, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TECO_H_ */
