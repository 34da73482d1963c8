// GIF89a encoder for batches of RGB uint8 animations, the TensorBoard image summaries of training (reference
// lib/ops.py:399-431 encodes them with ffmpeg's palettegen + paletteuse; this follows the same recipe -- one palette per
// animation, Sierra-2-4A error diffusion, 3 fps -- exactly as DESIGN.md section 4.8 specifies it).
// tests/golden/gif_oracle.py states every stage on the host; tests/test_gif_host.py pins it to cv2 and PIL.
//
// Stages (one kernel each, all on the caller's stream):
//   gif_palette   one CTA per animation: median cut over every pixel of every frame, one 8-bit label per pixel and one
//                 3 x 256-bin histogram per box, so a split is one pass over the labels and no sort or hash
//   gif_dither    one CTA per frame: Sierra-2-4A as a wavefront, one thread per row, row y two pixels behind row y - 1
//   gif_lzw       one thread per frame: GIF LZW with the dictionary hashed in shared memory, packed LSB first
//   gif_layout    one thread: each frame's offset in the output and each animation's size
//   gif_assemble  one CTA per frame: header and global table (first frame), Graphic Control Extension, image
//                 descriptor, the LZW data in 255-byte sub-blocks, trailer (last frame)
// Plus teco_convert_image_u8: tf.image.convert_image_dtype(x, uint8, saturate=True), optionally after deprocess.
#include "teco_common.cuh"

namespace {

constexpr int MAX_SIDE = 65535;                  // the 16-bit sides of the logical screen and image descriptor
constexpr long long MAX_ANIM_PIXELS = 1LL << 28; // labels and indices use 32-bit offsets within an animation
constexpr int PAL_T = 1024;
constexpr int DITHER_T = 256;
constexpr int ASM_T = 256;
constexpr int HIST = 3 * 256;                    // per box: R, G, B histograms
constexpr int HDR_BYTES = 6 + 7 + 768 + 19;      // signature, logical screen, global table, NETSCAPE2.0 extension
constexpr int FRAME_HDR = 8 + 10 + 1;            // Graphic Control Extension, image descriptor, minimum code size
constexpr int DELAY_CS = 33;                     // 3 fps (the reference's summary fps)
constexpr int CLEAR = 256, EOI = 257, FIRST_CODE = 258, MAX_CODES = 4096;
constexpr int HASH_BITS = 13, HASH_SLOTS = 1 << HASH_BITS;   // load factor <= 3838 / 8192
constexpr uint32_t EMPTY = 0xFFFFFFFFu;          // key (4095, 255) never occurs: the table resets once code 4095 exists

// LZW bytes of one frame of P pixels, at most.  Codes: the first Clear, one per emitted string (each covers >= 1 pixel,
// so <= P), one mid-stream Clear per 4096 - 258 = 3838 table additions (each addition follows an emitted string, so
// <= P / 3838), and EOI: codes <= P + P / 3838 + 2, each at most 12 bits.
__host__ __device__ inline long long lzw_cap(long long P) { return ((P + P / 3838 + 2) * 12 + 7) / 8; }
// Bytes of one frame's block in the file given nb LZW bytes: headers, a length byte per 255-byte sub-block, terminator.
__host__ __device__ inline long long frame_bytes(long long nb) { return FRAME_HDR + nb + (nb + 254) / 255 + 1; }
inline long long align256(long long v) { return (v + 255) & ~255LL; }
inline long long align16(long long v) { return (v + 15) & ~15LL; }

struct Plan {
  int N, T, H, W;
  long long Pf, Pa;                            // pixels per frame, per animation
  long long lab_stride, idx_stride, err_stride, lzw_stride;
  long long off_lab, off_hist, off_pal, off_npal, off_idx, off_err, off_lzw, off_nb, off_foff, off_aoff;
  long long ws_bytes, out_cap;
};

Plan make_plan(int N, int T, int H, int W) {
  Plan p{};
  p.N = N; p.T = T; p.H = H; p.W = W;
  p.Pf = (long long)H * W;
  p.Pa = p.Pf * T;
  const long long NT = (long long)N * T;
  p.lab_stride = align16(p.Pa);
  p.idx_stride = align16(p.Pf);
  p.err_stride = align16((long long)W * 3 * 4);
  p.lzw_stride = align16(lzw_cap(p.Pf));
  long long o = 0;
  p.off_lab = o;  o = align256(o + N * p.lab_stride);
  p.off_hist = o; o = align256(o + (long long)N * 256 * HIST * 4);
  p.off_pal = o;  o = align256(o + (long long)N * 256 * 4);
  p.off_npal = o; o = align256(o + (long long)N * 4);
  p.off_idx = o;  o = align256(o + NT * p.idx_stride);
  p.off_err = o;  o = align256(o + NT * p.err_stride);
  p.off_lzw = o;  o = align256(o + NT * p.lzw_stride);
  p.off_nb = o;   o = align256(o + NT * 8);
  p.off_foff = o; o = align256(o + NT * 8);
  p.off_aoff = o; o = align256(o + (long long)N * 8);
  p.ws_bytes = o;
  p.out_cap = N * (HDR_BYTES + T * frame_bytes(lzw_cap(p.Pf)) + 1);
  return p;
}

bool plan_ok(int N, int T, int H, int W) {
  return N >= 1 && T >= 1 && H >= 1 && W >= 1 && H <= MAX_SIDE && W <= MAX_SIDE &&
         (long long)T * H * W <= MAX_ANIM_PIXELS && (long long)N * T <= (1LL << 30);
}

struct Bufs {
  uint8_t* lab;       // [N][lab_stride] box of every pixel
  int* hist;          // [N][256 boxes][768]
  uint32_t* pal;      // [N][256] 0x00BBGGRR
  int* npal;          // [N]
  uint8_t* idx;       // [N*T][idx_stride] palette index of every pixel
  int* err;           // [N*T][err_stride / 4] the row buffer of errors for the next row
  uint8_t* lzw;       // [N*T][lzw_stride]
  long long* nb;      // [N*T] LZW bytes
  long long* foff;    // [N*T] offset of the frame's block in out
  long long* aoff;    // [N] offset of the animation in out
};

Bufs carve(const Plan& p, void* ws) {
  uint8_t* b = (uint8_t*)ws;
  Bufs u;
  u.lab = b + p.off_lab;
  u.hist = (int*)(b + p.off_hist);
  u.pal = (uint32_t*)(b + p.off_pal);
  u.npal = (int*)(b + p.off_npal);
  u.idx = b + p.off_idx;
  u.err = (int*)(b + p.off_err);
  u.lzw = b + p.off_lzw;
  u.nb = (long long*)(b + p.off_nb);
  u.foff = (long long*)(b + p.off_foff);
  u.aoff = (long long*)(b + p.off_aoff);
  return u;
}

// ------------------------------------------------------------------------------------------------------ palette
// Stats of one box from its histogram h (768 bins): pixel count, per-channel min and max.  The caller has set
// cnt[i] = 0, mn[i][c] = 256, mx[i][c] = -1 and synchronised.
__device__ void box_stats(int hv, int k, int i, int* cnt, int* mn, int* mx) {
  if (k < HIST && hv > 0) {
    atomicMin(&mn[i * 3 + k / 256], k % 256);
    atomicMax(&mx[i * 3 + k / 256], k % 256);
  }
  int c = k < 256 ? hv : 0;                    // the R histogram counts every pixel once
  c = __reduce_add_sync(0xffffffffu, c);
  if ((k & 31) == 0 && c) atomicAdd(&cnt[i], c);
}

__global__ void __launch_bounds__(PAL_T) gif_palette(const uint8_t* __restrict__ rgb, Plan p, Bufs u) {
  __shared__ int hc[HIST];
  __shared__ int cnt[256], mn[256 * 3], mx[256 * 3];
  __shared__ long long s_red[PAL_T / 32];
  __shared__ int s_scan[8], s_v;
  const int a = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const long long P = p.Pa;
  const uint8_t* px = rgb + (long long)a * P * 3;
  uint8_t* lab = u.lab + (long long)a * p.lab_stride;
  int* hist = u.hist + (long long)a * 256 * HIST;

  for (int k = tid; k < HIST; k += PAL_T) hc[k] = 0;
  for (int k = tid; k < 256; k += PAL_T) cnt[k] = 0;
  for (int k = tid; k < 256 * 3; k += PAL_T) { mn[k] = 256; mx[k] = -1; }
  __syncthreads();
  for (long long i = tid; i < P; i += PAL_T) {          // box 0: every pixel
    lab[i] = 0;
    atomicAdd(&hc[px[3 * i]], 1);
    atomicAdd(&hc[256 + px[3 * i + 1]], 1);
    atomicAdd(&hc[512 + px[3 * i + 2]], 1);
  }
  __syncthreads();
  if (tid < HIST) hist[tid] = hc[tid];
  box_stats(tid < HIST ? hc[tid] : 0, tid, 0, cnt, mn, mx);
  __syncthreads();

  int nbox = 1;
  while (nbox < 256) {
    // the splittable box with the most pixels, the lowest index on a tie: max of (count << 8 | 255 - index)
    long long key = -1;
    if (tid < nbox) {
      const bool split = mx[tid * 3] > mn[tid * 3] || mx[tid * 3 + 1] > mn[tid * 3 + 1] || mx[tid * 3 + 2] > mn[tid * 3 + 2];
      if (split) key = ((long long)cnt[tid] << 8) | (255 - tid);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) key = max(key, __shfl_xor_sync(0xffffffffu, key, o));
    if (lane == 0) s_red[wid] = key;
    __syncthreads();
    key = s_red[0];
    for (int w = 1; w < 8; ++w) key = max(key, s_red[w]);   // boxes live in the first 256 threads (8 warps)
    if (key < 0) break;                                     // every box holds one colour
    const int b = 255 - (int)(key & 255);
    int axis = 0, best = mx[b * 3] - mn[b * 3];             // largest max - min; ties R, then G, then B
    if (mx[b * 3 + 1] - mn[b * 3 + 1] > best) { axis = 1; best = mx[b * 3 + 1] - mn[b * 3 + 1]; }
    if (mx[b * 3 + 2] - mn[b * 3 + 2] > best) axis = 2;
    const int lo = mn[b * 3 + axis], hi = mx[b * 3 + axis], n = cnt[b];

    // split value: the smallest v in [lo, hi - 1] with 2 count(axis <= v) >= n, else hi - 1
    int h = tid < 256 ? hist[b * HIST + axis * 256 + tid] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, h, o);
      if (lane >= o) h += t;
    }
    if (tid < 256 && lane == 31) s_scan[wid] = h;
    if (tid == 0) s_v = hi - 1;
    for (int k = tid; k < HIST; k += PAL_T) hc[k] = 0;
    __syncthreads();
    if (tid < 256) {
      for (int w = 0; w < wid; ++w) h += s_scan[w];
      if (tid >= lo && tid < hi && 2LL * h >= n) atomicMin(&s_v, tid);
    }
    __syncthreads();
    const int v = s_v;

    // pixels of box b above v move to box nbox; hc collects the new box's histogram
    const uint32_t bb = 0x01010101u * (uint32_t)b;
    const long long nq = P >> 2;
    uint32_t* lab4 = reinterpret_cast<uint32_t*>(lab);
    for (long long q = tid; q < nq; q += PAL_T) {
      const uint32_t l = lab4[q];
      const uint32_t m = __vcmpeq4(l, bb);
      if (!m) continue;
      uint32_t nl = l;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (!((m >> (8 * k)) & 0xFF)) continue;
        const uint8_t* pp = px + 3 * (4 * q + k);
        if (pp[axis] > v) {
          nl = (nl & ~(0xFFu << (8 * k))) | ((uint32_t)nbox << (8 * k));
          atomicAdd(&hc[pp[0]], 1);
          atomicAdd(&hc[256 + pp[1]], 1);
          atomicAdd(&hc[512 + pp[2]], 1);
        }
      }
      if (nl != l) lab4[q] = nl;
    }
    for (long long i = 4 * nq + tid; i < P; i += PAL_T) {
      if (lab[i] != b) continue;
      const uint8_t* pp = px + 3 * i;
      if (pp[axis] > v) {
        lab[i] = (uint8_t)nbox;
        atomicAdd(&hc[pp[0]], 1);
        atomicAdd(&hc[256 + pp[1]], 1);
        atomicAdd(&hc[512 + pp[2]], 1);
      }
    }
    if (tid == 0) { cnt[b] = 0; cnt[nbox] = 0; }
    if (tid < 3) { mn[b * 3 + tid] = mn[nbox * 3 + tid] = 256; mx[b * 3 + tid] = mx[nbox * 3 + tid] = -1; }
    __syncthreads();
    int hn = 0, hp = 0;
    if (tid < HIST) {
      hn = hc[tid];
      hp = hist[b * HIST + tid] - hn;
      hist[b * HIST + tid] = hp;
      hist[nbox * HIST + tid] = hn;
    }
    box_stats(hp, tid, b, cnt, mn, mx);
    box_stats(hn, tid, nbox, cnt, mn, mx);
    ++nbox;
    __syncthreads();
  }

  // entry = per-channel (sum + n / 2) / n over the box's pixels: one warp per box
  for (int i = wid; i < nbox; i += PAL_T / 32) {
    const int* hb = hist + i * HIST;
    long long s[3] = {0, 0, 0};
    for (int k = lane; k < 256; k += 32) {
      s[0] += (long long)k * hb[k];
      s[1] += (long long)k * hb[256 + k];
      s[2] += (long long)k * hb[512 + k];
    }
    uint32_t e = 0;
    const long long n = cnt[i];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
      for (int o = 16; o; o >>= 1) s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
      e |= (uint32_t)((s[c] + n / 2) / n) << (8 * c);
    }
    if (lane == 0) u.pal[a * 256 + i] = e;
  }
  if (tid == 0) u.npal[a] = nbox;
}

// ------------------------------------------------------------------------------------------------------- dither
// Sierra-2-4A: pixel (x, y) sends (2e) / 4 right, e / 4 to (x - 1, y + 1) and e / 4 to (x, y + 1).  Row y's thread
// handles pixel x at step x + 2y: (x + 1, y - 1) is then done.  err[x] holds what row y - 1 sent to (x, y): row y - 1
// writes it at step x + 1 + 2(y - 1) (after its pixel x + 1), row y reads it at step x + 2y, and row y writes err[x]
// again at step x + 1 + 2y.  In one step row r reads err[s - 2r] and writes err[s - 2r - 1] (and err[W - 1] at its last
// pixel, read by row r + 1 two steps later): no two rows touch the same entry, so one row buffer serves the frame.
// Rows beyond the CTA run in further passes; the buffer then holds the previous pass's last row.
__global__ void __launch_bounds__(DITHER_T) gif_dither(const uint8_t* __restrict__ rgb, Plan p, Bufs u) {
  __shared__ uint32_t spal[256];
  const int f = blockIdx.x, a = f / p.T, tid = threadIdx.x, H = p.H, W = p.W;
  const int npal = u.npal[a];
  for (int k = tid; k < npal; k += DITHER_T) spal[k] = u.pal[a * 256 + k];
  const uint8_t* src = rgb + (long long)f * p.Pf * 3;
  uint8_t* out = u.idx + (long long)f * p.idx_stride;
  int* err = u.err + (long long)f * (p.err_stride / 4);
  for (int k = tid; k < 3 * W; k += DITHER_T) err[k] = 0;
  __syncthreads();
  for (int r0 = 0; r0 < H; r0 += DITHER_T) {
    const int rows = min(DITHER_T, H - r0), y = r0 + tid;
    int cr = 0, cg = 0, cb = 0;          // error carried to the right
    int pr = 0, pg = 0, pb = 0;          // e of the previous pixel (x - 1)
    const int steps = W + 2 * (rows - 1);
    for (int s = 0; s < steps; ++s) {
      const int x = s - 2 * tid;
      if (tid < rows && x >= 0 && x < W) {
        const uint8_t* sp = src + ((long long)y * W + x) * 3;
        const int r = min(max((int)sp[0] + cr + err[3 * x], 0), 255);
        const int g = min(max((int)sp[1] + cg + err[3 * x + 1], 0), 255);
        const int b = min(max((int)sp[2] + cb + err[3 * x + 2], 0), 255);
        const uint32_t c = (uint32_t)r | ((uint32_t)g << 8) | ((uint32_t)b << 16);
        int best = 0;
        uint32_t bd = 0xFFFFFFFFu;
        for (int j = 0; j < npal; ++j) {
          const uint32_t d4 = __vabsdiffu4(c, spal[j]);
          const uint32_t d = __dp4a(d4, d4, 0u);
          if (d < bd) { bd = d; best = j; }
        }
        out[(long long)y * W + x] = (uint8_t)best;
        const uint32_t q = spal[best];
        const int er = r - (int)(q & 255), eg = g - (int)((q >> 8) & 255), eb = b - (int)((q >> 16) & 255);
        cr = (2 * er) / 4; cg = (2 * eg) / 4; cb = (2 * eb) / 4;
        if (x > 0) {
          err[3 * (x - 1)] = pr / 4 + er / 4;
          err[3 * (x - 1) + 1] = pg / 4 + eg / 4;
          err[3 * (x - 1) + 2] = pb / 4 + eb / 4;
        }
        if (x == W - 1) {
          err[3 * x] = er / 4;
          err[3 * x + 1] = eg / 4;
          err[3 * x + 2] = eb / 4;
        }
        pr = er; pg = eg; pb = eb;
      }
      __syncthreads();
    }
  }
}

// ---------------------------------------------------------------------------------------------------------- LZW
struct BitOut {
  uint8_t* o;
  long long n;
  unsigned long long acc;
  int nacc;
  __device__ void put(int code, int width) {
    acc |= (unsigned long long)code << nacc;
    nacc += width;
    while (nacc >= 8) {
      o[n++] = (uint8_t)acc;
      acc >>= 8;
      nacc -= 8;
    }
  }
};

__device__ void clear_table(uint32_t* tab) {
  uint4* t4 = reinterpret_cast<uint4*>(tab);
  for (int k = 0; k < HASH_SLOTS / 4; ++k) t4[k] = make_uint4(EMPTY, EMPTY, EMPTY, EMPTY);
}

__global__ void __launch_bounds__(1) gif_lzw(Plan p, Bufs u) {
  __shared__ __align__(16) uint32_t tab[HASH_SLOTS];    // (prefix code << 8 | byte) << 12 | code
  const int f = blockIdx.x;
  const uint8_t* in = u.idx + (long long)f * p.idx_stride;
  const uint4* in16 = reinterpret_cast<const uint4*>(in);
  BitOut bo{u.lzw + (long long)f * p.lzw_stride, 0, 0ull, 0};
  const long long P = p.Pf;
  clear_table(tab);
  int width = 9, next = FIRST_CODE;
  bo.put(CLEAR, width);
  uint4 w = in16[0];
  int cur = w.x & 255;
  for (long long i = 1; i < P; ++i) {
    if ((i & 15) == 0) w = in16[i >> 4];
    const int k = (int)(i & 15);
    const uint32_t word = k < 4 ? w.x : k < 8 ? w.y : k < 12 ? w.z : w.w;
    const int c = (word >> (8 * (k & 3))) & 255;
    const uint32_t key = ((uint32_t)cur << 8) | (uint32_t)c;
    uint32_t h = (key * 2654435761u) >> (32 - HASH_BITS);
    uint32_t e;
    while ((e = tab[h]) != EMPTY && (e >> 12) != key) h = (h + 1) & (HASH_SLOTS - 1);
    if (e != EMPTY) {
      cur = (int)(e & 0xFFF);
      continue;
    }
    bo.put(cur, width);
    if (next == (1 << width) && width < 12) ++width;
    tab[h] = (key << 12) | (uint32_t)next;
    if (++next == MAX_CODES) {
      bo.put(CLEAR, 12);
      clear_table(tab);
      width = 9;
      next = FIRST_CODE;
    }
    cur = c;
  }
  bo.put(cur, width);
  if (next == (1 << width) && width < 12) ++width;
  bo.put(EOI, width);
  if (bo.nacc) bo.o[bo.n++] = (uint8_t)bo.acc;
  u.nb[f] = bo.n;
}

// ------------------------------------------------------------------------------------------------ file assembly
__global__ void gif_layout(Plan p, Bufs u, int64_t* __restrict__ out_len) {
  if (threadIdx.x != 0) return;
  long long o = 0;
  for (int a = 0; a < p.N; ++a) {
    const long long a0 = o;
    u.aoff[a] = o;
    o += HDR_BYTES;
    for (int t = 0; t < p.T; ++t) {
      const int f = a * p.T + t;
      u.foff[f] = o;
      o += frame_bytes(u.nb[f]);
    }
    o += 1;                                          // trailer
    out_len[a] = o - a0;
  }
}

__device__ __forceinline__ void put16(uint8_t* o, int v) { o[0] = (uint8_t)v; o[1] = (uint8_t)(v >> 8); }

__global__ void __launch_bounds__(ASM_T) gif_assemble(Plan p, Bufs u, uint8_t* __restrict__ out) {
  const int f = blockIdx.x, a = f / p.T, t = f % p.T, tid = threadIdx.x;
  if (t == 0) {
    uint8_t* o = out + u.aoff[a];
    const int npal = u.npal[a];
    for (int k = tid; k < 768; k += ASM_T) {
      const int i = k / 3;
      o[13 + k] = i < npal ? (uint8_t)(u.pal[a * 256 + i] >> (8 * (k % 3))) : 0;
    }
    if (tid == 0) {
      const char sig[6] = {'G', 'I', 'F', '8', '9', 'a'};
      for (int k = 0; k < 6; ++k) o[k] = (uint8_t)sig[k];
      put16(o + 6, p.W);
      put16(o + 8, p.H);
      o[10] = 0xF7;                                  // global table of 2^(7+1) entries, 8 bits per primary
      o[11] = 0;                                     // background
      o[12] = 0;                                     // aspect
      const uint8_t app[19] = {0x21, 0xFF, 0x0B, 'N', 'E', 'T', 'S', 'C', 'A', 'P', 'E', '2', '.', '0', 0x03, 0x01, 0, 0, 0};
      for (int k = 0; k < 19; ++k) o[13 + 768 + k] = app[k];
    }
  }
  uint8_t* o = out + u.foff[f];
  const long long nb = u.nb[f];
  if (tid == 0) {
    o[0] = 0x21; o[1] = 0xF9; o[2] = 0x04; o[3] = 0x00;   // Graphic Control Extension: no transparency
    put16(o + 4, DELAY_CS);
    o[6] = 0; o[7] = 0;
    o[8] = 0x2C;                                         // image descriptor: (0, 0), W x H, no local table
    put16(o + 9, 0); put16(o + 11, 0); put16(o + 13, p.W); put16(o + 15, p.H);
    o[17] = 0;
    o[18] = 8;                                           // minimum code size
  }
  const uint8_t* z = u.lzw + (long long)f * p.lzw_stride;
  const long long nblk = (nb + 254) / 255, total = nb + nblk;
  uint8_t* d = o + FRAME_HDR;
  for (long long j = tid; j < total; j += ASM_T) {
    const long long k = j >> 8, r = j & 255;
    d[j] = r == 0 ? (uint8_t)min(255LL, nb - 255 * k) : z[255 * k + r - 1];
  }
  if (tid == 0) {
    d[total] = 0;                                        // block terminator
    if (t == p.T - 1) d[total + 1] = 0x3B;               // trailer
  }
}

// ------------------------------------------------------------------------------------------------- quantisation
// tf.image.convert_image_dtype(x, tf.uint8, saturate=True) (reference lib/ops.py:475): trunc(clamp(x * 255.5, 0, 255))
// in float32, after deprocess (x + 1) / 2 when asked.  fmaxf first: NaN -> 0.
__global__ void convert_image_u8_kernel(const float* __restrict__ x, uint8_t* __restrict__ y, long long n, int deprocess) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float v = x[i];
    if (deprocess) v = __fmul_rn(__fadd_rn(v, 1.0f), 0.5f);
    y[i] = (uint8_t)fminf(fmaxf(__fmul_rn(v, 255.5f), 0.0f), 255.0f);
  }
}

}  // namespace

extern "C" {

int teco_convert_image_u8(const float* x, uint8_t* y, int64_t n, int32_t deprocess, void* stream) {
  TECO_CHECK_ARG(x && y && n > 0, "teco_convert_image_u8: bad argument");
  TECO_CHECK_ARG(deprocess == 0 || deprocess == 1, "teco_convert_image_u8: deprocess must be 0 or 1");
  const long long blocks = (n + 255) / 256 < 2048 ? (n + 255) / 256 : 2048;
  convert_image_u8_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(x, y, n, deprocess);
  TECO_CUDA_LAUNCH_CHECK("teco_convert_image_u8");
  return TECO_OK;
}

int teco_gif_plan_bytes(int32_t N, int32_t T, int32_t H, int32_t W, int64_t* workspace_bytes_host,
                        int64_t* out_capacity_host) {
  TECO_CHECK_ARG(workspace_bytes_host && out_capacity_host, "teco_gif_plan_bytes: NULL argument");
  TECO_CHECK_ARG(plan_ok(N, T, H, W),
                 "teco_gif_plan_bytes: bad animation batch N=%d T=%d %dx%d (N, T >= 1, 1 <= H, W <= %d, T*H*W <= 2^28)",
                 N, T, H, W, MAX_SIDE);
  const Plan p = make_plan(N, T, H, W);
  *workspace_bytes_host = p.ws_bytes;
  *out_capacity_host = p.out_cap;
  return TECO_OK;
}

int teco_gif_encode_rgb8(const uint8_t* rgb, int32_t N, int32_t T, int32_t H, int32_t W, void* workspace,
                         int64_t workspace_bytes, uint8_t* out, int64_t out_capacity, int64_t* out_len, void* stream) {
  TECO_CHECK_ARG(rgb && workspace && out && out_len, "teco_gif_encode_rgb8: NULL argument");
  TECO_CHECK_ARG(plan_ok(N, T, H, W),
                 "teco_gif_encode_rgb8: bad animation batch N=%d T=%d %dx%d (N, T >= 1, 1 <= H, W <= %d, T*H*W <= 2^28)",
                 N, T, H, W, MAX_SIDE);
  const Plan p = make_plan(N, T, H, W);
  TECO_CHECK_ARG(workspace_bytes >= p.ws_bytes && out_capacity >= p.out_cap,
                 "teco_gif_encode_rgb8: buffers of %lld / %lld bytes, the plan needs %lld / %lld",
                 (long long)workspace_bytes, (long long)out_capacity, p.ws_bytes, p.out_cap);
  TECO_CHECK_ARG(((uintptr_t)workspace & 255) == 0, "teco_gif_encode_rgb8: workspace must be 256-byte aligned");
  const cudaStream_t st = (cudaStream_t)stream;
  const Bufs u = carve(p, workspace);
  const unsigned NT = (unsigned)((long long)N * T);
  gif_palette<<<N, PAL_T, 0, st>>>(rgb, p, u);
  gif_dither<<<NT, DITHER_T, 0, st>>>(rgb, p, u);
  gif_lzw<<<NT, 1, 0, st>>>(p, u);
  gif_layout<<<1, 32, 0, st>>>(p, u, out_len);
  gif_assemble<<<NT, ASM_T, 0, st>>>(p, u, out);
  TECO_CUDA_LAUNCH_CHECK("teco_gif_encode_rgb8");
  return TECO_OK;
}

}  // extern "C"
