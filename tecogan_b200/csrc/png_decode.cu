// PNG decoder for a batch of files, byte-identical to cv2.imread(path, IMREAD_COLOR) on the subset it accepts:
// DESIGN.md section 4.7.  The host (tecogan_b200/png.py) walks the chunks, checks every CRC and routes each file; the
// device inflates, unfilters and expands the files it was given and reports per file whether the stream decoded
// exactly.  Any status but PNGD_OK means the caller decodes that file with cv2 instead.
//
// Stages (all on the caller's stream, nothing allocated):
//   png_inflate   one warp per file: the zlib header, every deflate block (Huffman tables built by the warp in shared
//                 memory, symbols decoded in lock step by all lanes, copies and literal runs written by the whole warp),
//                 the exact length, the Adler-32 of the inflated bytes.  Output: the filtered rows in the workspace.
//   png_unfilter  one CTA per file, rows in order: None / Up in parallel, Sub as a per-channel byte-lane scan,
//                 Avg / Paeth on one thread per byte of a pixel.  In place in the workspace.
//   png_expand    per file and row: grey, grey + alpha, RGB, RGBA and palette pixels to RGB at the destination.
#include "teco_common.cuh"

namespace {

// Descriptor columns (int64 [nfiles, PNGD_COLS], device memory), and status codes: include/teco.h.
enum { D_SRC_OFF, D_SRC_LEN, D_H, D_W, D_COLOUR, D_DEPTH, D_PLTE_OFF, D_PLTE_N, D_DST_OFF, D_DST_PITCH, D_WS_OFF, D_COLS };
enum {
  S_OK = 0, S_HEADER = 1, S_BLOCK = 2, S_CODE = 3, S_SYMBOL = 4, S_DISTANCE = 5, S_TRUNCATED = 6, S_OVERRUN = 7,
  S_SHORT = 8, S_ADLER = 9, S_TRAILING = 10, S_FILTER = 11, S_PALETTE = 12, S_DESC = 13
};

constexpr int MAX_DIM = 65500;
constexpr int FAST = 10;                                // primary Huffman table: 2^10 entries, longer codes walk counts
constexpr int INFLATE_WARPS = 4;
constexpr int UNFILTER_T = 256;
constexpr int EXPAND_T = 256, EXPAND_ROWS = 64;
constexpr uint32_t ADLER_MOD = 65521;

__constant__ uint16_t c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                        31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,   65,    97,    129,
                                         193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t c_cl_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__host__ __device__ inline int channels_of(int colour) {
  return colour == 2 ? 3 : colour == 4 ? 2 : colour == 6 ? 4 : 1;
}
// The accepted (colour type, bit depth) pairs: DESIGN.md section 4.7.
__host__ __device__ inline bool format_ok(long long colour, long long depth) {
  if (colour == 2 || colour == 4 || colour == 6) return depth == 8;
  if (colour == 0 || colour == 3) return depth == 1 || depth == 2 || depth == 4 || depth == 8;
  return false;
}
__host__ __device__ inline long long row_bytes(long long W, int colour, int depth) {
  return (W * channels_of(colour) * depth + 7) / 8;
}
__host__ __device__ inline long long filtered_bytes(long long H, long long W, int colour, int depth) {
  return H * (row_bytes(W, colour, depth) + 1);
}

// One Huffman code: the primary table (symbol << 4 | length; length 0: longer than FAST bits or unused) and the
// canonical counts and sorted symbols the longer codes are decoded from.
struct Huff {
  uint16_t fast[1 << FAST];
  uint16_t count[16];
  uint16_t sym[288];
};

struct WarpSmem {
  Huff lit, dist;
  uint8_t lens[32 + 286 + 30];                          // [0, 32): fixed or code-length lengths; [32, ..): a block's
  uint16_t offs[16], first[16];
};

// LSB-first bit reader over src[0, len): every lane of the warp holds the same state and reads the same bytes.
struct Bits {
  const uint8_t* src;
  long long len, pos;                                   // next byte to load
  uint64_t acc;
  int nb;
  __device__ void refill() {
    while (nb <= 56 && pos < len) { acc |= (uint64_t)src[pos++] << nb; nb += 8; }
  }
  // n <= 32 bits, or false when the stream ends first.
  __device__ bool get(int n, uint32_t* v) {
    if (nb < n) refill();
    if (nb < n) return false;
    *v = (uint32_t)(acc & ((1ull << n) - 1));
    acc >>= n;
    nb -= n;
    return true;
  }
  // Drop to the next byte boundary; the byte position of the next unread byte.
  __device__ long long align() {
    const int drop = nb & 7;
    acc >>= drop;
    nb -= drop;
    const long long p = pos - nb / 8;
    pos = p; acc = 0; nb = 0;
    return p;
  }
};

// Builds h from lens[0, n) with the whole warp.  `whole`: the code must be complete (zlib's rule for the literal /
// length and code-length codes); otherwise an incomplete code is taken only as a single code of length 1 or no code at
// all (zlib's rule for distances).  Returns false for an over-subscribed or refused incomplete code.
__device__ bool build_huff(Huff& h, const uint8_t* lens, int n, bool whole, WarpSmem& s, int lane) {
  for (int i = lane; i < (1 << FAST); i += 32) h.fast[i] = 0;
  __shared__ int ok_flag[INFLATE_WARPS];
  const int w = threadIdx.x >> 5;
  if (lane == 0) {
    int cnt[16];
    for (int l = 0; l < 16; ++l) cnt[l] = 0;
    for (int i = 0; i < n; ++i) ++cnt[lens[i]];
    cnt[0] = 0;
    int left = 1, ok = 1;
    for (int l = 1; l < 16; ++l) {
      left = (left << 1) - cnt[l];
      if (left < 0) ok = 0;
    }
    int used = 0, maxl = 0;
    for (int l = 1; l < 16; ++l) { used += cnt[l]; if (cnt[l]) maxl = l; }
    if (ok && left > 0) {
      if (whole) ok = 0;
      else if (!(used == 0 || (used == 1 && maxl == 1))) ok = 0;
    }
    int off = 0, code = 0;
    for (int l = 1; l < 16; ++l) {
      h.count[l] = (uint16_t)cnt[l];
      s.offs[l] = (uint16_t)off;
      code = (code + cnt[l - 1]) << 1;                  // RFC 1951 3.2.2: the first code of length l
      s.first[l] = (uint16_t)code;
      off += cnt[l];
    }
    h.count[0] = 0;
    int next[16];
    for (int l = 1; l < 16; ++l) next[l] = s.offs[l];
    for (int i = 0; i < n; ++i)
      if (lens[i]) h.sym[next[lens[i]]++] = (uint16_t)i;
    ok_flag[w] = ok;
  }
  __syncwarp();
  const int ok = ok_flag[w];
  if (!ok) return false;
  int total = 0;
  for (int l = 1; l < 16; ++l) total += h.count[l];
  for (int j = lane; j < total; j += 32) {
    const int sy = h.sym[j], l = lens[sy];
    if (l > FAST) continue;
    const uint32_t code = s.first[l] + (uint32_t)(j - s.offs[l]);
    const uint32_t rev = __brev(code) >> (32 - l);
    const uint16_t e = (uint16_t)((sy << 4) | l);
    for (uint32_t k = rev; k < (1u << FAST); k += 1u << l) h.fast[k] = e;
  }
  __syncwarp();
  return true;
}

// One symbol of h, or -1 (a bit pattern outside the code), or -2 (the stream ends inside the code).
__device__ int decode_sym(const Huff& h, Bits& b) {
  if (b.nb < 15) b.refill();
  const uint32_t e = h.fast[b.acc & ((1u << FAST) - 1)];
  int l = e & 15, sy;
  if (l) {
    sy = e >> 4;
  } else {                                              // canonical walk, one bit at a time (zlib's puff)
    int code = 0, first = 0, index = 0;
    sy = -1;
    for (l = 1; l < 16; ++l) {
      code |= (int)((b.acc >> (l - 1)) & 1);
      const int count = h.count[l];
      if (code - count < first) { sy = h.sym[index + (code - first)]; break; }
      index += count;
      first = (first + count) << 1;
      code <<= 1;
    }
    if (sy < 0) return b.nb < 15 ? -2 : -1;
  }
  if (l > b.nb) return -2;
  b.acc >>= l;
  b.nb -= l;
  return sy;
}

__device__ void fixed_lens(WarpSmem& s, int lane, bool dist) {
  if (!dist)
    for (int i = lane; i < 288; i += 32) s.lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
  else
    for (int i = lane; i < 32; i += 32) s.lens[i] = 5;
  __syncwarp();
}

// Inflates file f's stream into ws + ws_off; returns a status.  All lanes run it in lock step.
__device__ int inflate_file(const uint8_t* src, const long long* d, uint8_t* out, long long F, WarpSmem& s, int lane) {
  Bits b{src + d[D_SRC_OFF], d[D_SRC_LEN], 0, 0, 0};
  uint32_t cmf, flg;
  if (!b.get(8, &cmf) || !b.get(8, &flg)) return S_TRUNCATED;
  if ((cmf & 15) != 8 || (cmf >> 4) > 7 || ((cmf << 8) | flg) % 31 != 0 || (flg & 32)) return S_HEADER;
  const long long window = 1ll << ((cmf >> 4) + 8);
  long long o = 0;                                       // bytes written
  uint32_t last = 0;
  do {
    uint32_t type;
    if (!b.get(1, &last) || !b.get(2, &type)) return S_TRUNCATED;
    if (type == 0) {                                     // stored
      const long long p = b.align();
      if (p + 4 > b.len) return S_TRUNCATED;
      const uint8_t* q = b.src + p;
      const uint32_t n = q[0] | (q[1] << 8), nn = q[2] | (q[3] << 8);
      if (n != (~nn & 0xFFFFu)) return S_BLOCK;
      if (p + 4 + n > b.len) return S_TRUNCATED;
      if (o + n > F) return S_OVERRUN;
      for (uint32_t k = lane; k < n; k += 32) out[o + k] = q[4 + k];
      o += n;
      b.pos = p + 4 + n;
      __syncwarp();
      continue;
    }
    if (type == 3) return S_BLOCK;
    if (type == 1) {
      fixed_lens(s, lane, false);
      build_huff(s.lit, s.lens, 288, true, s, lane);
      fixed_lens(s, lane, true);
      build_huff(s.dist, s.lens, 32, true, s, lane);
    } else {                                             // dynamic: the code-length code, then both codes' lengths
      uint32_t hlit, hdist, hclen;
      if (!b.get(5, &hlit) || !b.get(5, &hdist) || !b.get(4, &hclen)) return S_TRUNCATED;
      const int nlen = hlit + 257, ndist = hdist + 1, ncl = hclen + 4;
      if (nlen > 286 || ndist > 30) return S_CODE;
      if (lane < 19) s.lens[lane] = 0;
      __syncwarp();
      for (int i = 0; i < ncl; ++i) {
        uint32_t v;
        if (!b.get(3, &v)) return S_TRUNCATED;
        if (lane == 0) s.lens[c_cl_order[i]] = (uint8_t)v;
      }
      __syncwarp();
      if (!build_huff(s.dist, s.lens, 19, true, s, lane)) return S_CODE;   // the code-length code, in dist's slot
      uint8_t lens_prev = 0;
      int i = 0;
      __syncwarp();
      while (i < nlen + ndist) {
        const int sy = decode_sym(s.dist, b);
        if (sy == -2) return S_TRUNCATED;
        if (sy < 0) return S_CODE;
        int rep = 1;
        uint8_t v = (uint8_t)sy;
        if (sy == 16) {
          uint32_t x;
          if (i == 0) return S_CODE;
          if (!b.get(2, &x)) return S_TRUNCATED;
          rep = 3 + x; v = lens_prev;
        } else if (sy == 17) {
          uint32_t x;
          if (!b.get(3, &x)) return S_TRUNCATED;
          rep = 3 + x; v = 0;
        } else if (sy == 18) {
          uint32_t x;
          if (!b.get(7, &x)) return S_TRUNCATED;
          rep = 11 + x; v = 0;
        }
        if (i + rep > nlen + ndist) return S_CODE;
        if (lane == 0) for (int k = 0; k < rep; ++k) s.lens[32 + i + k] = v;   // lens[32..]: out of build_huff's way
        i += rep;
        lens_prev = v;
      }
      __syncwarp();
      if (s.lens[32 + 256] == 0) return S_CODE;          // no end-of-block code
      if (!build_huff(s.lit, s.lens + 32, nlen, true, s, lane)) return S_CODE;
      if (!build_huff(s.dist, s.lens + 32 + nlen, ndist, false, s, lane)) return S_CODE;
    }
    // Literals collect in lane registers (lane k holds the k-th of a run) and are written 32 at a time.
    int nlit = 0;
    uint8_t mine = 0;
    for (;;) {
      const int sy = decode_sym(s.lit, b);
      if (sy == -2) return S_TRUNCATED;
      if (sy < 0) return S_SYMBOL;
      if (sy < 256) {
        if (lane == nlit) mine = (uint8_t)sy;
        if (++nlit == 32) {
          if (o + 32 > F) return S_OVERRUN;
          out[o + lane] = mine;
          o += 32;
          nlit = 0;
          __syncwarp();
        }
        continue;
      }
      if (nlit) {
        if (o + nlit > F) return S_OVERRUN;
        if (lane < nlit) out[o + lane] = mine;
        o += nlit;
        nlit = 0;
        __syncwarp();
      }
      if (sy == 256) break;
      if (sy > 285) return S_SYMBOL;
      uint32_t x;
      const int li = sy - 257;
      if (!b.get(c_len_extra[li], &x)) return S_TRUNCATED;
      const int len = c_len_base[li] + (int)x;
      const int ds = decode_sym(s.dist, b);
      if (ds == -2) return S_TRUNCATED;
      if (ds < 0 || ds > 29) return S_SYMBOL;
      if (!b.get(c_dist_extra[ds], &x)) return S_TRUNCATED;
      const long long dist = c_dist_base[ds] + (long long)x;
      if (dist > o || dist > window) return S_DISTANCE;
      if (o + len > F) return S_OVERRUN;
      // out[o + k] = out[o - dist + k mod dist]: every source byte precedes o, so lanes copy independently.
      for (int k = lane; k < len; k += 32) out[o + k] = out[o - dist + (dist >= len ? k : k % dist)];
      o += len;
      __syncwarp();
    }
  } while (!last);
  if (o != F) return S_SHORT;
  const long long p = b.align();
  if (p + 4 > b.len) return S_TRUNCATED;
  const uint8_t* q = b.src + p;
  const uint32_t want = ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3];
  // Adler-32 of out[0, F): a = 1 + sum x_i, b = F + sum (F - i) x_i, both mod 65521; lanes take 4 KiB pieces.
  unsigned long long sa = 0, sb = 0;
  for (long long c0 = (long long)lane * 4096; c0 < F; c0 += 32 * 4096) {
    const long long c1 = min(F, c0 + 4096);
    unsigned long long ta = 0, tb = 0;
    uint32_t wt = (uint32_t)((F - c0) % ADLER_MOD);     // (F - i) mod 65521, stepped down with i
    for (long long i = c0; i < c1; ++i) {
      const uint32_t v = out[i];
      ta += v;
      tb += (unsigned long long)wt * v;
      wt = wt ? wt - 1 : ADLER_MOD - 1;
    }
    sa += ta % ADLER_MOD;
    sb += tb % ADLER_MOD;
  }
#pragma unroll
  for (int k = 16; k > 0; k >>= 1) {
    sa += __shfl_xor_sync(0xffffffffu, sa, k);
    sb += __shfl_xor_sync(0xffffffffu, sb, k);
  }
  const uint32_t a = (uint32_t)((1 + sa) % ADLER_MOD), bb = (uint32_t)((F % ADLER_MOD + sb) % ADLER_MOD);
  if (((bb << 16) | a) != want) return S_ADLER;
  if (p + 4 != b.len) return S_TRAILING;
  return S_OK;
}

// The descriptor's ranges lie inside the buffers and its format is one the decoder takes.
__device__ bool desc_ok(const long long* d, long long src_bytes, long long ws_bytes, long long dst_bytes) {
  const long long H = d[D_H], W = d[D_W], colour = d[D_COLOUR], depth = d[D_DEPTH];
  if (H < 1 || W < 1 || H > MAX_DIM || W > MAX_DIM || !format_ok(colour, depth)) return false;
  if (d[D_SRC_OFF] < 0 || d[D_SRC_LEN] < 0 || d[D_SRC_OFF] + d[D_SRC_LEN] > src_bytes) return false;
  if (d[D_WS_OFF] < 0 || d[D_WS_OFF] + filtered_bytes(H, W, (int)colour, (int)depth) > ws_bytes) return false;
  if (d[D_DST_OFF] < 0 || d[D_DST_PITCH] < 3 * W || d[D_DST_OFF] + (H - 1) * d[D_DST_PITCH] + 3 * W > dst_bytes) return false;
  if (colour == 3 && (d[D_PLTE_N] < 1 || d[D_PLTE_N] > 256 || d[D_PLTE_OFF] < 0 || d[D_PLTE_OFF] + 3 * d[D_PLTE_N] > src_bytes))
    return false;
  return true;
}

__global__ void __launch_bounds__(32 * INFLATE_WARPS) png_inflate(const uint8_t* __restrict__ src, long long src_bytes,
                                                                  const long long* __restrict__ desc, int nfiles,
                                                                  uint8_t* ws, long long ws_bytes, long long dst_bytes,
                                                                  int* status) {
  __shared__ WarpSmem smem[INFLATE_WARPS];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int f = blockIdx.x * INFLATE_WARPS + w;
  if (f >= nfiles) return;
  const long long* d = desc + (long long)f * D_COLS;
  int st;
  if (!desc_ok(d, src_bytes, ws_bytes, dst_bytes)) {
    st = S_DESC;
  } else {
    const long long F = filtered_bytes(d[D_H], d[D_W], (int)d[D_COLOUR], (int)d[D_DEPTH]);
    st = inflate_file(src, d, ws + d[D_WS_OFF], F, smem[w], lane);
  }
  if (lane == 0) status[f] = st;
}

// Inclusive scan of 4-byte lanes (each byte its own sum mod 256) over the CTA.
__device__ uint32_t cta_scan_vadd4(uint32_t v, uint32_t* sm, uint32_t* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int k = 1; k < 32; k <<= 1) {
    const uint32_t u = __shfl_up_sync(0xffffffffu, v, k);
    if (lane >= k) v = __vadd4(v, u);
  }
  if (lane == 31) sm[w] = v;
  __syncthreads();
  if (w == 0) {
    uint32_t t = lane < UNFILTER_T / 32 ? sm[lane] : 0u;
#pragma unroll
    for (int k = 1; k < 32; k <<= 1) {
      const uint32_t u = __shfl_up_sync(0xffffffffu, t, k);
      if (lane >= k) t = __vadd4(t, u);
    }
    if (lane < UNFILTER_T / 32) sm[32 + lane] = t;
  }
  __syncthreads();
  if (w > 0) v = __vadd4(v, sm[32 + w - 1]);
  *total = sm[32 + UNFILTER_T / 32 - 1];
  __syncthreads();
  return v;
}

__device__ __forceinline__ uint32_t load_px(const uint8_t* p, int bpp) {
  uint32_t v = 0;
  for (int c = 0; c < bpp; ++c) v |= (uint32_t)p[c] << (8 * c);
  return v;
}
__device__ __forceinline__ void store_px(uint8_t* p, uint32_t v, int bpp) {
  for (int c = 0; c < bpp; ++c) p[c] = (uint8_t)(v >> (8 * c));
}

__device__ __forceinline__ uint8_t paeth(int a, int b, int c) {
  const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (uint8_t)(pa <= pb && pa <= pc ? a : pb <= pc ? b : c);
}

// Rows in order (each filter but None and Sub reads the row above): one CTA per file.
__global__ void __launch_bounds__(UNFILTER_T) png_unfilter(const long long* __restrict__ desc, uint8_t* ws, int* status) {
  __shared__ uint32_t sm[64];
  const int f = blockIdx.x;
  if (status[f] != S_OK) return;
  const long long* d = desc + (long long)f * D_COLS;
  const int colour = (int)d[D_COLOUR], depth = (int)d[D_DEPTH];
  const long long H = d[D_H], rb = row_bytes(d[D_W], colour, depth);
  const int bpp = max(1, channels_of(colour) * depth / 8);
  uint8_t* img = ws + d[D_WS_OFF];
  const int t = threadIdx.x;
  for (long long y = 0; y < H; ++y) {
    uint8_t* cur = img + y * (rb + 1) + 1;
    const uint8_t* up = y ? cur - (rb + 1) : nullptr;
    const int ft = cur[-1];
    if (ft > 4) {
      if (t == 0) status[f] = S_FILTER;
      return;
    }
    if (ft == 2 && up) {
      for (long long i = t; i < rb; i += UNFILTER_T) cur[i] = (uint8_t)(cur[i] + up[i]);
    } else if (ft == 1) {                                // per-channel prefix sums of whole pixels
      const long long npx = rb / bpp;                    // rb is a multiple of bpp when bpp > 1
      const long long per = (npx + UNFILTER_T - 1) / UNFILTER_T, p0 = t * per, p1 = min(npx, p0 + per);
      uint32_t sum = 0;
      for (long long p = p0; p < p1; ++p) sum = __vadd4(sum, load_px(cur + p * bpp, bpp));
      uint32_t total;
      uint32_t run = cta_scan_vadd4(sum, sm, &total);
      run = __vsub4(run, sum);                           // exclusive
      for (long long p = p0; p < p1; ++p) {
        run = __vadd4(run, load_px(cur + p * bpp, bpp));
        store_px(cur + p * bpp, run, bpp);
      }
    } else if (ft == 3 || ft == 4) {                     // sequential along the row, one thread per byte of a pixel
      if (t < bpp) {
        int left = 0, upleft = 0;
        for (long long i = t; i < rb; i += bpp) {
          const int above = up ? up[i] : 0;
          const int pred = ft == 3 ? (left + above) >> 1 : paeth(left, above, upleft);
          left = (uint8_t)(cur[i] + pred);
          cur[i] = (uint8_t)left;
          upleft = above;
        }
      }
    }
    __syncthreads();
  }
}

// Unfiltered rows -> RGB at dst + dst_off, row pitch dst_pitch.
__global__ void __launch_bounds__(EXPAND_T) png_expand(const uint8_t* __restrict__ src, const long long* __restrict__ desc,
                                                       const uint8_t* __restrict__ ws, uint8_t* dst, int* status) {
  const int f = blockIdx.x;
  if (status[f] != S_OK) return;
  const long long* d = desc + (long long)f * D_COLS;
  const int colour = (int)d[D_COLOUR], depth = (int)d[D_DEPTH];
  const long long H = d[D_H], W = d[D_W], rb = row_bytes(W, colour, depth), pitch = d[D_DST_PITCH];
  const int nplte = (int)d[D_PLTE_N];
  const uint8_t* plte = src + d[D_PLTE_OFF];
  const int maxv = (1 << depth) - 1, scale = 255 / maxv;  // grey below 8 bits: 0..2^d - 1 onto 0..255
  bool bad = false;
  for (long long y = blockIdx.y; y < H; y += gridDim.y) {
    const uint8_t* row = ws + d[D_WS_OFF] + y * (rb + 1) + 1;
    uint8_t* o = dst + d[D_DST_OFF] + y * pitch;
    for (long long x = threadIdx.x; x < W; x += EXPAND_T) {
      uint8_t r, g, b;
      if (colour == 2) {
        r = row[3 * x]; g = row[3 * x + 1]; b = row[3 * x + 2];
      } else if (colour == 6) {
        r = row[4 * x]; g = row[4 * x + 1]; b = row[4 * x + 2];
      } else if (colour == 4) {
        r = g = b = row[2 * x];
      } else {
        const long long bit = x * depth;
        const int v = (row[bit >> 3] >> (8 - depth - (int)(bit & 7))) & maxv;
        if (colour == 0) {
          r = g = b = (uint8_t)(v * scale);
        } else {
          if (v >= nplte) { bad = true; continue; }
          r = plte[3 * v]; g = plte[3 * v + 1]; b = plte[3 * v + 2];
        }
      }
      o[3 * x] = r; o[3 * x + 1] = g; o[3 * x + 2] = b;
    }
  }
  if (bad) status[f] = S_PALETTE;
}

}  // namespace

extern "C" {

int teco_png_decode_plan_bytes(int32_t H, int32_t W, int32_t colour, int32_t depth, int64_t* workspace_bytes_host) {
  TECO_CHECK_ARG(workspace_bytes_host, "teco_png_decode_plan_bytes: NULL argument");
  TECO_CHECK_ARG(H >= 1 && W >= 1 && H <= MAX_DIM && W <= MAX_DIM,
                 "teco_png_decode_plan_bytes: bad frame size %dx%d (1 <= H, W <= %d)", H, W, MAX_DIM);
  TECO_CHECK_ARG(format_ok(colour, depth), "teco_png_decode_plan_bytes: colour type %d at bit depth %d is not decoded on "
                 "the device", colour, depth);
  *workspace_bytes_host = (filtered_bytes(H, W, colour, depth) + 255) & ~255ll;
  return TECO_OK;
}

int teco_png_decode_rgb8(const uint8_t* src, int64_t src_bytes, const int64_t* desc, int32_t nfiles, void* workspace,
                         int64_t workspace_bytes, uint8_t* dst, int64_t dst_bytes, int32_t* status, void* stream) {
  TECO_CHECK_ARG(src && desc && workspace && dst && status, "teco_png_decode_rgb8: NULL argument");
  TECO_CHECK_ARG(nfiles >= 1 && nfiles <= (1 << 24), "teco_png_decode_rgb8: %d files (1 .. 2^24)", nfiles);
  TECO_CHECK_ARG(src_bytes >= 0 && workspace_bytes >= 0 && dst_bytes >= 0, "teco_png_decode_rgb8: negative buffer size");
  const cudaStream_t st = (cudaStream_t)stream;
  const long long* dd = reinterpret_cast<const long long*>(desc);
  png_inflate<<<(nfiles + INFLATE_WARPS - 1) / INFLATE_WARPS, 32 * INFLATE_WARPS, 0, st>>>(
      src, src_bytes, dd, nfiles, (uint8_t*)workspace, workspace_bytes, dst_bytes, status);
  png_unfilter<<<nfiles, UNFILTER_T, 0, st>>>(dd, (uint8_t*)workspace, status);
  png_expand<<<dim3(nfiles, EXPAND_ROWS), EXPAND_T, 0, st>>>(src, dd, (const uint8_t*)workspace, dst, status);
  TECO_CUDA_LAUNCH_CHECK("teco_png_decode_rgb8");
  return TECO_OK;
}

}  // extern "C"
