// PNG encoder for RGB uint8 frames, byte-identical to cv2.imwrite (libpng, zlib level 1, Z_RLE): DESIGN.md section 4.5.
//
// S = the filtered image: per row the filter byte (1 = Sub; 0 = None for rows of width 1) and the byte differences.
// Z_RLE deflate of S: every maximal run of equal bytes is a literal followed by distance-1 matches of 258 and one
// match of the remainder when it is at least 3 (else literals); a block ends after every 16 383 symbols and after the
// last.  Each block is coded stored, static or dynamic, whichever is shortest, with zlib's Huffman construction.
// tests/golden/png_oracle.py states every stage on the host; tests/test_png_host.py pins it to cv2 and zlib.
//
// Stages (one kernel each, all on the caller's stream, sizes read from the device where the host cannot know them):
//   png_filter          S, run starts per tile, Adler-32 partial sums per tile, zeroes the zlib buffer
//   png_scan            exclusive scan of per-tile counts (runs, then tokens); Adler-32 of S
//   png_runs            start position of every run
//   png_run_tokens      tokens per run, summed per tile   | then png_scan
//   png_token_offsets   first token of every run
//   png_tokens          every token (literal byte or match length) and the S position of every block start
//   png_block_trees     per deflate block: histogram, zlib's trees, block type, the dynamic header's bits
//   png_block_offsets   one thread: each block's bit offset (a stored block's padding depends on it), zlib header,
//                       Adler-32, the file length
//   png_emit            per block: the header, the tokens at scanned bit offsets OR-ed into 32-bit words, stored bytes
//   png_assemble        per IDAT chunk: length, tag, data, CRC-32 (segment CRCs combined); signature, IHDR, IEND
#include "teco_common.cuh"

namespace {

constexpr int TILE = 4096, TILE_T = 256, TILE_V = TILE / TILE_T;   // scan tiles: 256 threads x 16 items
constexpr int BLOCK_SYMS = 16383;                                  // zlib's literal buffer (16 384) minus one
constexpr int EMIT_T = 512, EMIT_V = 32;                           // 512 x 32 >= BLOCK_SYMS tokens per block
constexpr int IDAT = 8192;
constexpr int L_CODES = 286, D_CODES = 30, BL_CODES = 19, END_BLOCK = 256, CODE_STRIDE = 288, DIST0 = 286;
constexpr int HEAP = 2 * L_CODES + 1;
constexpr int HDR_WORDS = 144;            // 14 + 19*3 + 316 * (7 + 7) = 4 495 bits at most
constexpr int KIND_STORED = 0, KIND_STATIC = 1, KIND_DYNAMIC = 2;
constexpr uint32_t ADLER_MOD = 65521;

__constant__ uint8_t c_len_base[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                       31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 0 /* 258 */};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint8_t c_bl_order[BL_CODES] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// Match length 3..258 -> index 0..28 of its length code (257 + index); 258 has its own code.
__device__ __forceinline__ int len_index(int len) {
  if (len == 258) return 28;
  int i = 0;
#pragma unroll 1
  while (i < 27 && c_len_base[i + 1] <= len) ++i;
  return i;
}
__device__ __forceinline__ int static_llen(int n) { return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8; }

// Workspace layout, from H and W alone (the host sizes it, the kernels carve it the same way).
struct Plan {
  long long L;            // bytes of S
  int ntile;              // scan tiles over S (and over runs, tokens: each is at most L)
  int zwords;             // 32-bit words of the zlib buffer
  int maxblk;             // deflate blocks at most
  int maxchunk;           // IDAT chunks at most
  long long zcap, out_cap, ws_bytes;
  long long off_s, off_r, off_o, off_tok, off_z, off_bstart, off_tiles, off_meta, off_blk, off_boff, off_code, off_hdr;
};

__host__ __device__ inline long long align256(long long x) { return (x + 255) & ~255ll; }

__host__ __device__ inline Plan make_plan(int H, int W) {
  Plan p;
  p.L = (long long)H * (3ll * W + 1);
  p.ntile = (int)((p.L + TILE - 1) / TILE);
  p.maxblk = (int)(p.L / BLOCK_SYMS) + 1;
  // A block is never longer than its stored form (5 bytes + its bytes), + zlib header, trailer and a spare word.
  p.zcap = p.L + 5ll * p.maxblk + 2 + 4 + 8;
  p.zwords = (int)((p.zcap + 3) / 4);
  p.zcap = 4ll * p.zwords;
  p.maxchunk = (int)((p.zcap + IDAT - 1) / IDAT);
  p.out_cap = 8 + 25 + p.zcap + 12ll * p.maxchunk + 12;
  long long o = 0;
  p.off_s = o;      o = align256(o + p.L + 16);
  p.off_r = o;      o = align256(o + 4 * (p.L + 1));
  p.off_o = o;      o = align256(o + 4 * (p.L + 1));
  p.off_tok = o;    o = align256(o + 2 * p.L);
  p.off_z = o;      o = align256(o + 4ll * p.zwords);
  p.off_bstart = o; o = align256(o + 4ll * (p.maxblk + 1));
  p.off_tiles = o;  o = align256(o + 4ll * 6 * p.ntile);     // run counts/offsets, token counts/offsets, Adler a/b
  p.off_meta = o;   o = align256(o + 8ll * 8);
  p.off_blk = o;    o = align256(o + 4ll * 4 * p.maxblk);    // kind, bits, header bits, stored length
  p.off_boff = o;   o = align256(o + 8ll * p.maxblk);        // bit offset of each block in the zlib stream
  p.off_code = o;   o = align256(o + 4ll * CODE_STRIDE * p.maxblk);   // (code << 8) | length per symbol
  p.off_hdr = o;    o = align256(o + 4ll * HDR_WORDS * p.maxblk);
  p.ws_bytes = o;
  return p;
}

// meta[]: the sizes only the device knows
enum { M_RUNS = 0, M_TOKENS = 1, M_BLOCKS = 2, M_ZLEN = 3, M_ADLER = 4 };

struct Bufs {
  uint8_t* s;
  int *r, *o;
  uint16_t* tok;
  uint32_t* z;
  int* bstart;
  int *run_cnt, *run_off, *tok_cnt, *tok_off;
  uint32_t *ad_a, *ad_b;
  long long* meta;
  int *kind, *bits, *hdr_bits, *stored;
  long long* boff;
  uint32_t* code;
  uint32_t* hdr;
};

inline Bufs carve(const Plan& p, void* ws) {
  uint8_t* b = (uint8_t*)ws;
  Bufs u;
  u.s = b + p.off_s;
  u.r = (int*)(b + p.off_r);
  u.o = (int*)(b + p.off_o);
  u.tok = (uint16_t*)(b + p.off_tok);
  u.z = (uint32_t*)(b + p.off_z);
  u.bstart = (int*)(b + p.off_bstart);
  int* t = (int*)(b + p.off_tiles);
  u.run_cnt = t; u.run_off = t + p.ntile; u.tok_cnt = t + 2 * p.ntile; u.tok_off = t + 3 * p.ntile;
  u.ad_a = (uint32_t*)(t + 4 * p.ntile); u.ad_b = (uint32_t*)(t + 5 * p.ntile);
  u.meta = (long long*)(b + p.off_meta);
  int* k = (int*)(b + p.off_blk);
  u.kind = k; u.bits = k + p.maxblk; u.hdr_bits = k + 2 * p.maxblk; u.stored = k + 3 * p.maxblk;
  u.boff = (long long*)(b + p.off_boff);
  u.code = (uint32_t*)(b + p.off_code);
  u.hdr = (uint32_t*)(b + p.off_hdr);
  return u;
}

// Byte i of S, straight from the frame.
__device__ __forceinline__ uint8_t s_byte(const uint8_t* __restrict__ rgb, long long i, int W, long long row) {
  const long long y = i / row, c = i - y * row;
  if (c == 0) return W > 1 ? 1 : 0;
  const uint8_t* p = rgb + y * (row - 1) + (c - 1);
  return (W > 1 && c > 3) ? (uint8_t)(p[0] - p[-3]) : p[0];
}

// ------------------------------------------------------------------------------------------------ filter
__global__ void __launch_bounds__(TILE_T) png_filter(const uint8_t* __restrict__ rgb, int W, Plan p, Bufs u) {
  __shared__ int sm[TILE_T / 32 + 1];
  __shared__ unsigned long long sa[TILE_T / 32], sb[TILE_T / 32];
  const long long row = 3ll * W + 1;
  const long long z0 = (long long)blockIdx.x * (TILE / 4);
  for (int k = threadIdx.x; k < TILE / 4; k += TILE_T)
    if (z0 + k < p.zwords) u.z[z0 + k] = 0u;
  if (blockIdx.x >= p.ntile) return;
  const long long i0 = (long long)blockIdx.x * TILE + threadIdx.x * TILE_V;
  int runs = 0;
  unsigned long long a = 0, b = 0;
  uint8_t prev = i0 > 0 && i0 < p.L ? s_byte(rgb, i0 - 1, W, row) : 0;
#pragma unroll 4
  for (int k = 0; k < TILE_V; ++k) {
    const long long i = i0 + k;
    if (i >= p.L) break;
    const uint8_t v = s_byte(rgb, i, W, row);
    u.s[i] = v;
    runs += (i == 0 || v != prev);
    prev = v;
    a += v;
    b += (unsigned long long)(p.L - i) * v;          // Adler-32's b = L + sum (L - i) S_i
  }
  int total;
  cta_exclusive_scan<TILE_T>(runs, sm, &total);
  a %= ADLER_MOD;
  b %= ADLER_MOD;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, d);
    b += __shfl_xor_sync(0xffffffffu, b, d);
  }
  if ((threadIdx.x & 31) == 0) { sa[threadIdx.x >> 5] = a; sb[threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long ta = 0, tb = 0;
    for (int w = 0; w < TILE_T / 32; ++w) { ta += sa[w]; tb += sb[w]; }
    u.run_cnt[blockIdx.x] = total;
    u.ad_a[blockIdx.x] = (uint32_t)(ta % ADLER_MOD);
    u.ad_b[blockIdx.x] = (uint32_t)(tb % ADLER_MOD);
  }
}

// ------------------------------------------------------------------------------------------------ tile scan
// One CTA: off[t] = sum of cnt[0..t), meta[slot] = the total.  With `adler`, also the Adler-32 of S into meta.
__global__ void __launch_bounds__(1024) png_scan(const int* __restrict__ cnt, int* __restrict__ off, int n, Plan p, Bufs u,
                                                 int slot, int adler) {
  __shared__ int sm[1024 / 32 + 1];
  __shared__ unsigned long long ra[32], rb[32];
  int carry = 0;
  for (int base = 0; base < n; base += 1024) {
    const int t = base + threadIdx.x;
    const int v = t < n ? cnt[t] : 0;
    int total;
    const int ex = cta_exclusive_scan<1024>(v, sm, &total);
    if (t < n) off[t] = carry + ex;
    carry += total;
  }
  if (threadIdx.x == 0) {
    u.meta[slot] = carry;
    if (slot == M_TOKENS) u.meta[M_BLOCKS] = carry / BLOCK_SYMS + 1;
  }
  if (!adler) return;
  unsigned long long a = 0, b = 0;
  for (int t = threadIdx.x; t < n; t += 1024) { a += u.ad_a[t]; b += u.ad_b[t]; }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, d);
    b += __shfl_xor_sync(0xffffffffu, b, d);
  }
  if ((threadIdx.x & 31) == 0) { ra[threadIdx.x >> 5] = a; rb[threadIdx.x >> 5] = b; }
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long ta = 1, tb = (unsigned long long)(p.L % ADLER_MOD);
    for (int w = 0; w < 32; ++w) { ta += ra[w]; tb += rb[w]; }
    u.meta[M_ADLER] = (long long)(((tb % ADLER_MOD) << 16) | (ta % ADLER_MOD));
  }
}

// ------------------------------------------------------------------------------------------------ runs, tokens
__global__ void __launch_bounds__(TILE_T) png_runs(Plan p, Bufs u) {
  __shared__ int sm[TILE_T / 32 + 1];
  if (blockIdx.x == 0 && threadIdx.x == 0) u.r[u.meta[M_RUNS]] = (int)p.L;
  const long long i0 = (long long)blockIdx.x * TILE + threadIdx.x * TILE_V;
  uint32_t flags = 0;
  int n = 0;
  for (int k = 0; k < TILE_V; ++k) {
    const long long i = i0 + k;
    if (i < p.L && (i == 0 || u.s[i] != u.s[i - 1])) { flags |= 1u << k; ++n; }
  }
  int total;
  int at = u.run_off[blockIdx.x] + cta_exclusive_scan<TILE_T>(n, sm, &total);
  for (int k = 0; k < TILE_V; ++k)
    if (flags >> k & 1) u.r[at++] = (int)(i0 + k);
}

__device__ __forceinline__ int run_tokens(int n) {
  const int tail = n - 1, rem = tail % 258;
  return 1 + tail / 258 + (rem >= 3 ? 1 : rem);
}

__global__ void __launch_bounds__(TILE_T) png_run_tokens(Bufs u) {
  __shared__ int sm[TILE_T / 32 + 1];
  const int nruns = (int)u.meta[M_RUNS];
  const int k0 = blockIdx.x * TILE + threadIdx.x * TILE_V;
  int t = 0;
  for (int k = k0; k < k0 + TILE_V && k < nruns; ++k) t += run_tokens(u.r[k + 1] - u.r[k]);
  int total;
  cta_exclusive_scan<TILE_T>(t, sm, &total);
  if (threadIdx.x == 0) u.tok_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(TILE_T) png_token_offsets(Bufs u) {
  __shared__ int sm[TILE_T / 32 + 1];
  const int nruns = (int)u.meta[M_RUNS];
  if (blockIdx.x == 0 && threadIdx.x == 0) u.o[nruns] = (int)u.meta[M_TOKENS];
  const int k0 = blockIdx.x * TILE + threadIdx.x * TILE_V;
  int cnt[TILE_V];
  int t = 0;
#pragma unroll
  for (int j = 0; j < TILE_V; ++j) {
    const int k = k0 + j;
    cnt[j] = k < nruns ? run_tokens(u.r[k + 1] - u.r[k]) : 0;
    t += cnt[j];
  }
  int total;
  int at = u.tok_off[blockIdx.x] + cta_exclusive_scan<TILE_T>(t, sm, &total);
#pragma unroll
  for (int j = 0; j < TILE_V; ++j) {
    if (k0 + j < nruns) u.o[k0 + j] = at;
    at += cnt[j];
  }
}

// One CTA per tile of 4 096 runs writes all their tokens: token -> run by binary search over the tile's offsets.
__global__ void __launch_bounds__(TILE_T) png_tokens(Plan p, Bufs u) {
  __shared__ int so[TILE + 1], sr[TILE + 1];
  const int nruns = (int)u.meta[M_RUNS], ntok = (int)u.meta[M_TOKENS];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const int nb = ntok / BLOCK_SYMS + 1;
    u.bstart[nb] = (int)p.L;
    if (ntok % BLOCK_SYMS == 0) u.bstart[nb - 1] = (int)p.L;   // the empty final block after an exact multiple
  }
  const int k0 = blockIdx.x * TILE;
  if (k0 >= nruns) return;
  const int nk = min(TILE, nruns - k0);
  for (int j = threadIdx.x; j <= nk; j += TILE_T) { so[j] = u.o[k0 + j]; sr[j] = u.r[k0 + j]; }
  __syncthreads();
  for (int t = so[0] + threadIdx.x; t < so[nk]; t += TILE_T) {
    int lo = 0, hi = nk - 1;                  // last j with so[j] <= t
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (so[mid] <= t) lo = mid; else hi = mid - 1;
    }
    const int m = t - so[lo], r = sr[lo], tail = sr[lo + 1] - r - 1;
    const int nfull = tail / 258, rem = tail % 258;
    int pos;
    uint16_t tk;
    if (m == 0) {
      pos = r;
      tk = u.s[r];
    } else if (m <= nfull) {
      pos = r + 1 + (m - 1) * 258;
      tk = 0x8000u | 258u;
    } else {
      pos = r + 1 + nfull * 258 + (m - nfull - 1);
      tk = rem >= 3 ? (uint16_t)(0x8000u | rem) : (uint16_t)u.s[r];
    }
    u.tok[t] = tk;
    if (t % BLOCK_SYMS == 0) u.bstart[t / BLOCK_SYMS] = pos;
  }
}

// ------------------------------------------------------------------------------------------------ Huffman trees
// zlib's construction (tests/golden/png_oracle.py: build_tree).  All arrays in shared memory, one thread.
struct TreeWork {
  int freq[HEAP], depth[HEAP], dad[HEAP], len[HEAP], heap[HEAP];
};

__device__ __forceinline__ bool smaller(const TreeWork& w, int a, int b) {
  return w.freq[a] < w.freq[b] || (w.freq[a] == w.freq[b] && w.depth[a] <= w.depth[b]);
}

__device__ void heap_down(TreeWork& w, int heap_len, int k) {
  const int v = w.heap[k];
  int j = k << 1;
  while (j <= heap_len) {
    if (j < heap_len && smaller(w, w.heap[j + 1], w.heap[j])) ++j;
    if (smaller(w, v, w.heap[j])) break;
    w.heap[k] = w.heap[j];
    k = j;
    j <<= 1;
  }
  w.heap[k] = v;
}

// freq[0..elems) in w.freq on entry; lengths in w.len[0..elems) on exit.  kind: 0 literal/length, 1 distance,
// 2 bit-length tree (no static code).  Returns max_code; adds to *opt and *stat.
__device__ int build_tree(TreeWork& w, int elems, int max_length, int kind, long long* opt, long long* stat) {
  const int nodes = 2 * elems + 1;
  int heap_len = 0, heap_max = nodes, max_code = -1;
  for (int n = 0; n < elems; ++n) {
    w.depth[n] = 0;
    if (w.freq[n]) w.heap[++heap_len] = max_code = n;
  }
  while (heap_len < 2) {
    const int node = max_code < 2 ? ++max_code : 0;
    w.heap[++heap_len] = node;
    w.freq[node] = 1;
    w.depth[node] = 0;
    *opt -= 1;
    if (kind == 0) *stat -= static_llen(node);
    if (kind == 1) *stat -= 5;
  }
  for (int k = heap_len / 2; k >= 1; --k) heap_down(w, heap_len, k);
  int node = elems;
  do {
    const int n = w.heap[1];
    w.heap[1] = w.heap[heap_len--];
    heap_down(w, heap_len, 1);
    const int m = w.heap[1];
    w.heap[--heap_max] = n;
    w.heap[--heap_max] = m;
    w.freq[node] = w.freq[n] + w.freq[m];
    w.depth[node] = max(w.depth[n], w.depth[m]) + 1;
    w.dad[n] = w.dad[m] = node;
    w.heap[1] = node++;
    heap_down(w, heap_len, 1);
  } while (heap_len >= 2);
  w.heap[--heap_max] = w.heap[1];

  int bl_count[16];
  for (int b = 0; b < 16; ++b) bl_count[b] = 0;
  int overflow = 0;
  w.len[w.heap[heap_max]] = 0;
  for (int h = heap_max + 1; h < nodes; ++h) {
    const int n = w.heap[h];
    int bits = w.len[w.dad[n]] + 1;
    if (bits > max_length) { bits = max_length; ++overflow; }
    w.len[n] = bits;
    if (n > max_code) continue;
    ++bl_count[bits];
    int xb = 0;
    if (kind == 0 && n >= 257) xb = c_len_extra[n - 257];
    if (kind == 2 && n >= 16) xb = n == 16 ? 2 : n == 17 ? 3 : 7;
    const long long f = w.freq[n];
    *opt += f * (bits + xb);
    if (kind == 0) *stat += f * (static_llen(n) + xb);
    if (kind == 1) *stat += f * 5;
  }
  if (overflow) {
    do {
      int bits = max_length - 1;
      while (bl_count[bits] == 0) --bits;
      --bl_count[bits];
      bl_count[bits + 1] += 2;
      --bl_count[max_length];
      overflow -= 2;
    } while (overflow > 0);
    int h = nodes;
    for (int bits = max_length; bits != 0; --bits) {
      int c = bl_count[bits];
      while (c != 0) {
        const int m = w.heap[--h];
        if (m > max_code) continue;
        if (w.len[m] != bits) {
          *opt += (long long)(bits - w.len[m]) * w.freq[m];
          w.len[m] = bits;
        }
        --c;
      }
    }
  }
  for (int n = 0; n < elems; ++n)
    if (w.freq[n] == 0 || n > max_code) w.len[n] = 0;
  return max_code;
}

// Canonical codes of lens[0..n), bit-reversed for LSB-first output: out[i] = (code << 8) | length.
__device__ void canonical(const int* lens, int n, uint32_t* out) {
  int count[16], next[16];
  for (int b = 0; b < 16; ++b) count[b] = 0;
  for (int i = 0; i < n; ++i) if (lens[i]) ++count[lens[i]];
  int code = 0;
  count[0] = 0;
  for (int b = 1; b < 16; ++b) { code = (code + count[b - 1]) << 1; next[b] = code; }
  for (int i = 0; i < n; ++i) {
    const int l = lens[i];
    out[i] = l ? ((__brev((uint32_t)next[l]++) >> (32 - l)) << 8) | (uint32_t)l : 0u;
  }
}

// Thread-private LSB-first bit writer into a plain word array.
struct BitWriter {
  uint32_t* w;
  int n;
  uint64_t acc;
  int nb;
  __device__ void put(uint32_t v, int bits) {
    acc |= (uint64_t)v << nb;
    nb += bits;
    while (nb >= 32) { w[n++] = (uint32_t)acc; acc >>= 32; nb -= 32; }
  }
  __device__ void flush() { if (nb) w[n++] = (uint32_t)acc; }
};

// The bit-length alphabet's run coding of lens[0..max_code] (tests/golden/png_oracle.py: length_runs): counts the
// symbols into blfreq, or with `bw` writes them using blcode.
__device__ void length_runs(const int* lens, int max_code, int* blfreq, const uint32_t* blcode, BitWriter* bw) {
  auto sym = [&](int s, int xv, int xb) {
    if (!bw) { ++blfreq[s]; return; }
    bw->put(blcode[s] >> 8, blcode[s] & 255);
    if (xb) bw->put(xv, xb);
  };
  int prev = -1, count = 0, nextlen = lens[0];
  int max_count = nextlen == 0 ? 138 : 7, min_count = nextlen == 0 ? 3 : 4;
  for (int n = 0; n <= max_code; ++n) {
    const int cur = nextlen;
    nextlen = n < max_code ? lens[n + 1] : -1;
    if (++count < max_count && cur == nextlen) continue;
    if (count < min_count) {
      for (; count > 0; --count) sym(cur, 0, 0);
    } else if (cur != 0) {
      if (cur != prev) { sym(cur, 0, 0); --count; }
      sym(16, count - 3, 2);
    } else if (count <= 10) {
      sym(17, count - 3, 3);
    } else {
      sym(18, count - 11, 7);
    }
    count = 0;
    prev = cur;
    if (nextlen == 0) { max_count = 138; min_count = 3; }
    else if (cur == nextlen) { max_count = 6; min_count = 3; }
    else { max_count = 7; min_count = 4; }
  }
}

__global__ void __launch_bounds__(256) png_block_trees(Bufs u) {
  __shared__ TreeWork w;
  __shared__ int hist[L_CODES], llen[288], dlen[D_CODES], bllen[BL_CODES], blfreq[BL_CODES];
  __shared__ uint32_t blcode[BL_CODES], dcode[D_CODES], scode[288];
  __shared__ int ndist;
  const int b = blockIdx.x, nb = (int)u.meta[M_BLOCKS], ntok = (int)u.meta[M_TOKENS];
  if (b >= nb) return;
  for (int i = threadIdx.x; i < L_CODES; i += blockDim.x) hist[i] = 0;
  if (threadIdx.x == 0) ndist = 0;
  __syncthreads();
  const int t0 = b * BLOCK_SYMS, t1 = min(ntok, t0 + BLOCK_SYMS);
  int nd = 0;
  for (int t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
    const uint16_t tk = u.tok[t];
    if (tk & 0x8000u) { atomicAdd(&hist[257 + len_index(tk & 0x1FF)], 1); ++nd; }
    else atomicAdd(&hist[tk], 1);
  }
  atomicAdd(&ndist, nd);
  __syncthreads();
  if (threadIdx.x != 0) return;

  long long opt = 0, stat = 0, dummy = 0;
  for (int i = 0; i < L_CODES; ++i) w.freq[i] = hist[i];
  w.freq[END_BLOCK] = 1;
  const int lmax = build_tree(w, L_CODES, 15, 0, &opt, &stat);
  for (int i = 0; i < L_CODES; ++i) llen[i] = w.len[i];
  for (int i = 0; i < D_CODES; ++i) w.freq[i] = 0;
  w.freq[0] = ndist;
  const int dmax = build_tree(w, D_CODES, 15, 1, &opt, &stat);
  for (int i = 0; i < D_CODES; ++i) dlen[i] = w.len[i];
  for (int i = 0; i < BL_CODES; ++i) blfreq[i] = 0;
  length_runs(llen, lmax, blfreq, nullptr, nullptr);
  length_runs(dlen, dmax, blfreq, nullptr, nullptr);
  for (int i = 0; i < BL_CODES; ++i) w.freq[i] = blfreq[i];
  build_tree(w, BL_CODES, 7, 2, &opt, &dummy);
  for (int i = 0; i < BL_CODES; ++i) bllen[i] = w.len[i];
  int max_bl = BL_CODES - 1;
  while (max_bl >= 3 && bllen[c_bl_order[max_bl]] == 0) --max_bl;
  opt += 3ll * (max_bl + 1) + 5 + 5 + 4;

  const long long opt_bytes0 = (opt + 3 + 7) >> 3, static_bytes = (stat + 3 + 7) >> 3;
  const long long opt_bytes = static_bytes <= opt_bytes0 ? static_bytes : opt_bytes0;
  const int stored_len = u.bstart[b + 1] - u.bstart[b];
  const int kind = stored_len + 4 <= opt_bytes ? KIND_STORED : static_bytes == opt_bytes ? KIND_STATIC : KIND_DYNAMIC;
  u.kind[b] = kind;
  u.stored[b] = stored_len;
  uint32_t* code = u.code + (size_t)b * CODE_STRIDE;
  int hb = 0;
  if (kind == KIND_DYNAMIC) {
    canonical(llen, L_CODES, code);
    canonical(dlen, D_CODES, dcode);
    code[DIST0] = dcode[0];
    canonical(bllen, BL_CODES, blcode);
    BitWriter bw{u.hdr + (size_t)b * HDR_WORDS, 0, 0, 0};
    bw.put(lmax + 1 - 257, 5);
    bw.put(dmax + 1 - 1, 5);
    bw.put(max_bl + 1 - 4, 4);
    for (int i = 0; i <= max_bl; ++i) bw.put(bllen[c_bl_order[i]], 3);
    length_runs(llen, lmax, nullptr, blcode, &bw);
    length_runs(dlen, dmax, nullptr, blcode, &bw);
    hb = bw.n * 32 + bw.nb;
    bw.flush();
    u.bits[b] = (int)(3 + opt);
  } else if (kind == KIND_STATIC) {
    for (int i = 0; i < 288; ++i) llen[i] = static_llen(i);
    canonical(llen, 288, scode);                       // the static code has 288 lengths, 286 and 287 never sent
    for (int i = 0; i < L_CODES; ++i) code[i] = scode[i];
    code[DIST0] = 5u;                                  // distance code 0: five zero bits
    u.bits[b] = (int)(3 + stat);
  } else {
    u.bits[b] = 0;
  }
  u.hdr_bits[b] = hb;
}

// ------------------------------------------------------------------------------------------------ offsets, emission
// One thread: the bit offset of every block (a stored block pads to a byte, so its length depends on where it starts),
// the zlib header, the Adler-32 trailer and the file length.
__global__ void png_block_offsets(int64_t* out_len, Bufs u) {
  const int nb = (int)u.meta[M_BLOCKS];
  long long off = 16;                                  // after the zlib header
  for (int b = 0; b < nb; ++b) {
    u.boff[b] = off;
    if (u.kind[b] == KIND_STORED) off = ((off + 3 + 7) & ~7ll) + 32 + 8ll * u.stored[b];
    else off += u.bits[b];
  }
  const long long end = (off + 7) >> 3;
  uint8_t* z = reinterpret_cast<uint8_t*>(u.z);
  const long long L = u.bstart[nb];
  int wb = 8;                                          // window bits: the smallest window holding S, 8..15
  while (wb < 15 && (1ll << wb) < L) ++wb;
  const int cmf = ((wb - 8) << 4) | 8;
  z[0] = (uint8_t)cmf;
  z[1] = (uint8_t)(31 - (cmf * 256) % 31);
  const uint32_t ad = (uint32_t)u.meta[M_ADLER];
  z[end] = ad >> 24; z[end + 1] = ad >> 16; z[end + 2] = ad >> 8; z[end + 3] = ad;
  const long long zlen = end + 4;
  u.meta[M_ZLEN] = zlen;
  *out_len = 8 + 25 + zlen + 12 * ((zlen + IDAT - 1) / IDAT) + 12;
}

// LSB-first bit writer OR-ing into the shared zlib buffer (its first and last words may belong to a neighbour too).
struct BitSink {
  uint32_t* z;
  long long word;
  uint64_t acc;
  int nb;
  __device__ BitSink(uint32_t* z_, long long bit) : z(z_), word(bit >> 5), acc(0), nb((int)(bit & 31)) {}
  __device__ void put(uint32_t v, int bits) {
    acc |= (uint64_t)v << nb;
    nb += bits;
    if (nb >= 32) { atomicOr(&z[word++], (uint32_t)acc); acc >>= 32; nb -= 32; }
  }
  __device__ void flush() { if (acc) atomicOr(&z[word], (uint32_t)acc); }
};

__global__ void __launch_bounds__(EMIT_T) png_emit(Bufs u) {
  __shared__ uint32_t code[CODE_STRIDE];
  __shared__ int sm[EMIT_T / 32 + 1];
  const int b = blockIdx.x, nb = (int)u.meta[M_BLOCKS], ntok = (int)u.meta[M_TOKENS];
  if (b >= nb) return;
  const long long off = u.boff[b];
  const int kind = u.kind[b], last = b == nb - 1;
  if (kind == KIND_STORED) {
    if (threadIdx.x == 0) { BitSink s(u.z, off); s.put(last, 3); s.flush(); }
    const long long sb = (off + 3 + 7) >> 3;         // first byte after the padding
    const int n = u.stored[b];
    const uint8_t* src = u.s + u.bstart[b];
    const uint32_t hdr = (uint32_t)n | ((uint32_t)(n ^ 0xFFFF) << 16);
    for (long long wd = (sb >> 2) + threadIdx.x; wd <= (sb + 4 + n - 1) >> 2; wd += EMIT_T) {
      uint32_t v = 0;
      for (int k = 0; k < 4; ++k) {
        const long long q = wd * 4 + k - sb;
        if (q < 0 || q >= 4 + n) continue;
        const uint32_t byte = q < 4 ? (hdr >> (8 * q)) & 255u : src[q - 4];
        v |= byte << (8 * k);
      }
      atomicOr(&u.z[wd], v);
    }
    return;
  }
  for (int i = threadIdx.x; i < CODE_STRIDE; i += EMIT_T) code[i] = u.code[(size_t)b * CODE_STRIDE + i];
  __syncthreads();
  const int hb = u.hdr_bits[b];
  if (threadIdx.x == 0) {
    BitSink s(u.z, off);
    s.put((kind == KIND_STATIC ? 2 : 4) + last, 3);
    const uint32_t* h = u.hdr + (size_t)b * HDR_WORDS;
    for (int k = 0; k < hb; k += 32) s.put(h[k >> 5], min(32, hb - k));
    s.flush();
  }
  const int t0 = b * BLOCK_SYMS, t1 = min(ntok, t0 + BLOCK_SYMS);
  const int my0 = t0 + threadIdx.x * EMIT_V, my1 = min(t1, my0 + EMIT_V);
  const uint32_t dist = code[DIST0];
  int bits = 0;
  for (int t = my0; t < my1; ++t) {
    const uint16_t tk = u.tok[t];
    if (tk & 0x8000u) {
      const int li = len_index(tk & 0x1FF);
      bits += (code[257 + li] & 255) + c_len_extra[li] + (dist & 255);
    } else {
      bits += code[tk] & 255;
    }
  }
  int total;
  const int before = cta_exclusive_scan<EMIT_T>(bits, sm, &total);
  const long long base = off + 3 + hb;
  if (my0 < my1) {
    BitSink s(u.z, base + before);
    for (int t = my0; t < my1; ++t) {
      const uint16_t tk = u.tok[t];
      if (tk & 0x8000u) {
        const int len = tk & 0x1FF, li = len_index(len);
        const uint32_t c = code[257 + li];
        s.put(c >> 8, c & 255);
        if (c_len_extra[li]) s.put(len - c_len_base[li], c_len_extra[li]);
        s.put(dist >> 8, dist & 255);
      } else {
        s.put(code[tk] >> 8, code[tk] & 255);
      }
    }
    s.flush();
  }
  if (threadIdx.x == EMIT_T - 1) {
    BitSink s(u.z, base + total);
    s.put(code[END_BLOCK] >> 8, code[END_BLOCK] & 255);
    s.flush();
  }
}

// ------------------------------------------------------------------------------------------------ PNG chunks
constexpr uint32_t CRC_POLY = 0xEDB88320u;

// a * b modulo the CRC-32 polynomial, in the reflected bit order (bit 31 is x^0).
__device__ uint32_t crc_mul(uint32_t a, uint32_t b) {
  uint32_t p = 0;
  for (uint32_t m = 0x80000000u; m; m >>= 1) {
    if (a & m) p ^= b;
    b = (b & 1) ? (b >> 1) ^ CRC_POLY : b >> 1;
  }
  return p;
}

// CRC register c advanced over n zero bytes: c * x^(8n).  x2n[k] = x^(8 * 2^k).
__device__ uint32_t crc_shift(uint32_t c, int n, const uint32_t* x2n) {
  for (int k = 0; n; ++k, n >>= 1)
    if (n & 1) c = crc_mul(c, x2n[k]);
  return c;
}

__device__ uint32_t put_be32(uint8_t* p, uint32_t v) {
  p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v;
  return v;
}

// One CTA per IDAT chunk; each thread takes a 33-byte segment of "IDAT" + data, the segment CRCs are combined.
constexpr int CRC_SEG = 33;
static_assert(CRC_SEG * TILE_T >= IDAT + 4, "segments cover a chunk");

__global__ void __launch_bounds__(TILE_T) png_assemble(int H, int W, uint8_t* __restrict__ out, Bufs u) {
  __shared__ uint32_t tab[256], x2n[16];
  __shared__ uint32_t red[TILE_T / 32];
  const long long zlen = u.meta[M_ZLEN];
  const int nchunk = (int)((zlen + IDAT - 1) / IDAT), c = blockIdx.x;
  if (c >= nchunk) return;
  {
    uint32_t v = threadIdx.x;
    for (int k = 0; k < 8; ++k) v = (v & 1) ? (v >> 1) ^ CRC_POLY : v >> 1;
    tab[threadIdx.x] = v;
  }
  if (threadIdx.x == 0) {
    x2n[0] = 0x00800000u;                              // x^8
    for (int k = 1; k < 16; ++k) x2n[k] = crc_mul(x2n[k - 1], x2n[k - 1]);
  }
  __syncthreads();
  const uint8_t* z = reinterpret_cast<const uint8_t*>(u.z) + (long long)c * IDAT;
  const int dlen = (int)min((long long)IDAT, zlen - (long long)c * IDAT), n = dlen + 4;
  uint8_t* o = out + 33 + (long long)c * (IDAT + 12);
  for (int i = threadIdx.x; i < dlen; i += TILE_T) o[8 + i] = z[i];
  const uint8_t tag[4] = {'I', 'D', 'A', 'T'};
  const int s0 = threadIdx.x * CRC_SEG, s1 = min(n, s0 + CRC_SEG);
  uint32_t r = 0;                                      // raw CRC (register 0) of the segment
  for (int i = s0; i < s1; ++i) r = tab[(r ^ (i < 4 ? tag[i] : z[i - 4])) & 255] ^ (r >> 8);
  if (s0 < s1) r = crc_shift(r, n - s1, x2n);
  else r = 0;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) r ^= __shfl_xor_sync(0xffffffffu, r, d);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = r;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t crc = 0;
    for (int k = 0; k < TILE_T / 32; ++k) crc ^= red[k];
    crc ^= crc_shift(0xFFFFFFFFu, n, x2n);             // the register's initial value, carried over all n bytes
    put_be32(o, (uint32_t)dlen);
    for (int k = 0; k < 4; ++k) o[4 + k] = tag[k];
    put_be32(o + 8 + dlen, ~crc);
    if (c == 0) {
      const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
      for (int k = 0; k < 8; ++k) out[k] = sig[k];
      uint8_t* ih = out + 8;
      put_be32(ih, 13);
      const uint8_t hd[17] = {'I', 'H', 'D', 'R', (uint8_t)(W >> 24), (uint8_t)(W >> 16), (uint8_t)(W >> 8), (uint8_t)W,
                              (uint8_t)(H >> 24), (uint8_t)(H >> 16), (uint8_t)(H >> 8), (uint8_t)H, 8, 2, 0, 0, 0};
      uint32_t cc = 0xFFFFFFFFu;
      for (int k = 0; k < 17; ++k) { ih[4 + k] = hd[k]; cc = tab[(cc ^ hd[k]) & 255] ^ (cc >> 8); }
      put_be32(ih + 21, ~cc);
    }
    if (c == nchunk - 1) {
      const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
      for (int k = 0; k < 12; ++k) o[dlen + 12 + k] = iend[k];
    }
  }
}

bool plan_ok(int H, int W) { return H >= 1 && W >= 1 && (long long)H * (3ll * W + 1) <= (1ll << 30); }

}  // namespace

extern "C" {

int teco_png_plan_bytes(int32_t H, int32_t W, int64_t* workspace_bytes_host, int64_t* out_capacity_host) {
  TECO_CHECK_ARG(workspace_bytes_host && out_capacity_host, "teco_png_plan_bytes: NULL argument");
  TECO_CHECK_ARG(plan_ok(H, W), "teco_png_plan_bytes: bad frame size %dx%d (H, W >= 1, H*(3W+1) <= 2^30)", H, W);
  const Plan p = make_plan(H, W);
  *workspace_bytes_host = p.ws_bytes;
  *out_capacity_host = p.out_cap;
  return TECO_OK;
}

int teco_png_encode_rgb8(const uint8_t* rgb, int32_t H, int32_t W, void* workspace, int64_t workspace_bytes, uint8_t* out,
                         int64_t out_capacity, int64_t* out_len, void* stream) {
  TECO_CHECK_ARG(rgb && workspace && out && out_len, "teco_png_encode_rgb8: NULL argument");
  TECO_CHECK_ARG(plan_ok(H, W), "teco_png_encode_rgb8: bad frame size %dx%d (H, W >= 1, H*(3W+1) <= 2^30)", H, W);
  const Plan p = make_plan(H, W);
  TECO_CHECK_ARG(workspace_bytes >= p.ws_bytes && out_capacity >= p.out_cap,
                 "teco_png_encode_rgb8: buffers of %lld / %lld bytes, the %dx%d plan needs %lld / %lld",
                 (long long)workspace_bytes, (long long)out_capacity, H, W, p.ws_bytes, p.out_cap);
  TECO_CHECK_ARG(((uintptr_t)workspace & 255) == 0, "teco_png_encode_rgb8: workspace must be 256-byte aligned");
  const cudaStream_t st = (cudaStream_t)stream;
  const Bufs u = carve(p, workspace);
  const int zt = (int)((p.zwords + TILE / 4 - 1) / (TILE / 4));
  png_filter<<<max(p.ntile, zt), TILE_T, 0, st>>>(rgb, W, p, u);
  png_scan<<<1, 1024, 0, st>>>(u.run_cnt, u.run_off, p.ntile, p, u, M_RUNS, 1);
  png_runs<<<p.ntile, TILE_T, 0, st>>>(p, u);
  png_run_tokens<<<p.ntile, TILE_T, 0, st>>>(u);
  png_scan<<<1, 1024, 0, st>>>(u.tok_cnt, u.tok_off, p.ntile, p, u, M_TOKENS, 0);
  png_token_offsets<<<p.ntile, TILE_T, 0, st>>>(u);
  png_tokens<<<p.ntile, TILE_T, 0, st>>>(p, u);
  png_block_trees<<<p.maxblk, 256, 0, st>>>(u);
  png_block_offsets<<<1, 1, 0, st>>>(out_len, u);
  png_emit<<<p.maxblk, EMIT_T, 0, st>>>(u);
  png_assemble<<<p.maxchunk, TILE_T, 0, st>>>(H, W, out, u);
  TECO_CUDA_LAUNCH_CHECK("teco_png_encode_rgb8");
  return TECO_OK;
}

}  // extern "C"
