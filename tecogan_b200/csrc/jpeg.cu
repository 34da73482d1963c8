// JPEG encoder for RGB uint8 frames, byte-identical to cv2.imwrite(path.jpg) with its defaults (libjpeg-turbo: baseline,
// quality 95, 4:2:0, islow FDCT, the Huffman tables of T.81 Annex K.3): DESIGN.md section 4.6.
// tests/golden/jpeg_oracle.py states every step on the host; tests/test_jpeg_host.py pins it to cv2.
//
// Stages (one kernel each, all on the caller's stream, sizes read from the device where the host cannot know them):
//   jpeg_blocks       per 4 MCUs: edge rules, colour conversion, h2v2 downsampling, FDCT, quantisation; the int16 zigzag
//                     coefficients of every block in scan order, dummy blocks included
//   jpeg_block_bits   per tile of 64 blocks, one warp per block: each block's coded length, and the tile's sum
//   jpeg_scan         exclusive scan of the tile sums into bit offsets; zeroes the words two tiles can share
//   jpeg_emit         per tile: its codes composed MSB first in shared memory, stored as 32-bit words (the first and last,
//                     which a neighbour tile may share, with atomicOr)
//   jpeg_stuff_count  per 4 096-byte tile of the entropy-coded data (last byte padded with 1-bits): its 0xFF bytes
//   jpeg_scan         exclusive scan of those counts
//   jpeg_assemble     the header, the data with a 0x00 after every 0xFF, EOI, and the file length
#include <initializer_list>

#include "teco_common.cuh"

namespace {

// ------------------------------------------------------------------------------------------------ format constants
constexpr int MAX_SIDE = 65500;                 // JPEG's own limit on H and W
constexpr int QUALITY = 95;                     // cv2's default IMWRITE_JPEG_QUALITY
constexpr int G = 4;                            // MCUs per CTA in jpeg_blocks
constexpr int BLK_T = G * 6 * 8;                // one thread per block row (FDCT pass 1), then per column (pass 2)
constexpr int PITCH = 9;                        // shared row pitch of an 8x8 block: no bank conflicts in either pass
constexpr int TILE_B = 64;                      // blocks per tile in jpeg_block_bits / jpeg_emit
constexpr int CODE_T = 256;                     // 8 warps, 8 blocks each
// Bits of one block at most: DC code 11 + 11 amplitude bits; each of the 63 AC positions 16 (code) + 10 (amplitude). A
// ZRL stands for 16 positions and EOB for at least one, so neither breaks the bound.
constexpr int MAX_BLOCK_BITS = 11 + 11 + 63 * (16 + 10);
constexpr int TILE_WORDS = (31 + TILE_B * MAX_BLOCK_BITS + 31) / 32;
constexpr int STUFF_T = 256, STUFF_V = 16, STUFF_TILE = STUFF_T * STUFF_V;   // bytes per tile in the stuffing stages
constexpr int HDR_BYTES = 2 + 18 + 2 * 69 + 19 + 2 * 33 + 2 * 183 + 14;      // SOI APP0 DQT*2 SOF0 DHT*4 SOS = 623

constexpr uint8_t kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// T.81 Tables K.1 and K.2, natural (row-major) order.
constexpr uint8_t kLumaBase[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                   14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                   18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                   49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kChromaBase[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                     24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
// T.81 Tables K.3 - K.6: code counts per length 1..16, then the symbols in code order.
constexpr uint8_t kDcLumaBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcLumaBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
constexpr uint8_t kAcLumaVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
    0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
    0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
    0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
    0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
    0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
    0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa};
constexpr uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
constexpr uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32, 0x81,
    0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34,
    0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44,
    0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92,
    0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4,
    0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6,
    0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa};

// libjpeg's quality scaling for quality >= 50: base * (200 - 2 * quality) / 100, rounded, clamped to 1..255.
constexpr int quant(int base) {
  const int v = (base * (200 - 2 * QUALITY) + 50) / 100;
  return v < 1 ? 1 : v > 255 ? 255 : v;
}

// What the kernels look up: Huffman codes as (code << 8) | length by symbol (0: no code), and the quantiser divisors.
struct Tables {
  uint32_t dc[2][16];       // luma, chroma; symbol = size category 0..11
  uint32_t ac[2][256];      // symbol = run << 4 | size
  uint16_t qdiv[2][64];     // 8 * Q in natural order (the FDCT's output is scaled by 8)
  uint8_t zigzag[64];
};

// T.81 Annex C: codes of each length are consecutive, and the next length starts at twice the last code + 1.
constexpr void huff_codes(const uint8_t (&bits)[16], const uint8_t* vals, uint32_t* out) {
  int code = 0, k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < bits[len - 1]; ++i) out[vals[k++]] = ((uint32_t)code++ << 8) | (uint32_t)len;
    code <<= 1;
  }
}

constexpr Tables make_tables() {
  Tables t{};
  huff_codes(kDcLumaBits, kDcVals, t.dc[0]);
  huff_codes(kDcChromaBits, kDcVals, t.dc[1]);
  huff_codes(kAcLumaBits, kAcLumaVals, t.ac[0]);
  huff_codes(kAcChromaBits, kAcChromaVals, t.ac[1]);
  for (int i = 0; i < 64; ++i) {
    t.qdiv[0][i] = (uint16_t)(8 * quant(kLumaBase[i]));
    t.qdiv[1][i] = (uint16_t)(8 * quant(kChromaBase[i]));
    t.zigzag[i] = kZigzag[i];
  }
  return t;
}

__constant__ Tables c_tab = make_tables();

// The 623 header bytes; only H and W (SOF0 bytes 5..8) depend on the frame.
struct Header {
  uint8_t b[HDR_BYTES];
};

Header make_header(int H, int W) {
  Header h{};
  int n = 0;
  auto put = [&](std::initializer_list<int> v) { for (int x : v) h.b[n++] = (uint8_t)x; };
  put({0xFF, 0xD8});
  put({0xFF, 0xE0, 0, 16, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0});   // JFIF 1.01, unit 0, 1:1, no thumbnail
  for (int t = 0; t < 2; ++t) {
    put({0xFF, 0xDB, 0, 67, t});
    for (int z = 0; z < 64; ++z) h.b[n++] = (uint8_t)quant((t ? kChromaBase : kLumaBase)[kZigzag[z]]);
  }
  put({0xFF, 0xC0, 0, 17, 8, H >> 8, H & 255, W >> 8, W & 255, 3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1});
  auto dht = [&](int cls_id, const uint8_t (&bits)[16], const uint8_t* vals) {
    int nv = 0;
    for (int i = 0; i < 16; ++i) nv += bits[i];
    put({0xFF, 0xC4, (3 + 16 + nv) >> 8, (3 + 16 + nv) & 255, cls_id});
    for (int i = 0; i < 16; ++i) h.b[n++] = bits[i];
    for (int i = 0; i < nv; ++i) h.b[n++] = vals[i];
  };
  dht(0x00, kDcLumaBits, kDcVals);
  dht(0x10, kAcLumaBits, kAcLumaVals);
  dht(0x01, kDcChromaBits, kDcVals);
  dht(0x11, kAcChromaBits, kAcChromaVals);
  put({0xFF, 0xDA, 0, 12, 3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0});
  return h;
}

// ------------------------------------------------------------------------------------------------ plan
struct Plan {
  int mw, mh;             // MCUs per row, MCU rows
  int bw, bh;             // real 8x8 luma blocks per row and column: ceil(W/8), ceil(H/8)
  long long nblk;         // 6 blocks per MCU: Y00 Y01 Y10 Y11 Cb Cr
  int ntile;              // tiles of TILE_B blocks
  long long max_bytes;    // entropy-coded bytes at most, before stuffing
  int nstuff;             // byte tiles at most
  long long zwords, out_cap, ws_bytes;
  long long off_coef, off_bits, off_tcnt, off_toff, off_z, off_fcnt, off_foff, off_meta;
};

__host__ __device__ inline long long align256(long long x) { return (x + 255) & ~255ll; }

inline Plan make_plan(int H, int W) {
  Plan p;
  p.mw = (W + 15) / 16;
  p.mh = (H + 15) / 16;
  p.bw = (W + 7) / 8;
  p.bh = (H + 7) / 8;
  p.nblk = 6ll * p.mw * p.mh;
  p.ntile = (int)((p.nblk + TILE_B - 1) / TILE_B);
  p.max_bytes = (p.nblk * MAX_BLOCK_BITS + 7) / 8;
  p.nstuff = (int)((p.max_bytes + STUFF_TILE - 1) / STUFF_TILE);
  p.zwords = (long long)p.nstuff * (STUFF_TILE / 4);       // whole tiles: jpeg_stuff_count reads 16 bytes per thread
  p.out_cap = HDR_BYTES + 2 * p.max_bytes + 2;               // every data byte stuffed, + EOI
  long long o = 0;
  p.off_coef = o; o = align256(o + 2 * 64 * p.nblk);
  p.off_bits = o; o = align256(o + 4 * p.nblk);
  p.off_tcnt = o; o = align256(o + 4ll * p.ntile);
  p.off_toff = o; o = align256(o + 8ll * p.ntile);
  p.off_z = o;    o = align256(o + 4 * p.zwords);
  p.off_fcnt = o; o = align256(o + 4ll * p.nstuff);
  p.off_foff = o; o = align256(o + 8ll * p.nstuff);
  p.off_meta = o; o = align256(o + 8 * 4);
  p.ws_bytes = o;
  return p;
}

// meta[]: the sizes only the device knows
enum { M_BITS = 0, M_FF = 1 };

struct Bufs {
  int16_t* coef;          // [nblk][64] zigzag order
  int* bits;              // coded bits per block
  int* tile_bits;
  long long* tile_off;    // bit offset of each tile
  uint32_t* z;            // the entropy-coded bits, MSB first in each word
  int* ff_cnt;
  long long* ff_off;
  long long* meta;
};

inline Bufs carve(const Plan& p, void* ws) {
  uint8_t* b = (uint8_t*)ws;
  return Bufs{(int16_t*)(b + p.off_coef), (int*)(b + p.off_bits),       (int*)(b + p.off_tcnt),
              (long long*)(b + p.off_toff), (uint32_t*)(b + p.off_z),   (int*)(b + p.off_fcnt),
              (long long*)(b + p.off_foff), (long long*)(b + p.off_meta)};
}

// ------------------------------------------------------------------------------------------------ blocks
// Colour conversion, 16 fractional bits (libjpeg's FIX(x) = round(x * 2^16)); Cb and Cr round with 2^15 - 1.
constexpr int fix16(double x) { return (int)(x * 65536.0 + 0.5); }
__device__ __forceinline__ int to_y(int r, int g, int b) {
  return (fix16(0.299) * r + fix16(0.587) * g + fix16(0.114) * b + (1 << 15)) >> 16;
}
__device__ __forceinline__ int to_cb(int r, int g, int b) {
  return (-fix16(0.16874) * r - fix16(0.33126) * g + fix16(0.5) * b + (128 << 16) + (1 << 15) - 1) >> 16;
}
__device__ __forceinline__ int to_cr(int r, int g, int b) {
  return (fix16(0.5) * r - fix16(0.41869) * g - fix16(0.08131) * b + (128 << 16) + (1 << 15) - 1) >> 16;
}

// The islow FDCT of 8 values at v[0], v[s], .., v[7s], in place (CONST_BITS 13, PASS1_BITS 2, round half up).  The
// FDCT is linear, so bounding each intermediate by sum |coefficient| * max |input| is exact for pass 1 (samples in
// -128..127): every pass-1 intermediate is below 1.1e7 and its outputs below 4 100.  With those as pass 2's inputs, every
// pass-2 intermediate is below 3.5e8 < 2^29, so int32 cannot overflow; the outputs are at most 8 192 (= 64 * 128).
constexpr int fix13(double x) { return (int)(x * 8192.0 + 0.5); }
template <bool PASS2>
__device__ __forceinline__ void fdct8(int* v, int s) {
  constexpr int n = PASS2 ? 13 + 2 : 13 - 2;
  auto descale = [](int x, int b) { return (x + (1 << (b - 1))) >> b; };
  const int t0 = v[0] + v[7 * s], t7 = v[0] - v[7 * s], t1 = v[s] + v[6 * s], t6 = v[s] - v[6 * s];
  const int t2 = v[2 * s] + v[5 * s], t5 = v[2 * s] - v[5 * s], t3 = v[3 * s] + v[4 * s], t4 = v[3 * s] - v[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  v[0] = PASS2 ? descale(t10 + t11, 2) : (t10 + t11) * 4;
  v[4 * s] = PASS2 ? descale(t10 - t11, 2) : (t10 - t11) * 4;
  const int e = (t12 + t13) * fix13(0.541196100);
  v[2 * s] = descale(e + t13 * fix13(0.765366865), n);
  v[6 * s] = descale(e - t12 * fix13(1.847759065), n);
  const int z5 = (t4 + t5 + t6 + t7) * fix13(1.175875602);
  const int z1 = -(t4 + t7) * fix13(0.899976223), z2 = -(t5 + t6) * fix13(2.562915447);
  const int z3 = -(t4 + t6) * fix13(1.961570560) + z5, z4 = -(t5 + t7) * fix13(0.390180644) + z5;
  v[7 * s] = descale(t4 * fix13(0.298631336) + z1 + z3, n);
  v[5 * s] = descale(t5 * fix13(2.053119869) + z2 + z4, n);
  v[3 * s] = descale(t6 * fix13(3.072711026) + z2 + z3, n);
  v[s] = descale(t7 * fix13(1.501321110) + z1 + z4, n);
}

__device__ __forceinline__ int quantise(int c, int d) {
  const int q = ((c < 0 ? -c : c) + (d >> 1)) / d;
  return c < 0 ? -q : q;
}

// CTA (blockIdx.x, blockIdx.y) = MCUs G*x .. G*x+G-1 of MCU row y.  Shared: 6 blocks per MCU, 8 rows of PITCH ints.
__global__ void __launch_bounds__(BLK_T) jpeg_blocks(const uint8_t* __restrict__ rgb, int H, int W, Plan p, Bufs u) {
  __shared__ int s[G * 6 * 8 * PITCH];
  __shared__ uint16_t qdiv[2][64];
  __shared__ uint8_t zz[64];
  const int my = blockIdx.y, mx0 = blockIdx.x * G, ng = min(G, p.mw - mx0), tid = threadIdx.x;
  if (tid < 128) qdiv[tid >> 6][tid & 63] = c_tab.qdiv[tid >> 6][tid & 63];
  if (tid < 64) zz[tid] = c_tab.zigzag[tid];
  auto px = [&](int y, int x, int& r, int& g, int& b) {
    const uint8_t* q = rgb + ((long long)y * W + x) * 3;
    r = q[0]; g = q[1]; b = q[2];
  };
  // Y: image rows and columns repeated past the edge (the blocks wholly outside are dummies, written below).
  for (int i = tid; i < 16 * 16 * G; i += BLK_T) {
    const int ly = i / (16 * G), lx = i % (16 * G);
    if (lx >= 16 * ng) continue;
    int r, g, b;
    px(min(my * 16 + ly, H - 1), min(mx0 * 16 + lx, W - 1), r, g, b);
    const int k = (ly >> 3) * 2 + ((lx >> 3) & 1);
    s[(((lx >> 4) * 6 + k) * 8 + (ly & 7)) * PITCH + (lx & 7)] = to_y(r, g, b) - 128;
  }
  // Cb, Cr: columns repeated to whole MCUs, rows to an even count; 2x2 sums + bias 1, 2, 1, 2, .. along each row, >> 2;
  // then the last downsampled row repeated down its block.
  const int crow_last = (H + 1) / 2 - 1;
  for (int i = tid; i < 8 * 8 * G; i += BLK_T) {
    const int ly = i / (8 * G), lx = i % (8 * G);
    if (lx >= 8 * ng) continue;
    const int cr = min(my * 8 + ly, crow_last), cx = mx0 * 8 + lx;
    const int y0 = 2 * cr, y1 = min(2 * cr + 1, H - 1), x0 = min(2 * cx, W - 1), x1 = min(2 * cx + 1, W - 1);
    int sb = 0, sr = 0;
    const int ys[2] = {y0, y1}, xs[2] = {x0, x1};
#pragma unroll
    for (int a = 0; a < 4; ++a) {
      int r, g, b;
      px(ys[a >> 1], xs[a & 1], r, g, b);
      sb += to_cb(r, g, b);
      sr += to_cr(r, g, b);
    }
    const int bias = 1 + (lx & 1);
    int* o = &s[((lx >> 3) * 6 * 8 + ly) * PITCH + (lx & 7)];
    o[4 * 8 * PITCH] = ((sb + bias) >> 2) - 128;
    o[5 * 8 * PITCH] = ((sr + bias) >> 2) - 128;
  }
  __syncthreads();
  const int blk = tid >> 3, line = tid & 7;
  if (blk < ng * 6) fdct8<false>(&s[(blk * 8 + line) * PITCH], 1);
  __syncthreads();
  if (blk < ng * 6) fdct8<true>(&s[blk * 8 * PITCH + line], PITCH);
  __syncthreads();
  // Quantise and reorder.  A luma block outside ceil(W/8) x ceil(H/8) is a dummy: zero AC, and the DC of the block before
  // it in the MCU, i.e. of the last real luma block before it (block 0 always is one).
  int16_t* out = u.coef + ((long long)my * p.mw + mx0) * 6 * 64;
  for (int i = tid; i < ng * 6 * 64; i += BLK_T) {
    const int b = i >> 6, z = i & 63, k = b % 6, m = b / 6;
    int src = b;
    if (k < 4) {
      const bool xin = 2 * (mx0 + m) + 1 < p.bw, yin = 2 * my + 1 < p.bh;
      const bool real = (!(k & 1) || xin) && (!(k & 2) || yin);
      if (!real) {
        if (z) { out[i] = 0; continue; }
        src = m * 6 + (k == 3 ? (xin ? 1 : yin ? 2 : 0) : k == 2 ? (xin ? 1 : 0) : 0);
      }
    }
    const int n = zz[z];
    out[i] = (int16_t)quantise(s[(src * 8 + (n >> 3)) * PITCH + (n & 7)], qdiv[k < 4 ? 0 : 1][n]);
  }
}

// ------------------------------------------------------------------------------------------------ Huffman coding
__device__ __forceinline__ int size_cat(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }
__device__ __forceinline__ uint32_t amplitude(int v, int s) { return (uint32_t)(v < 0 ? v + (1 << s) - 1 : v); }
__device__ __forceinline__ uint32_t low_mask(int n) { return n >= 32 ? ~0u : (1u << n) - 1u; }

// The block before b of the same component in scan order, or -1 where the DC predictor starts at 0.
__device__ __forceinline__ long long prev_block(long long b) {
  const long long m = b / 6;
  const int k = (int)(b - 6 * m);
  if (k >= 1 && k <= 3) return b - 1;
  if (m == 0) return -1;
  return k == 0 ? b - 3 : b - 6;
}

// Lane l of a warp codes zigzag positions 2l and 2l+1 of block b: lane 0 the DC difference, lane 31 the EOB when
// position 63 is zero.  put(bits, n) receives each code with its amplitude bits appended (n <= 27), in stream order.
template <class Put>
__device__ __forceinline__ void lane_codes(const int16_t* __restrict__ coef, long long b, int lane, const uint32_t* sdc,
                                           const uint32_t* sac, Put&& put) {
  const int t = (b % 6) < 4 ? 0 : 1;
  const uint32_t pair = reinterpret_cast<const uint32_t*>(coef + b * 64)[lane];
  const int v0 = (int16_t)(pair & 0xFFFFu), v1 = (int16_t)(pair >> 16);
  const uint32_t even = __ballot_sync(0xffffffffu, v0 != 0) & ~1u;   // nonzero AC at positions 2j (0 is the DC)
  const uint32_t odd = __ballot_sync(0xffffffffu, v1 != 0);          // nonzero AC at positions 2j+1
  const uint32_t* dc = sdc + 16 * t;
  const uint32_t* ac = sac + 256 * t;
  auto code = [&](uint32_t c, int v, int sz) { put(((c >> 8) << sz) | amplitude(v, sz), (int)(c & 255) + sz); };
  auto ac_code = [&](int pos, int v) {
    const uint32_t e = even & low_mask((pos + 1) >> 1), o = odd & low_mask(pos >> 1);   // nonzero AC before pos
    const int last = max(e ? 2 * (31 - __clz(e)) : 0, o ? 2 * (31 - __clz(o)) + 1 : 0);
    int run = pos - last - 1;
    for (; run >= 16; run -= 16) put(ac[0xF0] >> 8, (int)(ac[0xF0] & 255));
    const int sz = size_cat(v);
    code(ac[(run << 4) | sz], v, sz);
  };
  if (lane == 0) {
    const long long pb = prev_block(b);
    const int diff = v0 - (pb < 0 ? 0 : (int)coef[pb * 64]);
    const int sz = size_cat(diff);
    code(dc[sz], diff, sz);
  } else if (v0) {
    ac_code(2 * lane, v0);
  }
  if (v1) ac_code(2 * lane + 1, v1);
  if (lane == 31 && !(odd >> 31)) put(ac[0x00] >> 8, (int)(ac[0x00] & 255));
}

__device__ __forceinline__ void load_codes(uint32_t* sdc, uint32_t* sac) {
  for (int i = threadIdx.x; i < 32; i += blockDim.x) sdc[i] = c_tab.dc[i >> 4][i & 15];
  for (int i = threadIdx.x; i < 512; i += blockDim.x) sac[i] = c_tab.ac[i >> 8][i & 255];
}

__device__ __forceinline__ int warp_total(int v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}

__global__ void __launch_bounds__(CODE_T) jpeg_block_bits(Plan p, Bufs u) {
  __shared__ uint32_t sdc[32], sac[512];
  __shared__ int part[CODE_T / 32];
  load_codes(sdc, sac);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int sum = 0;
  for (int j = 0; j < TILE_B / (CODE_T / 32); ++j) {
    const long long b = (long long)blockIdx.x * TILE_B + warp * (TILE_B / (CODE_T / 32)) + j;
    if (b >= p.nblk) break;                            // uniform across the warp
    int n = 0;
    lane_codes(u.coef, b, lane, sdc, sac, [&](uint32_t, int len) { n += len; });
    n = warp_total(n);
    if (lane == 0) u.bits[b] = n;
    sum += n;
  }
  if (lane == 0) part[warp] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
    for (int w = 0; w < CODE_T / 32; ++w) t += part[w];
    u.tile_bits[blockIdx.x] = t;
  }
}

// ------------------------------------------------------------------------------------------------ scans
// One CTA: off[t] = sum of cnt[0..t).  Stage 0, the block tiles: bit offsets, meta[M_BITS] = the total, and the first
// and last word of every tile zeroed (jpeg_emit ORs into them; it stores the words in between).  Stage 1, the byte
// tiles of the data (as many as meta[M_BITS] needs): 0xFF bytes before each, meta[M_FF] = the total.
__global__ void __launch_bounds__(1024) jpeg_scan(const int* __restrict__ cnt, long long* __restrict__ off, int n,
                                                  int stage, Bufs u) {
  __shared__ int sm[1024 / 32 + 1];
  if (stage == 1) n = (int)(((u.meta[M_BITS] + 7) / 8 + STUFF_TILE - 1) / STUFF_TILE);
  long long carry = 0;
  for (int base = 0; base < n; base += 1024) {
    const int t = base + threadIdx.x;
    const int v = t < n ? cnt[t] : 0;
    int total;
    const long long o = carry + cta_exclusive_scan<1024>(v, sm, &total);
    if (t < n) {
      off[t] = o;
      if (stage == 0) {
        u.z[o >> 5] = 0u;
        u.z[(o + v - 1) >> 5] = 0u;
      }
    }
    carry += total;
  }
  if (threadIdx.x == 0) u.meta[stage == 0 ? M_BITS : M_FF] = carry;
}

// ------------------------------------------------------------------------------------------------ emission
// MSB-first writer into a shared word array at a bit position.
struct SmemBits {
  uint32_t* w;
  int pos;
  __device__ void put(uint32_t v, int n) {
    const int i = pos >> 5, o = pos & 31;
    if (o + n <= 32) {
      atomicOr(&w[i], v << (32 - o - n));
    } else {
      atomicOr(&w[i], v >> (o + n - 32));
      atomicOr(&w[i + 1], v << (64 - o - n));
    }
    pos += n;
  }
};

__global__ void __launch_bounds__(CODE_T) jpeg_emit(Plan p, Bufs u) {
  __shared__ uint32_t sdc[32], sac[512];
  __shared__ uint32_t sw[TILE_WORDS];
  __shared__ int boff[TILE_B];
  __shared__ int sm[CODE_T / 32 + 1];
  const long long b0 = (long long)blockIdx.x * TILE_B;
  const int nb = (int)min((long long)TILE_B, p.nblk - b0);
  const long long base = u.tile_off[blockIdx.x];
  const int lead = (int)(base & 31);
  int total;
  const int before = cta_exclusive_scan<CODE_T>(threadIdx.x < nb ? u.bits[b0 + threadIdx.x] : 0, sm, &total);
  if (threadIdx.x < TILE_B) boff[threadIdx.x] = lead + before;
  const int nw = (lead + total + 31) >> 5;
  for (int i = threadIdx.x; i < nw; i += CODE_T) sw[i] = 0u;
  load_codes(sdc, sac);
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = 0; j < TILE_B / (CODE_T / 32); ++j) {
    const int lb = warp * (TILE_B / (CODE_T / 32)) + j;
    if (lb >= nb) break;
    int n = 0;
    lane_codes(u.coef, b0 + lb, lane, sdc, sac, [&](uint32_t, int len) { n += len; });
    int x = n;                                         // inclusive scan over the lanes
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    SmemBits sink{sw, boff[lb] + x - n};
    lane_codes(u.coef, b0 + lb, lane, sdc, sac, [&](uint32_t v, int len) { sink.put(v, len); });
  }
  __syncthreads();
  uint32_t* z = u.z + (base >> 5);
  for (int i = threadIdx.x; i < nw; i += CODE_T) {
    if (i == 0 || i == nw - 1) atomicOr(&z[i], sw[i]);
    else z[i] = sw[i];
  }
}

// ------------------------------------------------------------------------------------------------ stuffing, assembly
// Bytes i0 .. i0+15 of the entropy-coded data (16-byte aligned), the last byte of the data padded with 1-bits; bytes
// past the data are 0.
__device__ __forceinline__ void data_bytes(const uint32_t* __restrict__ z, long long i0, long long nbits, uint8_t* v) {
  const long long nbytes = (nbits + 7) >> 3;
  const uint4 q = *reinterpret_cast<const uint4*>(z + (i0 >> 2));
  const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
  for (int k = 0; k < STUFF_V; ++k) {
    const long long i = i0 + k;
    uint32_t x = (w[k >> 2] >> (24 - 8 * (k & 3))) & 255u;
    if (i == nbytes - 1) x |= (1u << (int)(8 * nbytes - nbits)) - 1u;
    v[k] = i < nbytes ? (uint8_t)x : 0;
  }
}

__global__ void __launch_bounds__(STUFF_T) jpeg_stuff_count(Bufs u) {
  __shared__ int sm[STUFF_T / 32 + 1];
  const long long nbits = u.meta[M_BITS], i0 = (long long)blockIdx.x * STUFF_TILE;
  if (i0 >= (nbits + 7) >> 3) return;                  // uniform across the CTA
  uint8_t v[STUFF_V];
  data_bytes(u.z, i0 + threadIdx.x * STUFF_V, nbits, v);
  int c = 0;
#pragma unroll
  for (int k = 0; k < STUFF_V; ++k) c += v[k] == 0xFF;
  int total;
  cta_exclusive_scan<STUFF_T>(c, sm, &total);
  if (threadIdx.x == 0) u.ff_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(STUFF_T) jpeg_assemble(Header hd, uint8_t* __restrict__ out,
                                                         int64_t* __restrict__ out_len, Bufs u) {
  __shared__ int sm[STUFF_T / 32 + 1];
  const long long nbits = u.meta[M_BITS], nbytes = (nbits + 7) >> 3, i0 = (long long)blockIdx.x * STUFF_TILE;
  const long long ntile = (nbytes + STUFF_TILE - 1) / STUFF_TILE;
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < HDR_BYTES; i += STUFF_T) out[i] = hd.b[i];
  if (blockIdx.x >= ntile) return;
  uint8_t v[STUFF_V];
  const long long i = i0 + threadIdx.x * STUFF_V;
  data_bytes(u.z, i, nbits, v);
  int c = 0;
#pragma unroll
  for (int k = 0; k < STUFF_V; ++k) c += v[k] == 0xFF;
  int total;
  const int before = cta_exclusive_scan<STUFF_T>(c, sm, &total);
  uint8_t* o = out + HDR_BYTES + i + u.ff_off[blockIdx.x] + before;
  const int n = (int)min((long long)STUFF_V, nbytes - i);
#pragma unroll
  for (int k = 0; k < STUFF_V; ++k) {
    if (k >= n) break;
    *o++ = v[k];
    if (v[k] == 0xFF) *o++ = 0;
  }
  if (blockIdx.x == ntile - 1 && threadIdx.x == 0) {
    const long long end = HDR_BYTES + nbytes + u.meta[M_FF];
    out[end] = 0xFF;
    out[end + 1] = 0xD9;
    *out_len = end + 2;
  }
}

bool plan_ok(int H, int W) { return H >= 1 && W >= 1 && H <= MAX_SIDE && W <= MAX_SIDE; }

}  // namespace

extern "C" {

int teco_jpeg_plan_bytes(int32_t H, int32_t W, int64_t* workspace_bytes_host, int64_t* out_capacity_host) {
  TECO_CHECK_ARG(workspace_bytes_host && out_capacity_host, "teco_jpeg_plan_bytes: NULL argument");
  TECO_CHECK_ARG(plan_ok(H, W), "teco_jpeg_plan_bytes: bad frame size %dx%d (1 <= H, W <= %d)", H, W, MAX_SIDE);
  const Plan p = make_plan(H, W);
  *workspace_bytes_host = p.ws_bytes;
  *out_capacity_host = p.out_cap;
  return TECO_OK;
}

int teco_jpeg_encode_rgb8(const uint8_t* rgb, int32_t H, int32_t W, void* workspace, int64_t workspace_bytes, uint8_t* out,
                          int64_t out_capacity, int64_t* out_len, void* stream) {
  TECO_CHECK_ARG(rgb && workspace && out && out_len, "teco_jpeg_encode_rgb8: NULL argument");
  TECO_CHECK_ARG(plan_ok(H, W), "teco_jpeg_encode_rgb8: bad frame size %dx%d (1 <= H, W <= %d)", H, W, MAX_SIDE);
  const Plan p = make_plan(H, W);
  TECO_CHECK_ARG(workspace_bytes >= p.ws_bytes && out_capacity >= p.out_cap,
                 "teco_jpeg_encode_rgb8: buffers of %lld / %lld bytes, the %dx%d plan needs %lld / %lld",
                 (long long)workspace_bytes, (long long)out_capacity, H, W, p.ws_bytes, p.out_cap);
  TECO_CHECK_ARG(((uintptr_t)workspace & 255) == 0, "teco_jpeg_encode_rgb8: workspace must be 256-byte aligned");
  const cudaStream_t st = (cudaStream_t)stream;
  const Bufs u = carve(p, workspace);
  jpeg_blocks<<<dim3((p.mw + G - 1) / G, p.mh), BLK_T, 0, st>>>(rgb, H, W, p, u);
  jpeg_block_bits<<<p.ntile, CODE_T, 0, st>>>(p, u);
  jpeg_scan<<<1, 1024, 0, st>>>(u.tile_bits, u.tile_off, p.ntile, 0, u);
  jpeg_emit<<<p.ntile, CODE_T, 0, st>>>(p, u);
  jpeg_stuff_count<<<p.nstuff, STUFF_T, 0, st>>>(u);
  jpeg_scan<<<1, 1024, 0, st>>>(u.ff_cnt, u.ff_off, 0, 1, u);
  jpeg_assemble<<<p.nstuff, STUFF_T, 0, st>>>(make_header(H, W), out, out_len, u);
  TECO_CUDA_LAUNCH_CHECK("teco_jpeg_encode_rgb8");
  return TECO_OK;
}

}  // extern "C"
