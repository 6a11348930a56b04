// jpeg_encode.cu — baseline JPEG of an 8-bit raster (GRAY8 or BGR8), byte for byte what libjpeg(-turbo) writes with
// its default settings, the standard Huffman tables and jpeg_set_quality(q, force_baseline = TRUE) (convention in
// include/aerial_mapper_b200.h, amb_jpeg_sampling).
//
// One thread per MCU (minimum coded unit: 1 gray block; Y, Cb, Cr at 4:4:4; Y0..Y3, Cb, Cr at 4:2:0), in five steps:
//   measure  every block of the MCU: colour conversion, 2x2 downsampling, islow DCT, quantisation; the quantised DC
//            of each block and the AC bits of the whole MCU are stored (12 + 8 bytes per MCU at 4:2:0)
//   length   the DC bits (prediction from the previous block of the same component in MCU order, 0 at a restart)
//            join the AC bits; exclusive scan -> the bit offset of every MCU
//   segments every restart interval is padded to a byte: its byte length, exclusive scan -> its byte offset
//   pack     every MCU recomputes its blocks and writes its codes at its bit offset into a zeroed word buffer (32-bit
//            words, most significant bit first); the words it shares with its neighbours are combined with atomicAdd,
//            which is an OR here because the bit ranges are disjoint, so the result does not depend on the order; the
//            last MCU of a restart interval pads it with 1 bits
//   stuff    0xFF bytes counted per 4 KB chunk, scan, then a copy that inserts 0x00 after every 0xFF and places
//            RST(n mod 8) in front of restart interval n >= 1
// The JPEG tiles of a Cloud-Optimized GeoTIFF (jpeg_encode.h) replace the last copy by a split: every restart interval,
// stuffed, becomes a stream of its own with a tile header in front and EOI behind, and no RST markers.
// Coefficients are recomputed by the pack step rather than stored: the scratch stays at ~0.08 (4:2:0) / 0.22 (4:4:4)
// byte per pixel plus the compressed stream twice, at any image size.
// Integer widths: every DCT intermediate fits int32 (|pass-1 output| <= 5793 for level-shifted 8-bit samples; the
// largest pass-2 sum of magnitudes is < 1.7e9), so libjpeg's 64-bit JLONG products give the same values.
#include <algorithm>
#include <cstring>

#include "jpeg_encode.h"

namespace amb {
namespace {

constexpr int kMcuThreads = 128;
constexpr int kStuffThreads = 256, kStuffBytes = 16, kStuffChunk = kStuffThreads * kStuffBytes;

#include "block_scan.inc"

// ---- standard tables (ITU-T T.81 Annex K) -----------------------------------------------------------------------------
const uint8_t kLumQuant[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                               14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                               18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                               49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const uint8_t kChromaQuant[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99,
                                  99, 99, 47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
const uint8_t kZigzag[64] =  // natural index of zig-zag position k (host; kZigzagDev on the device)
    {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                             41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                             30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
__constant__ uint8_t kZigzagDev[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                       41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                       30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
const uint8_t kDcLumBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
const uint8_t kDcChromaBits[16] = {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0};
const uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
const uint8_t kAcLumBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
const uint8_t kAcLumVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
    0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
    0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
    0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
    0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
    0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
    0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
    0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
    0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};
const uint8_t kAcChromaBits[16] = {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77};
const uint8_t kAcChromaVals[162] = {
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
    0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
    0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
    0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
    0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
    0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
    0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
    0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// Per-encode constants, passed by value and copied to shared memory by every block of the MCU kernels.
struct JpegTables {
  uint32_t ac[2][256];  // (code length << 16) | code, [0] luma, [1] chroma; indexed by (run << 4) | size
  uint32_t dc[2][16];   // indexed by size
  uint16_t div[2][64];  // quantisation divisors 8 * quantval, natural order
};

struct JpegShape {
  const unsigned char* img;
  unsigned long long stride;    // bytes between image rows
  int32_t w, h;
  int32_t kind;                 // 0 gray, 1 BGR 4:4:4, 2 BGR 4:2:0
  int32_t bpm;                  // blocks per MCU: 1, 3, 6
  int32_t mcus_x;               // MCUs per MCU row
  unsigned long long n_mcu;
  unsigned long long interval;  // restart interval in MCUs, 0 = none
  int32_t y_bw, y_bh;           // 4:2:0: luma width / height in blocks (blocks beyond are dummies)
  int32_t c_rows;               // 4:2:0: ceil(h / 2), the chroma rows downsampled from image rows
};

__device__ __forceinline__ int bit_length(uint32_t a) {
#ifdef AMB_CUDA_EMU
  return a ? 32 - __builtin_clz(a) : 0;
#else
  return 32 - __clz(a);
#endif
}

// jccolor.c rgb_ycc_convert, 16-bit fixed point; comp 0 Y, 1 Cb, 2 Cr of the BGR pixel at p
__device__ __forceinline__ int ycc(const unsigned char* p, int comp) {
  const int b = __ldg(p), g = __ldg(p + 1), r = __ldg(p + 2);
  if (comp == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  if (comp == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// The 8x8 samples (level-shifted) of block (bx, by) of component `comp`.  Edges as libjpeg: image columns and rows are
// replicated to the block / MCU multiple before conversion; at 4:2:0 the chroma plane is the 2x2 average of the
// replicated image with bias 1, 2, 1, 2 ... along each row, and chroma rows past ceil(h / 2) repeat the last one.
__device__ __forceinline__ void load_block(const JpegShape& s, int comp, int bx, int by, int32_t d[64]) {
  const bool sub = s.kind == 2 && comp > 0;
#pragma unroll
  for (int y = 0; y < 8; ++y) {
    int v0, v1 = 0;
    if (sub) {
      const int cy = min(by * 8 + y, s.c_rows - 1);
      v0 = min(2 * cy, s.h - 1);
      v1 = min(2 * cy + 1, s.h - 1);
    } else {
      v0 = min(by * 8 + y, s.h - 1);
    }
    const unsigned char* r0 = s.img + static_cast<unsigned long long>(v0) * s.stride;
    const unsigned char* r1 = s.img + static_cast<unsigned long long>(v1) * s.stride;
#pragma unroll
    for (int x = 0; x < 8; ++x) {
      int v;
      if (s.kind == 0) {
        v = __ldg(r0 + min(bx * 8 + x, s.w - 1));
      } else if (!sub) {
        v = ycc(r0 + 3 * min(bx * 8 + x, s.w - 1), comp);
      } else {
        const int c0 = 3 * min(2 * (bx * 8 + x), s.w - 1), c1 = 3 * min(2 * (bx * 8 + x) + 1, s.w - 1);
        v = (ycc(r0 + c0, comp) + ycc(r0 + c1, comp) + ycc(r1 + c0, comp) + ycc(r1 + c1, comp) + 1 + (x & 1)) >> 2;
      }
      d[y * 8 + x] = v - 128;
    }
  }
}

// jfdctint.c (islow): CONST_BITS 13, PASS1_BITS 2; one 1-D pass over 8 elements of d with the given stride
template <bool LAST>
__device__ __forceinline__ void fdct_pass(int32_t* v, int st) {
  constexpr int SH = LAST ? 15 : 11;
  const int32_t t0 = v[0] + v[7 * st], t7 = v[0] - v[7 * st], t1 = v[st] + v[6 * st], t6 = v[st] - v[6 * st];
  const int32_t t2 = v[2 * st] + v[5 * st], t5 = v[2 * st] - v[5 * st], t3 = v[3 * st] + v[4 * st],
                t4 = v[3 * st] - v[4 * st];
  const int32_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  v[0] = LAST ? (t10 + t11 + 2) >> 2 : (t10 + t11) * 4;
  v[4 * st] = LAST ? (t10 - t11 + 2) >> 2 : (t10 - t11) * 4;
  const int32_t z1 = (t12 + t13) * 4433;
  v[2 * st] = (z1 + t13 * 6270 + (1 << (SH - 1))) >> SH;
  v[6 * st] = (z1 - t12 * 15137 + (1 << (SH - 1))) >> SH;
  const int32_t z5 = (t4 + t6 + t5 + t7) * 9633;
  const int32_t a1 = -(t4 + t7) * 7373, a2 = -(t5 + t6) * 20995, a3 = -(t4 + t6) * 16069 + z5,
                a4 = -(t5 + t7) * 3196 + z5;
  v[7 * st] = (t4 * 2446 + a1 + a3 + (1 << (SH - 1))) >> SH;
  v[5 * st] = (t5 * 16819 + a2 + a4 + (1 << (SH - 1))) >> SH;
  v[3 * st] = (t6 * 25172 + a2 + a3 + (1 << (SH - 1))) >> SH;
  v[st] = (t7 * 12299 + a1 + a4 + (1 << (SH - 1))) >> SH;
}

// Block j of MCU m (dummy blocks included): quantised coefficients in zig-zag order
__device__ __forceinline__ void mcu_block(const JpegShape& s, const JpegTables& t, unsigned long long m, int j,
                                          int32_t q[64]) {
  const int mx = static_cast<int>(m % static_cast<unsigned long long>(s.mcus_x));
  const int my = static_cast<int>(m / static_cast<unsigned long long>(s.mcus_x));
  int comp = s.kind == 0 ? 0 : (s.kind == 1 ? j : max(j - 3, 0));
  int bx = mx, by = my;
  bool dummy = false;
  if (s.kind == 2 && j < 4) {
    bx = 2 * mx + (j & 1);
    by = 2 * my + (j >> 1);
    // jccoefct.c: a dummy block past the right edge takes the DC of its left neighbour; one below the bottom edge
    // takes the DC of the MCU's top-right block, itself a dummy with the top-left DC when the right edge cuts it
    if (by >= s.y_bh) {
      dummy = true;
      by = 2 * my;
      bx = 2 * mx + 1;
    }
    if (bx >= s.y_bw) {
      dummy = true;
      bx -= 1;
    }
  }
  int32_t d[64];
  load_block(s, comp, bx, by, d);
#pragma unroll
  for (int r = 0; r < 8; ++r) fdct_pass<false>(d + 8 * r, 1);
#pragma unroll
  for (int c = 0; c < 8; ++c) fdct_pass<true>(d + c, 8);
  const uint16_t* div = t.div[comp > 0 ? 1 : 0];
#pragma unroll
  for (int k = 0; k < 64; ++k) {
    const int n = kZigzagDev[k];
    const int32_t v = d[n];
    const int32_t dv = div[n];
    const int32_t a = ((v < 0 ? -v : v) + (dv >> 1)) / dv;  // half away from zero, on the magnitude
    q[k] = (k > 0 && dummy) ? 0 : (v < 0 ? -a : a);
  }
}

__device__ __forceinline__ int table_of(const JpegShape& s, int j) { return (s.kind == 2 ? j >= 4 : j > 0) ? 1 : 0; }

// The DC prediction of block j of MCU m: the previous block of the same component in MCU order, 0 at a restart
__device__ __forceinline__ int dc_pred(const JpegShape& s, const int16_t* __restrict__ dc, unsigned long long m, int j) {
  if (s.kind == 2 && j > 0 && j < 4) return dc[m * 6 + j - 1];
  if (m == 0 || (s.interval && m % s.interval == 0)) return 0;
  const int last = s.kind == 2 && j == 0 ? 3 : j;
  return dc[(m - 1) * s.bpm + last];
}

__device__ __forceinline__ uint32_t dc_bits(const JpegTables& t, int tab, int diff) {
  const int n = bit_length(static_cast<uint32_t>(diff < 0 ? -diff : diff));
  return (t.dc[tab][n] >> 16) + n;
}

__device__ __forceinline__ void copy_tables(JpegTables& sm, const JpegTables& t) {
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&t);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&sm);
  for (int i = threadIdx.x; i < static_cast<int>(sizeof(JpegTables) / 4); i += blockDim.x) dst[i] = src[i];
  __syncthreads();
}

// measure: per MCU, the quantised DC of every block and the bits of all AC codes
__global__ void __launch_bounds__(kMcuThreads)
    jpeg_measure_kernel(const JpegShape s, const JpegTables t, int16_t* __restrict__ dc,
                        unsigned long long* __restrict__ bits) {
  __shared__ JpegTables sm;
  copy_tables(sm, t);
  const unsigned long long m = static_cast<unsigned long long>(blockIdx.x) * kMcuThreads + threadIdx.x;
  if (m >= s.n_mcu) return;
  uint32_t total = 0;
  for (int j = 0; j < s.bpm; ++j) {
    int32_t q[64];
    mcu_block(s, sm, m, j, q);
    dc[m * s.bpm + j] = static_cast<int16_t>(q[0]);
    const uint32_t* ac = sm.ac[table_of(s, j)];
    int run = 0;
#pragma unroll
    for (int k = 1; k < 64; ++k) {
      const int32_t v = q[k];
      if (v == 0) {
        ++run;
      } else {
        for (; run > 15; run -= 16) total += ac[0xF0] >> 16;
        const int n = bit_length(static_cast<uint32_t>(v < 0 ? -v : v));
        total += (ac[(run << 4) | n] >> 16) + n;
        run = 0;
      }
    }
    if (run) total += ac[0] >> 16;
  }
  bits[m] = total;
}

// length: the DC bits join the AC bits of every MCU
__global__ void __launch_bounds__(256) jpeg_length_kernel(const JpegShape s, const JpegTables t,
                                                          const int16_t* __restrict__ dc,
                                                          unsigned long long* __restrict__ bits) {
  __shared__ JpegTables sm;
  copy_tables(sm, t);
  const unsigned long long m = static_cast<unsigned long long>(blockIdx.x) * 256 + threadIdx.x;
  if (m >= s.n_mcu) return;
  unsigned long long add = 0;
  for (int j = 0; j < s.bpm; ++j) add += dc_bits(sm, table_of(s, j), dc[m * s.bpm + j] - dc_pred(s, dc, m, j));
  bits[m] += add;
}

// segments: byte length of every restart interval from the MCU bit offsets (mcu_off[n_mcu] = total)
__global__ void jpeg_segment_kernel(const JpegShape s, const unsigned long long* __restrict__ mcu_off,
                                    unsigned long long n_seg, unsigned long long* __restrict__ seg) {
  const unsigned long long k = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k >= n_seg) return;
  const unsigned long long f = s.interval ? k * s.interval : 0ull;
  const unsigned long long e = s.interval && f + s.interval < s.n_mcu ? f + s.interval : s.n_mcu;
  seg[k] = (mcu_off[e] - mcu_off[f] + 7) >> 3;
}

// MSB-first bit writer over 32-bit words; the first and the last word of an MCU may be shared with its neighbours
struct BitSink {
  uint32_t* words;
  unsigned long long w;  // current word
  unsigned long long acc;
  int n;                 // bits in acc, left-aligned (the first n of them belong to earlier MCUs and are 0)
  bool shared;
  __device__ __forceinline__ BitSink(uint32_t* out, unsigned long long pos)
      : words(out), w(pos >> 5), acc(0), n(static_cast<int>(pos & 31)), shared(n != 0) {}
  __device__ __forceinline__ void put(uint32_t code, int len) {  // len 1..27
    acc |= static_cast<unsigned long long>(code & ((1u << len) - 1u)) << (64 - n - len);
    n += len;
    if (n >= 32) {
      const uint32_t v = static_cast<uint32_t>(acc >> 32);
      if (shared)
        atomicAdd(words + w, v);  // disjoint bits: the sum is the OR
      else
        words[w] = v;
      shared = false;
      ++w;
      acc <<= 32;
      n -= 32;
    }
  }
  __device__ __forceinline__ void finish() {
    if (n > 0) atomicAdd(words + w, static_cast<uint32_t>(acc >> 32));
  }
};

__device__ __forceinline__ void put_value(BitSink& o, uint32_t hc, int v, int n) {  // Huffman code, then n value bits
  const int len = static_cast<int>(hc >> 16);
  const uint32_t extra = static_cast<uint32_t>(v < 0 ? v - 1 : v) & ((1u << n) - 1u);
  o.put(((hc & 0xffffu) << n) | extra, len + n);
}

// pack: every MCU writes its codes at 8 * seg_off[segment] + (its bit offset - its segment's first bit offset)
__global__ void __launch_bounds__(kMcuThreads)
    jpeg_pack_kernel(const JpegShape s, const JpegTables t, const int16_t* __restrict__ dc,
                     const unsigned long long* __restrict__ mcu_off, const unsigned long long* __restrict__ seg_off,
                     uint32_t* __restrict__ words) {
  __shared__ JpegTables sm;
  copy_tables(sm, t);
  const unsigned long long m = static_cast<unsigned long long>(blockIdx.x) * kMcuThreads + threadIdx.x;
  if (m >= s.n_mcu) return;
  const unsigned long long sg = s.interval ? m / s.interval : 0ull, f = s.interval ? sg * s.interval : 0ull;
  const unsigned long long pos0 = 8ull * seg_off[sg] + (mcu_off[m] - mcu_off[f]);
  BitSink o(words, pos0);
  for (int j = 0; j < s.bpm; ++j) {
    int32_t q[64];
    mcu_block(s, sm, m, j, q);
    const int tab = table_of(s, j);
    const int diff = q[0] - dc_pred(s, dc, m, j);
    const int nd = bit_length(static_cast<uint32_t>(diff < 0 ? -diff : diff));
    if (nd)
      put_value(o, sm.dc[tab][nd], diff, nd);
    else
      o.put(sm.dc[tab][0] & 0xffffu, static_cast<int>(sm.dc[tab][0] >> 16));
    const uint32_t* ac = sm.ac[tab];
    int run = 0;
#pragma unroll
    for (int k = 1; k < 64; ++k) {
      const int32_t v = q[k];
      if (v == 0) {
        ++run;
      } else {
        for (; run > 15; run -= 16) o.put(ac[0xF0] & 0xffffu, static_cast<int>(ac[0xF0] >> 16));
        const int n = bit_length(static_cast<uint32_t>(v < 0 ? -v : v));
        put_value(o, ac[(run << 4) | n], v, n);
        run = 0;
      }
    }
    if (run) o.put(ac[0] & 0xffffu, static_cast<int>(ac[0] >> 16));
  }
  const bool seg_end = m + 1 == s.n_mcu || (s.interval && (m + 1) % s.interval == 0);
  if (seg_end) {
    const unsigned long long end = pos0 + (mcu_off[m + 1] - mcu_off[m]);
    const int pad = static_cast<int>((8 - (end & 7)) & 7);
    if (pad) o.put(0xffu, pad);  // pending bits are padded with 1s before a marker
  }
  o.finish();
}

__device__ __forceinline__ unsigned int stream_byte(const uint32_t* words, unsigned long long i) {
  return (words[i >> 2] >> (24 - 8 * static_cast<int>(i & 3))) & 0xffu;
}

// stuff, 1: 0xFF bytes of every 4 KB chunk of the stream
__global__ void __launch_bounds__(kStuffThreads)
    jpeg_ff_count_kernel(const uint32_t* __restrict__ words, unsigned long long n_bytes,
                         unsigned long long* __restrict__ counts) {
  const unsigned long long i0 = static_cast<unsigned long long>(blockIdx.x) * kStuffChunk + threadIdx.x * kStuffBytes;
  unsigned long long c = 0;
  for (int k = 0; k < kStuffBytes; ++k)
    if (i0 + k < n_bytes && stream_byte(words, i0 + k) == 0xffu) ++c;
  unsigned long long total;
  block_exclusive<kStuffThreads>(c, &total);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// stuff, 2: byte i goes to i + (0xFF bytes before it) + 2 * (its restart interval); RST markers in front of intervals >= 1
__global__ void __launch_bounds__(kStuffThreads)
    jpeg_stuff_kernel(const uint32_t* __restrict__ words, unsigned long long n_bytes,
                      const unsigned long long* __restrict__ ff_off, const unsigned long long* __restrict__ seg_off,
                      unsigned long long n_seg, unsigned char* __restrict__ out) {
  const unsigned long long i0 = static_cast<unsigned long long>(blockIdx.x) * kStuffChunk + threadIdx.x * kStuffBytes;
  unsigned long long c = 0;
  for (int k = 0; k < kStuffBytes; ++k)
    if (i0 + k < n_bytes && stream_byte(words, i0 + k) == 0xffu) ++c;
  unsigned long long total;
  unsigned long long ff = ff_off[blockIdx.x] + block_exclusive<kStuffThreads>(c, &total);
  if (i0 >= n_bytes) return;
  unsigned long long lo = 0, hi = n_seg - 1;  // the last interval starting at or before i0
  while (lo < hi) {
    const unsigned long long mid = (lo + hi + 1) >> 1;
    if (seg_off[mid] <= i0)
      lo = mid;
    else
      hi = mid - 1;
  }
  unsigned long long sg = lo;
  for (int k = 0; k < kStuffBytes && i0 + k < n_bytes; ++k) {
    const unsigned long long i = i0 + k;
    while (sg + 1 < n_seg && seg_off[sg + 1] <= i) ++sg;
    const unsigned long long p = i + ff + 2 * sg;
    if (sg > 0 && seg_off[sg] == i) {
      out[p - 2] = 0xff;
      out[p - 1] = static_cast<unsigned char>(0xd0 + ((sg - 1) & 7));
    }
    const unsigned int b = stream_byte(words, i);
    out[p] = static_cast<unsigned char>(b);
    if (b == 0xffu) {
      out[p + 1] = 0;
      ++ff;
    }
  }
}

// The constant header of every tile stream of jpeg_split_kernel: SOI, SOF0, SOS
struct TileHead {
  unsigned char b[48];
  int32_t len;
};

// split, 2: byte i of interval sg goes to i + (0xFF bytes before it) + sg * (head.len + 2) + head.len, so that every
// interval becomes a stream of its own: the header in front, EOI behind, no RST marker.  start[sg]: where its stream
// begins (every interval holds at least one byte, so exactly one thread meets its first byte).
__global__ void __launch_bounds__(kStuffThreads)
    jpeg_split_kernel(const uint32_t* __restrict__ words, unsigned long long n_bytes,
                      const unsigned long long* __restrict__ ff_off, const unsigned long long* __restrict__ seg_off,
                      unsigned long long n_seg, const TileHead head, unsigned char* __restrict__ out,
                      unsigned long long* __restrict__ start) {
  const unsigned long long i0 = static_cast<unsigned long long>(blockIdx.x) * kStuffChunk + threadIdx.x * kStuffBytes;
  unsigned long long c = 0;
  for (int k = 0; k < kStuffBytes; ++k)
    if (i0 + k < n_bytes && stream_byte(words, i0 + k) == 0xffu) ++c;
  unsigned long long total;
  unsigned long long ff = ff_off[blockIdx.x] + block_exclusive<kStuffThreads>(c, &total);
  if (i0 >= n_bytes) return;
  unsigned long long lo = 0, hi = n_seg - 1;  // the last interval starting at or before i0
  while (lo < hi) {
    const unsigned long long mid = (lo + hi + 1) >> 1;
    if (seg_off[mid] <= i0)
      lo = mid;
    else
      hi = mid - 1;
  }
  unsigned long long sg = lo;
  const unsigned long long gap = static_cast<unsigned long long>(head.len) + 2;
  for (int k = 0; k < kStuffBytes && i0 + k < n_bytes; ++k) {
    const unsigned long long i = i0 + k;
    while (sg + 1 < n_seg && seg_off[sg + 1] <= i) ++sg;
    const unsigned long long p = i + ff + sg * gap + head.len;
    if (seg_off[sg] == i) {
      for (int j = 0; j < head.len; ++j) out[p - head.len + j] = head.b[j];
      start[sg] = p - head.len;
    }
    const unsigned int b = stream_byte(words, i);
    out[p] = static_cast<unsigned char>(b);
    unsigned long long e = p + 1;
    if (b == 0xffu) {
      out[e++] = 0;
      ++ff;
    }
    if (i + 1 == (sg + 1 < n_seg ? seg_off[sg + 1] : n_bytes)) {  // the interval's last byte: EOI
      out[e] = 0xff;
      out[e + 1] = 0xd9;
    }
  }
}

// the length of every stream of jpeg_split_kernel, `total` bytes in all
__global__ void jpeg_tile_bytes_kernel(const unsigned long long* __restrict__ start, unsigned long long n_seg,
                                       unsigned long long total, uint32_t* __restrict__ len) {
  const unsigned long long k = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (k < n_seg) len[k] = static_cast<uint32_t>((k + 1 < n_seg ? start[k + 1] : total) - start[k]);
}

// ---- host side -------------------------------------------------------------------------------------------------------
// The image's MCU grid, without the 65535 limits of the file format: AMB_OK or AMB_ERR_UNSUPPORTED (channels, quality,
// sampling, a negative interval); w, h > 0 are the caller's to check
int jpeg_shape(int32_t w, int32_t h, int channels, int quality, int sampling, int32_t interval, JpegParams* p) {
  if ((channels != 1 && channels != 3) || quality < 1 || quality > 100 ||
      (sampling != AMB_JPEG_420 && sampling != AMB_JPEG_444) || interval < 0)
    return AMB_ERR_UNSUPPORTED;
  p->w = w;
  p->h = h;
  p->channels = channels;
  p->quality = quality;
  p->sampling = sampling;
  p->interval = interval;
  p->kind = channels == 1 ? 0 : sampling == AMB_JPEG_444 ? 1 : 2;
  p->bpm = p->kind == 0 ? 1 : p->kind == 1 ? 3 : 6;
  const int mcu = p->kind == 2 ? 16 : 8;
  p->mcus_x = (w + mcu - 1) / mcu;
  p->mcus_y = (h + mcu - 1) / mcu;
  p->n_mcu = static_cast<unsigned long long>(p->mcus_x) * static_cast<unsigned long long>(p->mcus_y);
  p->n_seg = interval ? (p->n_mcu + interval - 1) / interval : 1ull;
  return AMB_OK;
}

// AMB_OK, AMB_ERR_INVALID_ARGUMENT (malformed) or AMB_ERR_UNSUPPORTED (outside the supported parameter set)
int jpeg_params(int32_t w, int32_t h, int channels, int quality, int sampling, int32_t interval, JpegParams* p) {
  if (w <= 0 || h <= 0) return AMB_ERR_INVALID_ARGUMENT;
  if (w > 65535 || h > 65535 || interval > 65535) return AMB_ERR_UNSUPPORTED;
  return jpeg_shape(w, h, channels, quality, sampling, interval, p);
}

// jcparam.c jpeg_quality_scaling + jpeg_add_quant_table(force_baseline)
void quant_table(const uint8_t* base, int quality, uint8_t out[64]) {
  const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int k = 0; k < 64; ++k) out[k] = static_cast<uint8_t>(std::min(std::max((base[k] * s + 50) / 100, 1), 255));
}

void huffman_codes(const uint8_t* bits, const uint8_t* vals, uint32_t* table) {
  uint32_t code = 0;
  int k = 0;
  for (int len = 1; len <= 16; ++len) {
    for (int i = 0; i < bits[len - 1]; ++i) table[vals[k++]] = (static_cast<uint32_t>(len) << 16) | code++;
    code <<= 1;
  }
}

void jpeg_tables(const JpegParams& p, JpegTables* t) {
  std::memset(t, 0, sizeof(*t));
  huffman_codes(kDcLumBits, kDcVals, t->dc[0]);
  huffman_codes(kDcChromaBits, kDcVals, t->dc[1]);
  huffman_codes(kAcLumBits, kAcLumVals, t->ac[0]);
  huffman_codes(kAcChromaBits, kAcChromaVals, t->ac[1]);
  uint8_t q[64];
  for (int c = 0; c < 2; ++c) {
    quant_table(c ? kChromaQuant : kLumQuant, p.quality, q);
    for (int k = 0; k < 64; ++k) t->div[c][k] = static_cast<uint16_t>(8 * q[k]);
  }
}

void put16(std::vector<unsigned char>& h, int v) {
  h.push_back(static_cast<unsigned char>(v >> 8));
  h.push_back(static_cast<unsigned char>(v & 0xff));
}

void put_dht(std::vector<unsigned char>& h, int cls_id, const uint8_t* bits, const uint8_t* vals) {
  int n = 0;
  for (int k = 0; k < 16; ++k) n += bits[k];
  h.push_back(0xff);
  h.push_back(0xc4);
  put16(h, 2 + 1 + 16 + n);
  h.push_back(static_cast<unsigned char>(cls_id));
  h.insert(h.end(), bits, bits + 16);
  h.insert(h.end(), vals, vals + n);
}

void put_dqt(std::vector<unsigned char>& h, const JpegParams& p) {  // one DQT per table
  for (int c = 0; c < (p.channels == 3 ? 2 : 1); ++c) {
    uint8_t q[64];
    quant_table(c ? kChromaQuant : kLumQuant, p.quality, q);
    h.push_back(0xff);
    h.push_back(0xdb);
    put16(h, 67);
    h.push_back(static_cast<unsigned char>(c));
    for (int k = 0; k < 64; ++k) h.push_back(q[kZigzag[k]]);
  }
}

void put_sof(std::vector<unsigned char>& h, const JpegParams& p) {
  const int nc = p.channels;
  h.push_back(0xff);
  h.push_back(0xc0);
  put16(h, 8 + 3 * nc);
  h.push_back(8);
  put16(h, p.h);
  put16(h, p.w);
  h.push_back(static_cast<unsigned char>(nc));
  for (int c = 0; c < nc; ++c) {
    h.push_back(static_cast<unsigned char>(c + 1));
    h.push_back(c == 0 && p.kind == 2 ? 0x22 : 0x11);
    h.push_back(c == 0 ? 0 : 1);
  }
}

void put_dhts(std::vector<unsigned char>& h, const JpegParams& p) {  // DC0 AC0 [DC1 AC1]
  put_dht(h, 0x00, kDcLumBits, kDcVals);
  put_dht(h, 0x10, kAcLumBits, kAcLumVals);
  if (p.channels == 3) {
    put_dht(h, 0x01, kDcChromaBits, kDcVals);
    put_dht(h, 0x11, kAcChromaBits, kAcChromaVals);
  }
}

void put_sos(std::vector<unsigned char>& h, const JpegParams& p) {
  const int nc = p.channels;
  h.push_back(0xff);
  h.push_back(0xda);
  put16(h, 6 + 2 * nc);
  h.push_back(static_cast<unsigned char>(nc));
  for (int c = 0; c < nc; ++c) {
    h.push_back(static_cast<unsigned char>(c + 1));
    h.push_back(c == 0 ? 0x00 : 0x11);
  }
  h.push_back(0);
  h.push_back(63);
  h.push_back(0);
}

// SOI, APP0 JFIF 1.01, DQT per table, SOF0, DHT DC0 AC0 [DC1 AC1], DRI if restarts, SOS — libjpeg's order
std::vector<unsigned char> jpeg_header(const JpegParams& p) {
  std::vector<unsigned char> h = {0xff, 0xd8, 0xff, 0xe0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00,
                                  0x01, 0x01, 0x00, 0x00, 0x01, 0x00, 0x01, 0x00, 0x00};
  put_dqt(h, p);
  put_sof(h, p);
  put_dhts(h, p);
  if (p.interval) {
    h.push_back(0xff);
    h.push_back(0xdd);
    put16(h, 4);
    put16(h, p.interval);
  }
  put_sos(h, p);
  return h;
}

unsigned int grid_of(unsigned long long n, int threads) {
  return static_cast<unsigned int>((n + threads - 1) / threads);
}

// The entropy-coded stream before byte stuffing, on the device: what the stuff and split steps read
struct JpegScan {
  const unsigned long long* seg_off;  // byte offset of every interval, n_seg + 1 entries
  const uint32_t* words;              // the stream
  const unsigned long long* ff_off;   // 0xFF bytes before every chunk of kStuffChunk bytes
  unsigned long long n_bytes, n_chunks, n_ff;
};

// measure, length, segments, pack and the 0xFF count of the image at d_img
int jpeg_scan(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, const JpegParams& p, JpegScan* r) {
  JpegShape s;
  s.img = d_img;
  s.stride = row_stride;
  s.w = p.w;
  s.h = p.h;
  s.kind = p.kind;
  s.bpm = p.bpm;
  s.mcus_x = p.mcus_x;
  s.n_mcu = p.n_mcu;
  s.interval = static_cast<unsigned long long>(p.interval);
  s.y_bw = (p.w + 7) / 8;
  s.y_bh = (p.h + 7) / 8;
  s.c_rows = (p.h + 1) / 2;
  JpegTables t;
  jpeg_tables(p, &t);
  cudaStream_t st = ctx->stream;

  // per MCU: DC values, bit lengths -> offsets (+ total), and the scan spine; per interval: byte lengths -> offsets
  const unsigned long long n = p.n_mcu, ns = p.n_seg;
  const size_t dc_bytes = (n * p.bpm * sizeof(int16_t) + 255) & ~size_t(255);
  const size_t off_bytes = ((n + 1) * 8 + 255) & ~size_t(255);
  const size_t seg_bytes = ((ns + 1) * 8 + 255) & ~size_t(255);
  AMB_CUDA(ctx, ctx->jpeg_mcu.reserve(dc_bytes + off_bytes + seg_bytes));
  int16_t* dc = ctx->jpeg_mcu.as<int16_t>();
  unsigned long long* mcu_off = reinterpret_cast<unsigned long long*>(ctx->jpeg_mcu.as<unsigned char>() + dc_bytes);
  unsigned long long* seg_off = reinterpret_cast<unsigned long long*>(ctx->jpeg_mcu.as<unsigned char>() + dc_bytes + off_bytes);
  AMB_CUDA(ctx, ctx->jpeg_spine.reserve(((n + kScanTile - 1) / kScanTile + 1) * 8));  // n >= ns
  unsigned long long* spine = ctx->jpeg_spine.as<unsigned long long>();

  jpeg_measure_kernel<<<grid_of(n, kMcuThreads), kMcuThreads, 0, st>>>(s, t, dc, mcu_off);
  jpeg_length_kernel<<<grid_of(n, 256), 256, 0, st>>>(s, t, dc, mcu_off);
  scan_u64(mcu_off, n, spine, st);
  jpeg_segment_kernel<<<grid_of(ns, 256), 256, 0, st>>>(s, mcu_off, ns, seg_off);
  scan_u64(seg_off, ns, spine, st);
  AMB_CUDA(ctx, cudaGetLastError());
  unsigned long long n_bytes = 0;
  int rc = read_u64(ctx, seg_off + ns, &n_bytes);
  if (rc != AMB_OK) return rc;

  // pack into zeroed words, then count the 0xFF bytes per chunk
  const unsigned long long n_chunks = (n_bytes + kStuffChunk - 1) / kStuffChunk;
  const size_t word_bytes = n_chunks * kStuffChunk + 16;
  AMB_CUDA(ctx, ctx->jpeg_words.reserve(word_bytes + (n_chunks + 1) * 8));
  uint32_t* words = ctx->jpeg_words.as<uint32_t>();
  unsigned long long* ff_off = reinterpret_cast<unsigned long long*>(ctx->jpeg_words.as<unsigned char>() + word_bytes);
  AMB_CUDA(ctx, cudaMemsetAsync(words, 0, word_bytes, st));
  jpeg_pack_kernel<<<grid_of(n, kMcuThreads), kMcuThreads, 0, st>>>(s, t, dc, mcu_off, seg_off, words);
  jpeg_ff_count_kernel<<<static_cast<unsigned int>(n_chunks), kStuffThreads, 0, st>>>(words, n_bytes, ff_off);
  AMB_CUDA(ctx, ctx->jpeg_spine.reserve((n_chunks + kScanTile - 1) / kScanTile * 8 + 8));
  scan_u64(ff_off, n_chunks, ctx->jpeg_spine.as<unsigned long long>(), st);
  AMB_CUDA(ctx, cudaGetLastError());
  unsigned long long n_ff = 0;
  rc = read_u64(ctx, ff_off + n_chunks, &n_ff);
  if (rc != AMB_OK) return rc;
  *r = JpegScan{seg_off, words, ff_off, n_bytes, n_chunks, n_ff};
  return AMB_OK;
}

int jpeg_encode(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, const JpegParams& p, void* host_out,
                size_t capacity, size_t* size) {
  JpegScan r;
  int rc = jpeg_scan(ctx, d_img, row_stride, p, &r);
  if (rc != AMB_OK) return rc;
  const std::vector<unsigned char> header = jpeg_header(p);
  const unsigned long long ns = p.n_seg;
  const size_t data = static_cast<size_t>(r.n_bytes + r.n_ff + 2 * (ns - 1));
  const size_t total = header.size() + data + 2;
  *size = total;
  if (capacity < total) return AMB_ERR_SIZE_MISMATCH;
  cudaStream_t st = ctx->stream;
  AMB_CUDA(ctx, ctx->jpeg_out.reserve(data));
  jpeg_stuff_kernel<<<static_cast<unsigned int>(r.n_chunks), kStuffThreads, 0, st>>>(
      r.words, r.n_bytes, r.ff_off, r.seg_off, ns, ctx->jpeg_out.as<unsigned char>());
  AMB_CUDA(ctx, cudaGetLastError());
  unsigned char* out = static_cast<unsigned char*>(host_out);
  rc = staged_d2h(ctx, out + header.size(), ctx->jpeg_out.ptr, data, st);
  if (rc != AMB_OK) return rc;
  std::memcpy(out, header.data(), header.size());
  out[total - 2] = 0xff;
  out[total - 1] = 0xd9;
  return AMB_OK;
}

}  // namespace

int jpeg_tile_params(int32_t tile, long long n_tiles, int channels, int quality, int sampling, JpegParams* p) {
  if (tile <= 0 || tile % 16 != 0 || n_tiles <= 0 || n_tiles * tile > 0x7fffffffll) return AMB_ERR_UNSUPPORTED;
  const int st = jpeg_shape(tile, static_cast<int32_t>(n_tiles * tile), channels, quality, sampling, 0, p);
  if (st != AMB_OK) return st;
  const int32_t side = tile / (p->kind == 2 ? 16 : 8);  // MCUs along a tile side
  p->interval = side * side;
  p->n_seg = static_cast<unsigned long long>(n_tiles);
  return AMB_OK;
}

unsigned long long jpeg_tiles_bound(const JpegParams& p) {
  // as amb_jpeg_max_size: every interval adds < 1 byte of padding, stuffing at most doubles the bytes; per tile the
  // header and EOI in place of the file's header and RST markers
  const unsigned long long head = 2 + 10 + 3 * p.channels + 8 + 2 * p.channels;  // SOI, SOF0, SOS
  const unsigned long long bytes = (p.n_mcu * p.bpm * (22 + 63 * 26) + 7) / 8 + p.n_seg;
  return 2 * bytes + (head + 2) * p.n_seg;
}

std::vector<unsigned char> jpeg_tables_stream(int channels, int quality) {
  JpegParams p{};
  p.channels = channels;
  p.quality = quality;
  std::vector<unsigned char> h = {0xff, 0xd8};
  put_dqt(h, p);
  put_dhts(h, p);
  h.push_back(0xff);
  h.push_back(0xd9);
  return h;
}

int jpeg_tiles_encode(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, const JpegParams& p,
                      void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes) {
  JpegScan r;
  int rc = jpeg_scan(ctx, d_img, row_stride, p, &r);
  if (rc != AMB_OK) return rc;
  JpegParams tp = p;  // the header of one tile: SOI, SOF0 (tile x tile), SOS
  tp.h = p.w;
  std::vector<unsigned char> h = {0xff, 0xd8};
  put_sof(h, tp);
  put_sos(h, tp);
  TileHead head;
  std::memcpy(head.b, h.data(), h.size());
  head.len = static_cast<int32_t>(h.size());
  const unsigned long long ns = p.n_seg;
  const size_t total = static_cast<size_t>(r.n_bytes + r.n_ff + ns * (h.size() + 2));
  *size = total;
  if (capacity < total) return AMB_ERR_SIZE_MISMATCH;
  cudaStream_t st = ctx->stream;
  const size_t data_bytes = (total + 255) & ~size_t(255);
  AMB_CUDA(ctx, ctx->jpeg_out.reserve(data_bytes + ns * 8 + ns * 4));
  unsigned char* out = ctx->jpeg_out.as<unsigned char>();
  unsigned long long* start = reinterpret_cast<unsigned long long*>(out + data_bytes);
  uint32_t* lens = reinterpret_cast<uint32_t*>(start + ns);
  jpeg_split_kernel<<<static_cast<unsigned int>(r.n_chunks), kStuffThreads, 0, st>>>(r.words, r.n_bytes, r.ff_off,
                                                                                     r.seg_off, ns, head, out, start);
  jpeg_tile_bytes_kernel<<<grid_of(ns, 256), 256, 0, st>>>(start, ns, total, lens);
  AMB_CUDA(ctx, cudaGetLastError());
  rc = staged_d2h(ctx, host_out, out, total, st);
  if (rc != AMB_OK) return rc;
  return staged_d2h(ctx, tile_bytes, lens, static_cast<size_t>(ns) * 4, st);
}

}  // namespace amb

using namespace amb;

extern "C" {

size_t amb_jpeg_max_size(int32_t width, int32_t height, int channels, int quality, int sampling,
                         int32_t restart_interval) {
  JpegParams p;
  if (jpeg_params(width, height, channels, quality, sampling, restart_interval, &p) != AMB_OK) return 0;
  // a block codes at most 11 + 11 DC bits and 63 AC codes of <= 16 + 10 bits; every interval adds < 1 byte of padding;
  // stuffing at most doubles the bytes; 2 marker bytes per restart, 2 for EOI
  const unsigned long long blocks = p.n_mcu * p.bpm;
  const unsigned long long bytes = (blocks * (22 + 63 * 26) + 7) / 8 + p.n_seg;
  return jpeg_header(p).size() + static_cast<size_t>(2 * bytes + 2 * p.n_seg + 2);
}

int amb_jpeg_encode_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                           int channels, int quality, int sampling, int32_t restart_interval, void* host_out,
                           size_t capacity, size_t* size) {
  if (!ctx || !d_image || !host_out || !size) return AMB_ERR_INVALID_ARGUMENT;
  JpegParams p;
  const int st = jpeg_params(width, height, channels, quality, sampling, restart_interval, &p);
  if (st != AMB_OK) return st;
  if (row_stride < static_cast<size_t>(width) * channels) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return jpeg_encode(ctx, static_cast<const unsigned char*>(d_image), row_stride, p, host_out, capacity, size);
}

int amb_export_jpeg(amb_ctx* ctx, int layer, int format, int quality, int sampling, int32_t restart_interval,
                    void* host_out, size_t capacity, size_t* size) {
  if (!ctx || !host_out || !size || layer < 0 || layer >= AMB_NUM_LAYERS ||
      (format != AMB_RASTER_GRAY8 && format != AMB_RASTER_BGR8))
    return AMB_ERR_INVALID_ARGUMENT;
  const int channels = format == AMB_RASTER_BGR8 ? 3 : 1;
  JpegParams p;
  const int st = jpeg_params(ctx->geom.rows, ctx->col_end - ctx->col_begin, channels, quality, sampling,
                             restart_interval, &p);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t stride = static_cast<size_t>(ctx->geom.rows) * channels;
  AMB_CUDA(ctx, ctx->raster_band.reserve(ctx->slab_cells() * channels));
  const int rc = amb_export_raster_device(ctx, layer, format, ctx->raster_band.ptr);
  if (rc != AMB_OK) return rc;
  return jpeg_encode(ctx, ctx->raster_band.as<unsigned char>(), stride, p, host_out, capacity, size);
}

}  // extern "C"
