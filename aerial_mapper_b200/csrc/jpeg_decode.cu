// jpeg_decode.cu — sequential Huffman JPEG files (1 or 3 components, 4:4:4 / 4:2:2 / 4:2:0) decoded on the device into
// 8-bit rasters, pixel for pixel what cv2.imread returns (convention in include/aerial_mapper_b200.h, "JPEG frames
// decoded on the device"; the header parser is jpeg_header.cc).
//
// The frames of a group go through one launch chain:
//   unstuff  per 4 KB chunk of every scan: the end of the scan (the first marker other than RSTn), then
//            0xFF 0x00 -> 0xFF and RSTn dropped, counted per chunk, one scan over all chunks, then copied; every RSTn
//            records the start of its restart segment in the unstuffed stream and is checked against its sequence
//            number
//   sync     every restart segment is cut into subsequences of kSubBits bits; a decoder state is (bit position, block
//            of the MCU, zig-zag index k) at a codeword boundary.  The entry state of a segment's first subsequence is
//            known; the others start from a guess (their first bit, block 0, k 0).  Each launch decodes every
//            subsequence from its entry state; at the next subsequence's start it compares its state with the one
//            recorded there, and if they differ records its own and carries on into that subsequence (Weißenberger &
//            Schmidt, ICPP 2018).  A launch that changes nothing ends the iteration: then every entry state follows
//            from its segment's known start, so they are all true.  Launch t makes entry t of every segment true, so
//            the iteration ends whatever the input, in the worst case as a sequential decode.  Errors met from a
//            guessed state only change the state recorded (invalid); they are not errors of the stream.
//   count    blocks started and DC differences per component in every subsequence; exclusive scans, taken relative to
//            the segment's first subsequence, give each subsequence its first block and its DC predictors (0 at a
//            restart; libjpeg's int predictor, summed modulo 2^32, stored as a 16-bit coefficient)
//   write    the true parse once more, each coefficient stored at its block (MCU order) in natural order; only this
//            pass reports corruption: a code no table holds, a run past coefficient 63, a segment whose MCUs need more
//            bits than it has (bits past the last MCU are ignored, as libjpeg does)
//   idct     one thread per block of the MCU rows asked for: dequantisation and the islow IDCT (jidctint.c, in the
//            16-bit lanes of libjpeg-turbo's SIMD code, see below), into one 8-bit plane per component
//   colour   one thread per output pixel: jdsample.c's fancy upsampling (triangle filters, box replication when the
//            chroma plane is at most 2 samples wide) and jdcolor.c's YCbCr -> BGR, Y alone for gray output, the gray
//            value three times for BGR output of a gray file
// Scratch per frame (kept by the context): the file, its unstuffed scan, 128 bytes of coefficients and 64 bytes of
// planes per block (dummy blocks of partial MCUs included), 80 bytes per subsequence (1 KB of scan).  Frames are
// grouped so that one group's scratch stays under kGroupBudget (a frame larger than the budget forms a group of its
// own).
#include <algorithm>
#include <cstring>
#include <vector>

#include "amb_context.h"
#include "jpeg_header.h"

namespace amb {
namespace {

#include "block_scan.inc"

constexpr int kChunkThreads = 256, kChunkBytes = 16, kChunk = kChunkThreads * kChunkBytes;
constexpr int kSubBits = 8192;          // bits per subsequence (2048: 2.2x the time per frame, host tables)
constexpr int kSyncHops = 32;           // subsequences a decoder may carry on into per sync launch
constexpr int kSyncLaunchesPerRead = 4; // sync launches queued between two reads of the change counters
constexpr size_t kGroupBudget = size_t(1) << 30;
constexpr uint64_t kInvalid = ~0ull;
constexpr uint32_t kNoSegment = 0xffffffffu;

__constant__ uint8_t kNaturalDev[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,
                                        12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
                                        35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
                                        58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

struct DecTable {
  uint16_t look[256];   // (length << 8) | symbol of the code the next 8 bits start with; 0: a longer code
  int32_t maxcode[17];  // [l]: the largest code of length l, -1 if none
  int32_t valoff[17];   // [l]: index in vals of the first code of length l, minus that code
  uint8_t vals[256];
};

struct DecFrame {
  DecTable dc[3], ac[3];     // per component
  uint16_t quant[3][64];     // per component, natural order
  int32_t width, height, ncomp, hmax, vmax, bpm, mcus_x, mcus_y;
  int32_t blk_comp[6], blk_dx[6], blk_dy[6];  // block j of an MCU: component, block offset in the MCU
  int32_t plane_w[3];        // bytes per plane row (MCU-padded)
  int32_t ri;                // restart interval in MCUs (n_mcu when there is none)
  int32_t n_seg;
  uint32_t seg_base;         // first of this frame's n_seg + 1 entries in the segment-start table (the last one: where
                             // an RSTn past the last segment's start ends it, if the scan has one)
  int32_t channels;          // output: 1 or 3
  int32_t row0, row1;        // output rows [row0, row1) (row0 is the first row written at `out`)
  int32_t mcu_row0, mcu_row1;  // MCU rows reconstructed
  unsigned long long n_mcu;
  unsigned long long file_off, scan_begin, scan_end;  // in the group's file buffer
  unsigned long long ub_off;   // the unstuffed scan in the group's stream buffer
  unsigned long long coef_off; // first block in the coefficient buffer
  unsigned long long plane_off[3];
  unsigned char* out;
  unsigned long long row_step;
};

struct SubInfo {
  unsigned long long begin;  // first bit (relative to the frame's unstuffed scan)
  unsigned long long end;    // first bit of the next subsequence, or the segment's end
  uint32_t frame, seg, first;  // first: index of the segment's first subsequence
  uint32_t last;             // the segment's last subsequence
};

__host__ __device__ __forceinline__ unsigned long long pack_state(unsigned long long pos, int j, int k) {
  return (pos << 16) | (static_cast<unsigned long long>(j) << 8) | static_cast<unsigned long long>(k);
}

// MSB-first reader of a frame's unstuffed scan; bytes past its end read as 0 (they are only ever reached from a guessed
// state, or by a segment that is short of bits, which the write pass reports)
struct Bits {
  const unsigned char* p;
  unsigned long long n, next, buf, pos;
  int nb;
  __device__ __forceinline__ Bits(const unsigned char* data, unsigned long long bytes, unsigned long long bit)
      : p(data), n(bytes), next(bit >> 3), buf(0), pos(bit), nb(0) {
    fill();
    const int s = static_cast<int>(bit & 7);
    buf <<= s;
    nb -= s;
  }
  __device__ __forceinline__ void fill() {
    while (nb <= 56) {
      const unsigned long long b = next < n ? p[next] : 0ull;
      ++next;
      buf |= b << (56 - nb);
      nb += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int k) const { return static_cast<uint32_t>(buf >> (64 - k)); }
  __device__ __forceinline__ void skip(int k) {
    buf <<= k;
    nb -= k;
    pos += k;
  }
};

// the next symbol of table t, -1 if no code matches
__device__ __forceinline__ int huff_decode(const DecTable& t, Bits& br) {
  const uint32_t lk = t.look[br.peek(8)];
  if (lk) {
    br.skip(static_cast<int>(lk >> 8));
    return static_cast<int>(lk & 0xff);
  }
  const int32_t code16 = static_cast<int32_t>(br.peek(16));
  for (int l = 9; l <= 16; ++l) {
    const int32_t c = code16 >> (16 - l);
    if (c <= t.maxcode[l]) {
      br.skip(l);
      const int32_t idx = c + t.valoff[l];
      return (idx >= 0 && idx < 256) ? t.vals[idx] : -1;
    }
  }
  return -1;
}

__device__ __forceinline__ int extend(Bits& br, int s) {  // s value bits, 1..15 (HUFF_EXTEND)
  const int r = static_cast<int>(br.peek(s));
  br.skip(s);
  return r < (1 << (s - 1)) ? r - (1 << s) + 1 : r;
}

// One codeword of block j (coefficient k) with its value bits.  Returns false on a code no table holds or a run past
// coefficient 63.  On a DC code *dc = the difference, *kout = 0; on a non-zero AC coefficient *kout = its zig-zag index
// and *v its value; otherwise *kout = -1.  A finished block moves j on and resets k.
__device__ __forceinline__ bool decode_step(const DecFrame& F, Bits& br, int& j, int& k, int* kout, int* v) {
  br.fill();
  const int c = F.blk_comp[j];
  *kout = -1;
  if (k == 0) {
    const int s = huff_decode(F.dc[c], br);
    if (s < 0 || s > 15) return false;
    *v = s ? extend(br, s) : 0;
    *kout = 0;
    k = 1;
  } else {
    const int rs = huff_decode(F.ac[c], br);
    if (rs < 0) return false;
    const int r = rs >> 4, s = rs & 15;
    if (s) {
      k += r;
      if (k > 63) return false;
      *v = extend(br, s);
      *kout = k;
      ++k;
    } else if (r == 15) {
      k += 16;
      if (k > 64) return false;
    } else {
      k = 64;  // EOB
    }
  }
  if (k == 64) {
    k = 0;
    j = j + 1 == F.bpm ? 0 : j + 1;
  }
  return true;
}

// ---- unstuff ------------------------------------------------------------------------------------------------------
struct ChunkInfo {
  unsigned long long begin, end;  // bytes of the group's file buffer (within one scan)
  uint32_t frame, pad_;
};

__device__ __forceinline__ bool is_rst(unsigned int b) { return b >= 0xd0 && b <= 0xd7; }

// the scan ends at the code byte of its first marker other than RSTn (0xFF 0xFF are fill bytes)
__global__ void __launch_bounds__(kChunkThreads)
    jdec_scan_end_kernel(const unsigned char* __restrict__ files, const ChunkInfo* __restrict__ chunks,
                         const DecFrame* __restrict__ frames, unsigned long long* __restrict__ scan_end) {
  const ChunkInfo ck = chunks[blockIdx.x];
  const unsigned long long i0 = ck.begin + threadIdx.x * kChunkBytes;
  const unsigned long long first = frames[ck.frame].scan_begin;
  for (int q = 0; q < kChunkBytes; ++q) {
    const unsigned long long i = i0 + q;
    if (i >= ck.end) break;
    const unsigned int b = files[i];
    if (i > first && files[i - 1] == 0xffu && b != 0 && b != 0xffu && !is_rst(b)) {
      atomicMin(scan_end + ck.frame, i - 1);
      break;
    }
  }
}

// per thread: (RST markers << 40) | bytes kept, of its kChunkBytes bytes before `end` (the chunk's end or the scan's);
// scan_end bounds the look at the next byte
__device__ __forceinline__ unsigned long long unstuff_count(const unsigned char* files, unsigned long long i0,
                                                            unsigned long long end, unsigned long long scan_end,
                                                            unsigned long long first) {
  unsigned long long kept = 0, rst = 0;
  for (int q = 0; q < kChunkBytes; ++q) {
    const unsigned long long i = i0 + q;
    if (i >= end) break;
    const unsigned int b = files[i];
    if (b == 0xffu) {
      if (i + 1 < scan_end && files[i + 1] == 0) ++kept;
    } else if (i > first && files[i - 1] == 0xffu) {
      if (is_rst(b)) ++rst;
    } else {
      ++kept;
    }
  }
  return (rst << 40) | kept;
}

__global__ void __launch_bounds__(kChunkThreads)
    jdec_unstuff_count_kernel(const unsigned char* __restrict__ files, const ChunkInfo* __restrict__ chunks,
                              const DecFrame* __restrict__ frames, const unsigned long long* __restrict__ scan_end,
                              unsigned long long* __restrict__ counts) {
  const ChunkInfo ck = chunks[blockIdx.x];
  const unsigned long long se = scan_end[ck.frame], end = ck.end < se ? ck.end : se;
  const unsigned long long c =
      unstuff_count(files, ck.begin + threadIdx.x * kChunkBytes, end, se, frames[ck.frame].scan_begin);
  unsigned long long total;
  block_exclusive<kChunkThreads>(c, &total);
  if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kChunkThreads)
    jdec_unstuff_copy_kernel(const unsigned char* __restrict__ files, const ChunkInfo* __restrict__ chunks,
                             const DecFrame* __restrict__ frames, const unsigned long long* __restrict__ scan_end,
                             const unsigned long long* __restrict__ offsets, const uint32_t* __restrict__ first_chunk,
                             unsigned char* __restrict__ ub, uint32_t* __restrict__ seg_start,
                             unsigned int* __restrict__ bad) {
  const ChunkInfo ck = chunks[blockIdx.x];
  const DecFrame& F = frames[ck.frame];
  const unsigned long long se = scan_end[ck.frame], end = ck.end < se ? ck.end : se;
  const unsigned long long i0 = ck.begin + threadIdx.x * kChunkBytes;
  const unsigned long long c = unstuff_count(files, i0, end, se, F.scan_begin);
  unsigned long long total;
  const unsigned long long at = offsets[blockIdx.x] + block_exclusive<kChunkThreads>(c, &total) -
                                offsets[first_chunk[ck.frame]];
  unsigned long long kept = at & ((1ull << 40) - 1), rst = at >> 40;
  unsigned char* out = ub + F.ub_off;
  for (int q = 0; q < kChunkBytes; ++q) {
    const unsigned long long i = i0 + q;
    if (i >= end) break;
    const unsigned int b = files[i];
    if (b == 0xffu) {
      if (i + 1 < se && files[i + 1] == 0) out[kept++] = 0xff;
    } else if (i > F.scan_begin && files[i - 1] == 0xffu) {
      if (is_rst(b)) {
        // RST number rst (0-based) opens segment rst + 1.  The first one past them ends the last segment, as libjpeg
        // stops its entropy data at any marker: MCUs that need bits beyond it are corrupt, an RST written after the
        // last MCU is not.  Later ones lie in data that is ignored.
        if (rst + 1 < static_cast<unsigned long long>(F.n_seg)) {
          seg_start[F.seg_base + rst + 1] = static_cast<uint32_t>(kept);
          if ((b & 7u) != (rst & 7u)) atomicMax(bad + ck.frame, 1u);
        } else if (rst + 1 == static_cast<unsigned long long>(F.n_seg)) {
          seg_start[F.seg_base + F.n_seg] = static_cast<uint32_t>(kept);
        }
        ++rst;
      }
    } else {
      out[kept++] = static_cast<unsigned char>(b);
    }
  }
}

// ---- entropy decode ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
    jdec_sync_kernel(const DecFrame* __restrict__ frames, const SubInfo* __restrict__ subs, unsigned long long n_sub,
                     const unsigned char* __restrict__ ub, const unsigned long long* __restrict__ ub_len,
                     unsigned long long* entry, unsigned int* counters, int iter) {
  if (iter > 0 && *reinterpret_cast<volatile unsigned int*>(counters + iter - 1) == 0) return;  // converged
  const unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_sub) return;
  const SubInfo si = subs[i];
  if (si.last) return;  // nothing after it in its segment
  const DecFrame& F = frames[si.frame];
  unsigned long long st = *reinterpret_cast<volatile unsigned long long*>(entry + i);
  unsigned long long t = i + 1;
  if (st == kInvalid) {
    if (*reinterpret_cast<volatile unsigned long long*>(entry + t) != kInvalid) {
      entry[t] = kInvalid;
      atomicAdd(counters + iter, 1u);
    }
    return;
  }
  Bits br(ub + F.ub_off, ub_len[si.frame], st >> 16);
  int j = static_cast<int>((st >> 8) & 0xff), k = static_cast<int>(st & 0xff);
  if (j >= F.bpm || k > 63) j = k = 0;
  for (int hop = 0; hop < kSyncHops; ++hop) {
    const unsigned long long stop = subs[t].begin;
    bool ok = true;
    while (br.pos < stop) {
      int kk, v;
      if (!decode_step(F, br, j, k, &kk, &v)) {
        ok = false;
        break;
      }
    }
    const unsigned long long now = ok ? pack_state(br.pos, j, k) : kInvalid;
    if (*reinterpret_cast<volatile unsigned long long*>(entry + t) == now) break;  // synchronised
    entry[t] = now;
    atomicAdd(counters + iter, 1u);
    if (!ok || subs[t].last) break;
    ++t;
  }
}

// blocks started and DC differences per component in every subsequence (the last one of a segment: 0)
__global__ void __launch_bounds__(128)
    jdec_count_kernel(const DecFrame* __restrict__ frames, const SubInfo* __restrict__ subs, unsigned long long n_sub,
                      const unsigned char* __restrict__ ub, const unsigned long long* __restrict__ ub_len,
                      const unsigned long long* __restrict__ entry, unsigned long long* __restrict__ sums) {
  const unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_sub) return;
  const SubInfo si = subs[i];
  unsigned long long blocks = 0, dc[3] = {0, 0, 0};
  const unsigned long long st = entry[i];
  if (!si.last && st != kInvalid) {
    const DecFrame& F = frames[si.frame];
    Bits br(ub + F.ub_off, ub_len[si.frame], st >> 16);
    int j = static_cast<int>((st >> 8) & 0xff), k = static_cast<int>(st & 0xff);
    if (j < F.bpm && k <= 63) {
      while (br.pos < si.end) {
        const int c = F.blk_comp[j];
        int kk, v;
        if (!decode_step(F, br, j, k, &kk, &v)) break;
        if (kk == 0) {
          ++blocks;
          dc[c] += static_cast<unsigned long long>(static_cast<long long>(v));
        }
      }
    }
  }
  sums[i] = blocks;
  sums[(n_sub + 1) + i] = dc[0];
  sums[2 * (n_sub + 1) + i] = dc[1];
  sums[3 * (n_sub + 1) + i] = dc[2];
}

__global__ void __launch_bounds__(128)
    jdec_write_kernel(const DecFrame* __restrict__ frames, const SubInfo* __restrict__ subs, unsigned long long n_sub,
                      const unsigned char* __restrict__ ub, const unsigned long long* __restrict__ ub_len,
                      const unsigned long long* __restrict__ entry, const unsigned long long* __restrict__ sums,
                      int16_t* __restrict__ coef, unsigned int* __restrict__ bad) {
  const unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n_sub) return;
  const SubInfo si = subs[i];
  const unsigned long long st = entry[i];
  if (st == kInvalid) return;  // a true parse that failed before here has been reported where it failed
  const DecFrame& F = frames[si.frame];
  const unsigned long long m0 = static_cast<unsigned long long>(si.seg) * F.ri;
  const unsigned long long seg_blocks = static_cast<unsigned long long>(F.bpm) *
                                        (F.n_mcu - m0 < static_cast<unsigned long long>(F.ri) ? F.n_mcu - m0 : F.ri);
  int j = static_cast<int>((st >> 8) & 0xff), k = static_cast<int>(st & 0xff);
  const unsigned long long before = sums[i] - sums[si.first];
  if (j >= F.bpm || k > 63 || (k > 0 && before == 0)) return;  // not a state a true parse reaches
  unsigned long long b = before - (k > 0 ? 1 : 0);  // the block being decoded (relative to the segment)
  if (b >= seg_blocks) return;                      // data after the segment's last MCU
  if (b % F.bpm != static_cast<unsigned long long>(j)) {
    atomicMax(bad + si.frame, 2u);
    return;
  }
  uint32_t dc[3];
  for (int c = 0; c < 3; ++c)
    dc[c] = static_cast<uint32_t>(sums[(c + 1) * (n_sub + 1) + i] - sums[(c + 1) * (n_sub + 1) + si.first]);
  Bits br(ub + F.ub_off, ub_len[si.frame], st >> 16);
  int16_t* blk = coef + (F.coef_off + m0 * F.bpm + b) * 64;
  while (si.last || br.pos < si.end) {
    const int c = F.blk_comp[j];
    int kk, v;
    if (br.pos > si.end || !decode_step(F, br, j, k, &kk, &v)) {
      atomicMax(bad + si.frame, 2u);
      return;
    }
    if (kk == 0) {
      dc[c] += static_cast<uint32_t>(v);
      blk[0] = static_cast<int16_t>(static_cast<int32_t>(dc[c]));
    } else if (kk > 0) {
      blk[kNaturalDev[kk]] = static_cast<int16_t>(v);
    }
    if (k == 0) {  // the block is complete
      ++b;
      blk += 64;
      if (b == seg_blocks) break;
    }
  }
  if (si.last && br.pos > si.end) atomicMax(bad + si.frame, 2u);  // the segment's MCUs need more bits than it has
}

// ---- reconstruction -------------------------------------------------------------------------------------------------
// The islow IDCT as libjpeg-turbo's x86 SIMD code computes it (jsimd_idct_islow, what OpenCV's builds run):
// jidctint.c's arithmetic, with the products of jidctint.c regrouped into pairs (exact), but with 16-bit lanes where
// that code has them: dequantised coefficients, the sums z2 + z3, z2 - z3, tmp0 + tmp2 and tmp1 + tmp3, and the pass-1
// workspace (saturated); a block whose AC rows 1..7 are all zero takes pass 1's shortcut (DC << PASS1_BITS in 16 bits);
// the outputs saturate to 0..255.  Wherever no intermediate leaves 16 bits (every stream an encoder writes from 8-bit
// samples) this is exactly jidctint.c, its `& RANGE_MASK` limit included; elsewhere (corrupt or synthetic coefficients)
// it is what cv2.imread returns.
__device__ __forceinline__ int32_t w16(int32_t v) { return static_cast<int16_t>(static_cast<uint16_t>(v & 0xffff)); }
__device__ __forceinline__ int32_t s16(int32_t v) { return min(max(v, -32768), 32767); }

// One 1-D pass over 8 values of 16 bits.  The arithmetic is the SIMD code's 32-bit lanes (pmaddwd, paddd: products of
// 16-bit values and constants, sums wrapping modulo 2^32), so it is done in uint32; SH: the descale shift (psrad).
template <int SH>
__device__ __forceinline__ void idct_pass(const int32_t* in, int32_t* out) {
  using u32 = uint32_t;
  auto mul = [](int32_t v, int32_t c) { return static_cast<u32>(v * c); };  // |v| <= 2^15, |c| < 2^15: no overflow
  const int32_t z2 = in[2], z3 = in[6];
  const u32 tmp3 = mul(z2, 4433 + 6270) + mul(z3, 4433), tmp2 = mul(z2, 4433) + mul(z3, 4433 - 15137);
  const u32 t0 = static_cast<u32>(w16(in[0] + in[4])) << 13, t1 = static_cast<u32>(w16(in[0] - in[4])) << 13;
  const u32 tmp10 = t0 + tmp3, tmp13 = t0 - tmp3, tmp11 = t1 + tmp2, tmp12 = t1 - tmp2;
  const int32_t o0 = in[7], o1 = in[5], o2 = in[3], o3 = in[1];
  const int32_t z3o = w16(o0 + o2), z4o = w16(o1 + o3);
  const u32 za = mul(z3o, 9633 - 16069) + mul(z4o, 9633), zb = mul(z3o, 9633) + mul(z4o, 9633 - 3196);
  const u32 a0 = mul(o0, 2446 - 7373) + mul(o3, -7373) + za, a3 = mul(o0, -7373) + mul(o3, 12299 - 7373) + zb;
  const u32 a1 = mul(o1, 16819 - 20995) + mul(o2, -20995) + zb, a2 = mul(o1, -20995) + mul(o2, 25172 - 20995) + za;
  constexpr u32 r = 1u << (SH - 1);
  out[0] = static_cast<int32_t>(tmp10 + a3 + r) >> SH;
  out[7] = static_cast<int32_t>(tmp10 - a3 + r) >> SH;
  out[1] = static_cast<int32_t>(tmp11 + a2 + r) >> SH;
  out[6] = static_cast<int32_t>(tmp11 - a2 + r) >> SH;
  out[2] = static_cast<int32_t>(tmp12 + a1 + r) >> SH;
  out[5] = static_cast<int32_t>(tmp12 - a1 + r) >> SH;
  out[3] = static_cast<int32_t>(tmp13 + a0 + r) >> SH;
  out[4] = static_cast<int32_t>(tmp13 - a0 + r) >> SH;
}

// one thread per block of the frame's MCU rows [mcu_row0, mcu_row1); thread blocks [f * tiles, (f + 1) * tiles) serve
// frame f
__global__ void __launch_bounds__(128)
    jdec_idct_kernel(const DecFrame* __restrict__ frames, unsigned int tiles, const int16_t* __restrict__ coef,
                     unsigned char* __restrict__ planes, const unsigned int* __restrict__ bad) {
  const unsigned int f = blockIdx.x / tiles, tile = blockIdx.x % tiles;
  const DecFrame& F = frames[f];
  if (bad[f]) return;
  const unsigned long long b0 = static_cast<unsigned long long>(F.mcu_row0) * F.mcus_x * F.bpm;
  const unsigned long long b = b0 + static_cast<unsigned long long>(tile) * blockDim.x + threadIdx.x;
  if (b >= static_cast<unsigned long long>(F.mcu_row1) * F.mcus_x * F.bpm) return;
  const int jb = static_cast<int>(b % F.bpm);
  const unsigned long long m = b / F.bpm;
  const int mx = static_cast<int>(m % F.mcus_x), my = static_cast<int>(m / F.mcus_x);
  const int c = F.blk_comp[jb];
  if (c > 0 && F.channels == 1) return;  // gray output reads Y only
  const int bx = mx * (c ? 1 : F.hmax) + F.blk_dx[jb], by = my * (c ? 1 : F.vmax) + F.blk_dy[jb];
  const int16_t* in = coef + (F.coef_off + b) * 64;
  const uint16_t* q = F.quant[c];
  int32_t ws[64], v[8], o[8];
  bool ac = false;
  for (int k = 8; k < 64; ++k) ac |= in[k] != 0;
  for (int col = 0; col < 8; ++col) {
    for (int r = 0; r < 8; ++r)
      v[r] = w16(static_cast<int32_t>(static_cast<uint32_t>(in[r * 8 + col]) * q[r * 8 + col]));
    if (!ac) {
      for (int r = 0; r < 8; ++r) ws[r * 8 + col] = w16(v[0] * 4);
      continue;
    }
    idct_pass<11>(v, o);  // CONST_BITS - PASS1_BITS
    for (int r = 0; r < 8; ++r) ws[r * 8 + col] = s16(o[r]);
  }
  unsigned char* dst = planes + F.plane_off[c] + static_cast<unsigned long long>(by) * 8 * F.plane_w[c] + bx * 8;
  for (int r = 0; r < 8; ++r) {
    idct_pass<18>(ws + r * 8, o);  // CONST_BITS + PASS1_BITS + 3
    for (int x = 0; x < 8; ++x)
      dst[static_cast<unsigned long long>(r) * F.plane_w[c] + x] =
          static_cast<unsigned char>(min(max(o[x], -128), 127) + 128);
  }
}

// jdsample.c: chroma sample of output pixel (x, y) from the plane p of cw x ch samples (ratios hr x vr of 1 or 2)
__device__ __forceinline__ int upsample(const unsigned char* p, int pw, int cw, int ch, int hr, int vr, int x, int y) {
  const int cx = x / hr, cy = y / vr;
  if (hr == 1 && vr == 1) return p[static_cast<long long>(cy) * pw + cx];
  if (cw <= 2) return p[static_cast<long long>(cy) * pw + cx];  // box replication (h2v1_upsample / h2v2_upsample)
  auto at = [&](int yy, int xx) {
    xx = min(max(xx, 0), cw - 1);
    return static_cast<int>(p[static_cast<long long>(yy) * pw + xx]);
  };
  const int dx = (x & 1) ? 1 : -1;
  if (vr == 1) {  // h2v1: 3/4 nearer + 1/4 further, biases 1 (even) and 2 (odd)
    return (at(cy, cx) * 3 + at(cy, cx + dx) + ((x & 1) ? 2 : 1)) >> 2;
  }
  // h2v2: column sums 3 * nearer row + further row, then 3/4 nearer column sum + 1/4 further, biases 8 and 7
  const int far = min(max(cy + ((y & 1) ? 1 : -1), 0), ch - 1);
  const int s0 = at(cy, cx) * 3 + at(far, cx), s1 = at(cy, cx + dx) * 3 + at(far, cx + dx);
  return (s0 * 3 + s1 + ((x & 1) ? 7 : 8)) >> 4;
}

__device__ __forceinline__ unsigned char clamp255(int v) { return static_cast<unsigned char>(min(max(v, 0), 255)); }

// one thread per output pixel of rows [row0, row1); thread blocks [f * tiles, (f + 1) * tiles) serve frame f
__global__ void __launch_bounds__(256)
    jdec_colour_kernel(const DecFrame* __restrict__ frames, unsigned int tiles,
                       const unsigned char* __restrict__ planes, const unsigned int* __restrict__ bad) {
  const unsigned int f = blockIdx.x / tiles, tile = blockIdx.x % tiles;
  const DecFrame& F = frames[f];
  if (bad[f]) return;
  const unsigned long long idx = static_cast<unsigned long long>(tile) * blockDim.x + threadIdx.x;
  const unsigned long long rows = static_cast<unsigned long long>(F.row1 - F.row0);
  if (idx >= rows * F.width) return;
  const int x = static_cast<int>(idx % F.width), y = F.row0 + static_cast<int>(idx / F.width);
  unsigned char* o = F.out + static_cast<unsigned long long>(y - F.row0) * F.row_step;
  const int Y = planes[F.plane_off[0] + static_cast<unsigned long long>(y) * F.plane_w[0] + x];
  if (F.channels == 1) {
    o[x] = static_cast<unsigned char>(Y);
    return;
  }
  if (F.ncomp == 1) {
    o[3 * x] = o[3 * x + 1] = o[3 * x + 2] = static_cast<unsigned char>(Y);
    return;
  }
  const int cw = (F.width + F.hmax - 1) / F.hmax, ch = (F.height + F.vmax - 1) / F.vmax;
  const int cb = upsample(planes + F.plane_off[1], F.plane_w[1], cw, ch, F.hmax, F.vmax, x, y) - 128;
  const int cr = upsample(planes + F.plane_off[2], F.plane_w[2], cw, ch, F.hmax, F.vmax, x, y) - 128;
  // jdcolor.c build_ycc_rgb_table, SCALEBITS 16
  const int r = Y + ((91881 * cr + 32768) >> 16);
  const int g = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int b = Y + ((116130 * cb + 32768) >> 16);
  o[3 * x] = clamp255(b);
  o[3 * x + 1] = clamp255(g);
  o[3 * x + 2] = clamp255(r);
}

// ---- host side ------------------------------------------------------------------------------------------------------
void build_table(const JpegHuffTable& t, DecTable* d) {
  std::memset(d, 0, sizeof(*d));
  int32_t code = 0;
  int p = 0;
  for (int l = 1; l <= 16; ++l) {
    d->valoff[l] = p - code;
    d->maxcode[l] = -1;
    for (int i = 0; i < t.bits[l - 1]; ++i, ++p, ++code) {
      if (l <= 8)
        for (int e = 0; e < (1 << (8 - l)); ++e)
          d->look[(code << (8 - l)) | e] = static_cast<uint16_t>((l << 8) | t.vals[p]);
      d->maxcode[l] = code;
    }
    code <<= 1;
  }
  std::memcpy(d->vals, t.vals, sizeof(d->vals));
}

// One frame of a decode: the file, its parsed header, and where its rows go
struct DecodeJob {
  const unsigned char* file;
  size_t bytes;
  JpegFrame hdr;
  unsigned char* out;    // device: row `row0` of the output
  size_t row_step;
  int channels;
  int32_t row0, row1;    // output rows
  int status;
};

unsigned long long n_mcu_of(const JpegFrame& h, int* mcus_x, int* mcus_y) {
  *mcus_x = (h.width + 8 * h.hmax - 1) / (8 * h.hmax);
  *mcus_y = (h.height + 8 * h.vmax - 1) / (8 * h.vmax);
  return static_cast<unsigned long long>(*mcus_x) * static_cast<unsigned long long>(*mcus_y);
}

int bpm_of(const JpegFrame& h) { return h.components == 1 ? 1 : h.hmax * h.vmax + 2; }

size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// device scratch of one frame (see the file's head)
size_t frame_scratch(const JpegFrame& h, size_t bytes) {
  int mx, my;
  const unsigned long long n_mcu = n_mcu_of(h, &mx, &my), blocks = n_mcu * bpm_of(h);
  const unsigned long long n_seg = h.restart_interval ? (n_mcu + h.restart_interval - 1) / h.restart_interval : 1;
  const unsigned long long subs = bytes * 8 / kSubBits + n_seg + 1;
  return 2 * align256(bytes) + blocks * 192 + subs * (sizeof(SubInfo) + 8 + 40) + (n_seg + 1) * 4 + sizeof(DecFrame) +
         4096;
}

template <typename T>
T* carve(unsigned char*& p, size_t count) {
  T* r = reinterpret_cast<T*>(p);
  p += align256(count * sizeof(T));
  return r;
}

// Decodes jobs[0, n) (headers parsed, status AMB_OK) as one group; sets each job's status
int decode_group(amb_ctx* ctx, DecodeJob* jobs, size_t n) {
  cudaStream_t st = ctx->stream;
  std::vector<DecFrame> frames(n);
  std::vector<ChunkInfo> chunks;
  std::vector<uint32_t> first_chunk(n + 1);
  std::vector<unsigned long long> scan_end(n);
  size_t file_bytes = 0, ub_bytes = 0, plane_bytes = 0;
  unsigned long long coef_blocks = 0;
  uint32_t n_segs = 0;
  for (size_t f = 0; f < n; ++f) {
    const JpegFrame& h = jobs[f].hdr;
    DecFrame& F = frames[f];
    std::memset(&F, 0, sizeof(F));
    for (int c = 0; c < h.components; ++c) {
      build_table(h.dc[h.comp_td[c]], &F.dc[c]);
      build_table(h.ac[h.comp_ta[c]], &F.ac[c]);
      std::memcpy(F.quant[c], h.quant[h.comp_tq[c]], sizeof(F.quant[c]));
    }
    F.width = h.width;
    F.height = h.height;
    F.ncomp = h.components;
    F.hmax = h.hmax;
    F.vmax = h.vmax;
    F.bpm = bpm_of(h);
    F.n_mcu = n_mcu_of(h, &F.mcus_x, &F.mcus_y);
    for (int j = 0; j < F.bpm; ++j) {
      const bool luma = j < h.hmax * h.vmax;
      F.blk_comp[j] = luma ? 0 : j - h.hmax * h.vmax + 1;
      F.blk_dx[j] = luma ? j % h.hmax : 0;
      F.blk_dy[j] = luma ? j / h.hmax : 0;
    }
    F.ri = h.restart_interval ? h.restart_interval : static_cast<int32_t>(F.n_mcu);
    F.n_seg = static_cast<int32_t>((F.n_mcu + F.ri - 1) / F.ri);
    F.seg_base = n_segs;
    n_segs += static_cast<uint32_t>(F.n_seg) + 1;
    F.channels = jobs[f].channels;
    F.row0 = jobs[f].row0;
    F.row1 = jobs[f].row1;
    // MCU rows of the output rows, with one more above and below for the vertical upsampling's context
    const int mh = 8 * h.vmax;
    F.mcu_row0 = std::max(F.row0 / mh - 1, 0);
    F.mcu_row1 = std::min((F.row1 + mh - 1) / mh + 1, F.mcus_y);
    F.file_off = file_bytes;
    F.scan_begin = file_bytes + h.scan_begin;
    F.scan_end = file_bytes + jobs[f].bytes;
    scan_end[f] = F.scan_end;
    F.ub_off = ub_bytes;
    F.coef_off = coef_blocks;
    F.plane_w[0] = F.mcus_x * h.hmax * 8;
    F.plane_w[1] = F.plane_w[2] = F.mcus_x * 8;
    F.plane_off[0] = plane_bytes;
    plane_bytes += align256(static_cast<size_t>(F.plane_w[0]) * F.mcus_y * h.vmax * 8);
    for (int c = 1; c < h.components; ++c) {
      F.plane_off[c] = plane_bytes;
      plane_bytes += align256(static_cast<size_t>(F.plane_w[c]) * F.mcus_y * 8);
    }
    F.out = jobs[f].out;
    F.row_step = jobs[f].row_step;
    first_chunk[f] = static_cast<uint32_t>(chunks.size());
    for (unsigned long long b = F.scan_begin; b < F.scan_end; b += kChunk)
      chunks.push_back(ChunkInfo{b, std::min<unsigned long long>(b + kChunk, F.scan_end), static_cast<uint32_t>(f), 0});
    file_bytes += align256(jobs[f].bytes);
    ub_bytes += align256(jobs[f].bytes - h.scan_begin + 8);
    coef_blocks += F.n_mcu * F.bpm;
  }
  first_chunk[n] = static_cast<uint32_t>(chunks.size());
  const size_t n_chunks = chunks.size();

  // files up (pinned or pageable: the library's staging path)
  AMB_CUDA(ctx, ctx->jdec_files.reserve(file_bytes + 256));
  for (size_t f = 0; f < n; ++f) {
    const int rc =
        staged_h2d(ctx, ctx->jdec_files.as<unsigned char>() + frames[f].file_off, jobs[f].file, jobs[f].bytes, st);
    if (rc != AMB_OK) return rc;
  }
  AMB_CUDA(ctx, ctx->jdec_stream.reserve(ub_bytes + 256));
  const size_t meta_bytes = align256(n * sizeof(DecFrame)) + align256(n_chunks * sizeof(ChunkInfo)) +
                            align256((n + 1) * 4) + align256(n * 8) + align256((n_chunks + 1) * 8) +
                            align256(((n_chunks + kScanTile - 1) / kScanTile + 1) * 8) + align256(n_segs * 4) +
                            align256(n * 4) + align256(kSyncLaunchesPerRead * 4);
  AMB_CUDA(ctx, ctx->jdec_meta.reserve(meta_bytes));
  unsigned char* mp = ctx->jdec_meta.as<unsigned char>();
  DecFrame* d_frames = carve<DecFrame>(mp, n);
  ChunkInfo* d_chunks = carve<ChunkInfo>(mp, n_chunks);
  uint32_t* d_first = carve<uint32_t>(mp, n + 1);
  unsigned long long* d_scan_end = carve<unsigned long long>(mp, n);
  unsigned long long* d_offsets = carve<unsigned long long>(mp, n_chunks + 1);
  unsigned long long* d_spine = carve<unsigned long long>(mp, (n_chunks + kScanTile - 1) / kScanTile + 1);
  uint32_t* d_seg = carve<uint32_t>(mp, n_segs);
  unsigned int* d_bad = carve<unsigned int>(mp, n);
  unsigned int* d_counters = carve<unsigned int>(mp, kSyncLaunchesPerRead);
  AMB_CUDA(ctx, cudaMemcpyAsync(d_frames, frames.data(), n * sizeof(DecFrame), cudaMemcpyHostToDevice, st));
  if (n_chunks)
    AMB_CUDA(ctx, cudaMemcpyAsync(d_chunks, chunks.data(), n_chunks * sizeof(ChunkInfo), cudaMemcpyHostToDevice, st));
  AMB_CUDA(ctx, cudaMemcpyAsync(d_first, first_chunk.data(), (n + 1) * 4, cudaMemcpyHostToDevice, st));
  AMB_CUDA(ctx, cudaMemcpyAsync(d_scan_end, scan_end.data(), n * 8, cudaMemcpyHostToDevice, st));
  AMB_CUDA(ctx, cudaMemsetAsync(d_seg, 0xff, n_segs * 4, st));
  AMB_CUDA(ctx, cudaMemsetAsync(d_bad, 0, n * 4, st));

  // ---- unstuff ----
  unsigned char* files = ctx->jdec_files.as<unsigned char>();
  unsigned char* ub = ctx->jdec_stream.as<unsigned char>();
  if (n_chunks) {
    const unsigned int g = static_cast<unsigned int>(n_chunks);
    jdec_scan_end_kernel<<<g, kChunkThreads, 0, st>>>(files, d_chunks, d_frames, d_scan_end);
    jdec_unstuff_count_kernel<<<g, kChunkThreads, 0, st>>>(files, d_chunks, d_frames, d_scan_end, d_offsets);
    scan_u64(d_offsets, n_chunks, d_spine, st);
    jdec_unstuff_copy_kernel<<<g, kChunkThreads, 0, st>>>(files, d_chunks, d_frames, d_scan_end, d_offsets, d_first, ub,
                                                         d_seg, d_bad);
    AMB_CUDA(ctx, cudaGetLastError());
  }
  std::vector<unsigned long long> offsets(n_chunks + 1, 0);
  std::vector<uint32_t> seg(n_segs);
  std::vector<unsigned int> bad(n);
  if (n_chunks)
    AMB_CUDA(ctx, cudaMemcpyAsync(offsets.data(), d_offsets, (n_chunks + 1) * 8, cudaMemcpyDeviceToHost, st));
  AMB_CUDA(ctx, cudaMemcpyAsync(seg.data(), d_seg, n_segs * 4, cudaMemcpyDeviceToHost, st));
  AMB_CUDA(ctx, cudaMemcpyAsync(bad.data(), d_bad, n * 4, cudaMemcpyDeviceToHost, st));
  AMB_CUDA(ctx, cudaStreamSynchronize(st));

  // ---- subsequences of every restart segment ----
  constexpr unsigned long long kMask40 = (1ull << 40) - 1;
  std::vector<SubInfo> subs;
  std::vector<unsigned long long> entry, ub_len(n, 0);
  for (size_t f = 0; f < n; ++f) {
    ub_len[f] = (offsets[first_chunk[f + 1]] - offsets[first_chunk[f]]) & kMask40;
    if (bad[f]) continue;
    const DecFrame& F = frames[f];
    seg[F.seg_base] = 0;
    for (int s = 0; s < F.n_seg && !bad[f]; ++s) {
      const unsigned long long b = seg[F.seg_base + s];
      const uint32_t last_end = seg[F.seg_base + F.n_seg];
      const unsigned long long e = s + 1 < F.n_seg ? seg[F.seg_base + s + 1]
                                                   : (last_end == kNoSegment ? ub_len[f] : last_end);
      if (b == kNoSegment || e == kNoSegment || e < b) {  // a restart marker is missing: the scan ends early
        bad[f] = 2;
        break;
      }
      const unsigned long long bits = 8 * (e - b);
      const unsigned long long ns = std::max<unsigned long long>(1, (bits + kSubBits - 1) / kSubBits);
      const uint32_t first = static_cast<uint32_t>(subs.size());
      for (unsigned long long q = 0; q < ns; ++q) {
        SubInfo si;
        si.begin = 8 * b + q * kSubBits;
        si.end = q + 1 < ns ? si.begin + kSubBits : 8 * e;
        si.frame = static_cast<uint32_t>(f);
        si.seg = static_cast<uint32_t>(s);
        si.first = first;
        si.last = q + 1 == ns ? 1u : 0u;
        subs.push_back(si);
        entry.push_back(pack_state(si.begin, 0, 0));  // exact for the first subsequence, a guess for the others
      }
    }
  }
  const unsigned long long n_sub = subs.size();
  AMB_CUDA(ctx, cudaMemcpyAsync(d_bad, bad.data(), n * 4, cudaMemcpyHostToDevice, st));
  if (n_sub) {
    const size_t sub_bytes = align256(n_sub * sizeof(SubInfo)) + align256(n_sub * 8) + align256(n * 8) +
                             4 * align256((n_sub + 1) * 8) + align256(((n_sub + kScanTile - 1) / kScanTile + 1) * 8);
    AMB_CUDA(ctx, ctx->jdec_subs.reserve(sub_bytes));
    unsigned char* sp = ctx->jdec_subs.as<unsigned char>();
    SubInfo* d_subs = carve<SubInfo>(sp, n_sub);
    unsigned long long* d_entry = carve<unsigned long long>(sp, n_sub);
    unsigned long long* d_ub_len = carve<unsigned long long>(sp, n);
    unsigned long long* d_sums = reinterpret_cast<unsigned long long*>(sp);
    sp += 4 * align256((n_sub + 1) * 8);
    unsigned long long* d_sub_spine = carve<unsigned long long>(sp, (n_sub + kScanTile - 1) / kScanTile + 1);
    AMB_CUDA(ctx, cudaMemcpyAsync(d_subs, subs.data(), n_sub * sizeof(SubInfo), cudaMemcpyHostToDevice, st));
    AMB_CUDA(ctx, cudaMemcpyAsync(d_entry, entry.data(), n_sub * 8, cudaMemcpyHostToDevice, st));
    AMB_CUDA(ctx, cudaMemcpyAsync(d_ub_len, ub_len.data(), n * 8, cudaMemcpyHostToDevice, st));
    const unsigned int g = static_cast<unsigned int>((n_sub + 127) / 128);

    // ---- synchronise the entry states ----
    for (;;) {
      AMB_CUDA(ctx, cudaMemsetAsync(d_counters, 0, kSyncLaunchesPerRead * 4, st));
      for (int t = 0; t < kSyncLaunchesPerRead; ++t)
        jdec_sync_kernel<<<g, 128, 0, st>>>(d_frames, d_subs, n_sub, ub, d_ub_len, d_entry, d_counters, t);
      AMB_CUDA(ctx, cudaGetLastError());
      unsigned int changes = 0;
      AMB_CUDA(ctx, cudaMemcpyAsync(&changes, d_counters + kSyncLaunchesPerRead - 1, 4, cudaMemcpyDeviceToHost, st));
      AMB_CUDA(ctx, cudaStreamSynchronize(st));
      if (changes == 0) break;
    }

    // ---- count, scan, write ----
    jdec_count_kernel<<<g, 128, 0, st>>>(d_frames, d_subs, n_sub, ub, d_ub_len, d_entry, d_sums);
    for (int a = 0; a < 4; ++a) scan_u64(d_sums + a * (n_sub + 1), n_sub, d_sub_spine, st);
    AMB_CUDA(ctx, ctx->jdec_coef.reserve(coef_blocks * 128 + plane_bytes + 256));
    AMB_CUDA(ctx, cudaMemsetAsync(ctx->jdec_coef.ptr, 0, coef_blocks * 128, st));
    int16_t* coef = ctx->jdec_coef.as<int16_t>();
    jdec_write_kernel<<<g, 128, 0, st>>>(d_frames, d_subs, n_sub, ub, d_ub_len, d_entry, d_sums, coef, d_bad);
    AMB_CUDA(ctx, cudaGetLastError());

    // ---- reconstruct the rows asked for ----
    unsigned char* planes = ctx->jdec_coef.as<unsigned char>() + align256(coef_blocks * 128);
    unsigned long long max_blocks = 0, max_px = 0;
    for (size_t f = 0; f < n; ++f) {
      const DecFrame& F = frames[f];
      max_blocks = std::max<unsigned long long>(
          max_blocks, static_cast<unsigned long long>(F.mcu_row1 - F.mcu_row0) * F.mcus_x * F.bpm);
      max_px = std::max<unsigned long long>(max_px, static_cast<unsigned long long>(F.row1 - F.row0) * F.width);
    }
    if (max_blocks && max_px) {
      const unsigned int bt = static_cast<unsigned int>((max_blocks + 127) / 128);
      const unsigned int pt = static_cast<unsigned int>((max_px + 255) / 256);
      jdec_idct_kernel<<<static_cast<unsigned int>(bt * n), 128, 0, st>>>(d_frames, bt, coef, planes, d_bad);
      jdec_colour_kernel<<<static_cast<unsigned int>(pt * n), 256, 0, st>>>(d_frames, pt, planes, d_bad);
      AMB_CUDA(ctx, cudaGetLastError());
    }
    AMB_CUDA(ctx, cudaMemcpyAsync(bad.data(), d_bad, n * 4, cudaMemcpyDeviceToHost, st));
  }
  AMB_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t f = 0; f < n; ++f) jobs[f].status = bad[f] ? AMB_ERR_CORRUPT_DATA : AMB_OK;
  return AMB_OK;
}

// Decodes every job whose status is AMB_OK, in groups of at most kGroupBudget bytes of scratch
int decode_jobs(amb_ctx* ctx, std::vector<DecodeJob>& jobs) {
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<DecodeJob> group;
  std::vector<size_t> index;
  size_t used = 0;
  auto flush = [&]() -> int {
    if (group.empty()) return AMB_OK;
    const int rc = decode_group(ctx, group.data(), group.size());
    if (rc != AMB_OK) return rc;
    for (size_t g = 0; g < group.size(); ++g) jobs[index[g]].status = group[g].status;
    group.clear();
    index.clear();
    used = 0;
    return AMB_OK;
  };
  for (size_t f = 0; f < jobs.size(); ++f) {
    if (jobs[f].status != AMB_OK || jobs[f].row1 <= jobs[f].row0) continue;
    const size_t need = frame_scratch(jobs[f].hdr, jobs[f].bytes);
    if (!group.empty() && (used + need > kGroupBudget || group.size() >= 65535)) {
      const int rc = flush();
      if (rc != AMB_OK) return rc;
    }
    group.push_back(jobs[f]);
    index.push_back(f);
    used += need;
  }
  return flush();
}

}  // namespace

int jpeg_decode_bands(amb_ctx* ctx, const JpegBands& in, unsigned char** band_ptr, int* band_pitch) {
  const size_t n = in.n;
  std::vector<DecodeJob> jobs(n);
  size_t total = 0;
  std::vector<size_t> off(n, 0);
  for (size_t f = 0; f < n; ++f) {
    DecodeJob& J = jobs[f];
    J.file = static_cast<const unsigned char*>(in.files[f]);
    J.bytes = in.file_bytes[f];
    J.hdr = in.headers[f];
    J.channels = in.channels;
    J.row0 = in.row0[f];
    J.row1 = in.row1[f];
    J.status = AMB_OK;
    J.row_step = align256(static_cast<size_t>(J.hdr.width) * in.channels);
    band_ptr[f] = nullptr;
    band_pitch[f] = static_cast<int>(J.row_step);
    if (J.row1 <= J.row0) continue;  // contributes nothing: never copied or decoded
    off[f] = total;
    total += J.row_step * static_cast<size_t>(J.row1 - J.row0);
  }
  AMB_CUDA(ctx, ctx->frames.reserve(total + 256));
  for (size_t f = 0; f < n; ++f) {
    if (jobs[f].row1 <= jobs[f].row0) continue;
    jobs[f].out = ctx->frames.as<unsigned char>() + off[f];
    band_ptr[f] = jobs[f].out;
  }
  const int rc = decode_jobs(ctx, jobs);
  if (rc != AMB_OK) return rc;
  for (size_t f = 0; f < n; ++f)
    if (jobs[f].status != AMB_OK) return jobs[f].status;
  return AMB_OK;
}

}  // namespace amb

using namespace amb;

extern "C" {

int amb_jpeg_info(const void* file, size_t bytes, int32_t* width, int32_t* height, int* components, int* sampling,
                  int32_t* restart_interval) {
  if (!file) return AMB_ERR_INVALID_ARGUMENT;
  JpegFrame h;
  const int rc = jpeg_parse(static_cast<const unsigned char*>(file), bytes, &h);
  if (rc != AMB_OK) return rc;
  if (width) *width = h.width;
  if (height) *height = h.height;
  if (components) *components = h.components;
  if (sampling) *sampling = h.sampling;
  if (restart_interval) *restart_interval = h.restart_interval;
  return AMB_OK;
}

int amb_jpeg_decode_device(amb_ctx* ctx, const void* const* files, const size_t* file_bytes, size_t n, int channels,
                           void* const* d_out, const size_t* row_step, int* status) {
  if (!ctx || !files || !file_bytes || !d_out || !row_step || !status || (channels != 1 && channels != 3))
    return AMB_ERR_INVALID_ARGUMENT;
  std::vector<DecodeJob> jobs(n);
  for (size_t f = 0; f < n; ++f) {
    DecodeJob& J = jobs[f];
    J.file = static_cast<const unsigned char*>(files[f]);
    J.bytes = file_bytes[f];
    J.status = jpeg_parse(J.file, J.bytes, &J.hdr);
    J.out = static_cast<unsigned char*>(d_out[f]);
    J.row_step = row_step[f];
    J.channels = channels;
    J.row0 = 0;
    J.row1 = J.hdr.height;
    if (J.status == AMB_OK && (!J.out || J.row_step < static_cast<size_t>(J.hdr.width) * channels))
      J.status = AMB_ERR_INVALID_ARGUMENT;
  }
  const int rc = decode_jobs(ctx, jobs);
  if (rc != AMB_OK) return rc;
  int first = AMB_OK;
  for (size_t f = 0; f < n; ++f) {
    status[f] = jobs[f].status;
    if (first == AMB_OK) first = jobs[f].status;
  }
  return first;
}

}  // extern "C"
