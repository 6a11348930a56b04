// deflate_encode.cu — the strips of a Deflate-compressed TIFF (Compression 8, Predictor 3 for F32, 2 for the 8-bit
// formats) of a raster in device memory (convention in include/aerial_mapper_b200.h, amb_deflate_strips_device).
//
// Every strip is an independent zlib stream.  Its predicted bytes are cut into segments of kSeg bytes, and five
// segments (65535 bytes) make one Deflate block, so a stored block never holds more than 65535 bytes.  Six steps:
//   predict  raster -> predicted strip bytes (BGR -> RGB, big-endian byte planes, differencing), one thread per byte
//   match    one CTA per segment: the segment and up to 32 KB of its strip's history in shared memory; a hash chain
//            (each position's link: the most recent earlier position with the same 3-byte hash; within the last 8
//            positions of a round the same 3 bytes) gives up to kChain candidates; every thread parses its chunk greedily from
//            the chunk's start, then one thread follows the true parse across the chunks and re-walks each chunk where
//            it enters elsewhere until it meets that chunk's parse; tokens, histograms and Adler-32 partial sums out
//   huffman  one warp per block: length-limited code lengths (15 bits, code-length code 7 bits), the header, the
//            cheapest of dynamic, fixed and stored (a coded block must not exceed its stored size, 8 * len + 40 bits)
//   layout   one thread per strip: bit position of every block, the strip's length and its Adler-32; scan -> offsets
//   pack     one CTA per segment writes its header and codes at its bit offset into zeroed 32-bit words (bit i of the
//            stream is bit i % 32 of word i / 32, i.e. little-endian bytes); words shared with a neighbour are combined
//            with atomicAdd, an OR here because the bit ranges are disjoint, so the result does not depend on the order
//   frame    zlib header (78 01) and the big-endian Adler-32 of every strip
// Everything is integer arithmetic on a fixed partition, so the bytes depend on the raster, the format and
// rows_per_strip only.
#include <algorithm>
#include <cstring>

#include "deflate_encode.h"

namespace amb {
namespace {

#include "block_scan.inc"

constexpr int kSeg = 13107;                        // bytes per segment; 5 segments = 65535 bytes = one block
constexpr int kSegsPerBlock = 5;
constexpr int kBlock = kSeg * kSegsPerBlock;
constexpr int kWindow = 32768;
constexpr int kMatchThreads = 128;
constexpr int kChunk = (kSeg + kMatchThreads - 1) / kMatchThreads;  // bytes each thread parses
constexpr int kHashBits = 13;
constexpr int kRecent = 8;                         // positions of a round searched for the same 3 bytes
constexpr int kChain = 4;                          // candidates tried per position
constexpr int kNumLit = 286, kNumDist = 30, kNumSym = kNumLit + kNumDist;
constexpr int kHeaderBytes = 576;                  // the largest dynamic header: 17 + 19 * 3 + 316 * 14 bits < 4608
// token words (uint16 per predicted byte): a token start holds 0x8000 | literal or 0x8100 + (length - 3), the byte
// after a match start its distance - 1 (< 0x8000); every other byte kNone
constexpr uint16_t kNone = 0xFFFFu, kLit = 0x8000u, kMatch = 0x8100u;

__device__ __forceinline__ unsigned long long min_u64(unsigned long long a, unsigned long long b) { return a < b ? a : b; }

__device__ __forceinline__ unsigned long long strip_len(const DeflateShape& s, int strip) {
  const int rows = min(s.rps, s.h - strip * s.rps);
  return static_cast<unsigned long long>(rows) * s.row_bytes;
}

__device__ __forceinline__ int floor_log2(uint32_t a) {  // a > 0
#ifdef AMB_CUDA_EMU
  return 31 - __builtin_clz(a);
#else
  return 31 - __clz(a);
#endif
}

// ---- predict ------------------------------------------------------------------------------------------------------------
// The byte k of a row before differencing: F32 plane k / w (most significant first) of sample k % w; 8-bit: sample k,
// the channels of a BGR pixel reversed
__device__ __forceinline__ unsigned int row_byte(const DeflateShape& s, const unsigned char* row, unsigned long long k) {
  if (s.bps == 4) {
    const unsigned long long plane = k / static_cast<unsigned long long>(s.w);
    const unsigned long long x = k - plane * s.w;
    const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(row) + x);
    return (v >> (24 - 8 * static_cast<int>(plane))) & 0xffu;
  }
  if (s.spp == 3) {
    const unsigned long long x = k / 3;
    return __ldg(row + 3 * x + (2 - static_cast<int>(k - 3 * x)));
  }
  return __ldg(row + k);
}

__global__ void __launch_bounds__(256)
    deflate_predict_kernel(const DeflateShape s, unsigned long long n, unsigned char* __restrict__ out) {
  const int step = s.bps == 4 ? 1 : s.spp;
  for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const unsigned long long r = i / s.row_bytes, k = i - r * s.row_bytes;
    const unsigned char* row = s.img + r * s.stride;
    unsigned int v = row_byte(s, row, k);
    if (s.predict && k >= static_cast<unsigned long long>(step)) v -= row_byte(s, row, k - step);
    out[i] = static_cast<unsigned char>(v);
  }
}

// ---- match ------------------------------------------------------------------------------------------------------------
struct MatchSmem {
  unsigned char* win;   // history + segment
  uint16_t* prev;       // per segment byte: distance to its candidate, 0 = none
  uint32_t* head;       // hash -> window position + 1 (chain building), then ...
  uint16_t* mark;       // ... per segment byte: the token starting there (kLit | byte, kMatch + length - 3) or kNone
  int hist_at;          // window offset of the segment
  int len;              // segment bytes
};

// The longest match (up to 258 bytes, not past the segment's end) at segment position p among its first kChain
// candidates (the chain continues through candidates inside the segment), or 0; *dist its distance (the nearest of
// equal lengths)
__device__ __forceinline__ int match_len(const MatchSmem& m, int p, int* dist) {
  const int a = m.hist_at + p, lim = min(258, m.len - p);
  int best = 0, q = a;
  for (int c = 0; c < kChain && q >= m.hist_at; ++c) {
    const int d = m.prev[q - m.hist_at];
    if (d == 0 || a - (q - d) > kWindow) break;
    q -= d;
    int l = 0;
    while (l < lim && m.win[q + l] == m.win[a + l]) ++l;
    if (l > best) {
      best = l;
      *dist = a - q;
      if (l == lim) break;
    }
  }
  return best;
}

// The token at segment position p: returns its length; *code its mark, *dist a match's distance
__device__ __forceinline__ int token_at(const MatchSmem& m, int p, uint16_t* code, int* dist) {
  const int l = match_len(m, p, dist);
  if (l >= 3) {
    *code = static_cast<uint16_t>(kMatch + l - 3);
    return l;
  }
  *code = static_cast<uint16_t>(kLit | m.win[m.hist_at + p]);
  return 1;
}

__device__ __forceinline__ bool is_start(uint16_t v) { return v >= kLit && v != kNone; }

__device__ __forceinline__ int len_code(int len, int* extra_bits, int* extra) {  // 3..258 -> 257..285
  const int v = len - 3;
  if (v < 8) {
    *extra_bits = 0;
    *extra = 0;
    return 257 + v;
  }
  if (v == 255) {
    *extra_bits = 0;
    *extra = 0;
    return 285;
  }
  const int nb = floor_log2(static_cast<uint32_t>(v));
  *extra_bits = nb - 2;
  *extra = v & ((1 << (nb - 2)) - 1);
  return 257 + 4 * (nb - 1) + ((v >> (nb - 2)) & 3);
}

__device__ __forceinline__ int dist_code(int d, int* extra_bits, int* extra) {  // 1..32768 -> 0..29
  const int v = d - 1;
  if (v < 4) {
    *extra_bits = 0;
    *extra = 0;
    return v;
  }
  const int nb = floor_log2(static_cast<uint32_t>(v));
  *extra_bits = nb - 1;
  *extra = v & ((1 << (nb - 1)) - 1);
  return 2 * nb + ((v >> (nb - 1)) & 1);
}

__device__ __forceinline__ uint32_t hash3(uint32_t key) { return (key * 2654435761u) >> (32 - kHashBits); }

// One CTA per segment g (strip g / segs, segment g % segs of it).  Out: tok (uint16 per predicted byte), the segment's
// histogram (286 literal/length + 30 distance counts) and its Adler-32 partial sums (sum of bytes, sum of index * byte)
__global__ void __launch_bounds__(kMatchThreads)
    deflate_match_kernel(const DeflateShape s, const unsigned char* __restrict__ pred, uint16_t* __restrict__ tok,
                         uint32_t* __restrict__ hist, unsigned long long* __restrict__ sums) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ uint32_t keys[kMatchThreads];
  __shared__ int exit_at[kMatchThreads];
  __shared__ uint32_t h_sm[kNumSym];
  const int g = blockIdx.x, strip = g / s.segs, k = g % s.segs;
  const unsigned long long n = strip_len(s, strip);
  const unsigned long long o = static_cast<unsigned long long>(k) * kSeg;
  const unsigned long long strip_at = static_cast<unsigned long long>(strip) * s.rps * s.row_bytes;
  const int tid = threadIdx.x;
  for (int i = tid; i < kNumSym; i += kMatchThreads) h_sm[i] = 0;
  if (o >= n) {  // a segment past the end of the last, shorter strip
    __syncthreads();
    for (int i = tid; i < kNumSym; i += kMatchThreads) hist[static_cast<unsigned long long>(g) * kNumSym + i] = 0;
    if (tid == 0) sums[2 * g] = sums[2 * g + 1] = 0;
    return;
  }
  MatchSmem m;
  m.len = static_cast<int>(min_u64(static_cast<unsigned long long>(kSeg), n - o));
  m.hist_at = static_cast<int>(min_u64(o, static_cast<unsigned long long>(kWindow)));
  const int wlen = m.hist_at + m.len;
  m.win = smem;
  m.prev = reinterpret_cast<uint16_t*>(smem + s.win_bytes);
  m.head = reinterpret_cast<uint32_t*>(smem + s.win_bytes + s.prev_bytes);
  m.mark = reinterpret_cast<uint16_t*>(m.head);
  const unsigned char* src = pred + strip_at + o - m.hist_at;
  for (int i = tid; i < wlen; i += kMatchThreads) m.win[i] = src[i];
  for (int i = tid; i < (1 << kHashBits); i += kMatchThreads) m.head[i] = 0;
  for (int i = tid; i < m.len; i += kMatchThreads) m.prev[i] = 0;
  __syncthreads();

  // chain: rounds of kMatchThreads positions; a position's candidate is the latest earlier one of its round with the
  // same 3 bytes among the last kRecent, else the latest of the earlier rounds with the same hash
  for (int base = 0; base + 2 < wlen; base += kMatchThreads) {
    const int p = base + tid;
    const bool valid = p + 2 < wlen;
    const uint32_t key = valid ? m.win[p] | (m.win[p + 1] << 8) | (m.win[p + 2] << 16) : 0xffffffffu;
    keys[tid] = key;
    __syncthreads();
    if (valid && p >= m.hist_at) {
      int q = -1;
      for (int j = tid - 1; j >= 0 && j >= tid - kRecent; --j)
        if (keys[j] == key) {
          q = base + j;
          break;
        }
      if (q < 0) q = static_cast<int>(m.head[hash3(key)]) - 1;
      if (q >= 0 && p - q <= kWindow) m.prev[p - m.hist_at] = static_cast<uint16_t>(p - q);
    }
    __syncthreads();
    if (valid) atomicMax(&m.head[hash3(key)], static_cast<uint32_t>(p + 1));
    __syncthreads();
  }
  for (int i = tid; i < m.len; i += kMatchThreads) m.mark[i] = kNone;
  __syncthreads();

  // speculative greedy parse: every thread from the start of its chunk
  const int c0 = tid * kChunk, c1 = min(c0 + kChunk, m.len);
  int pos = c0;
  while (pos < c1) {
    uint16_t code;
    int d;
    const int l = token_at(m, pos, &code, &d);
    m.mark[pos] = code;
    pos += l;
  }
  exit_at[tid] = max(pos, c0);
  __syncthreads();

  // the true parse enters chunk t at P; where that is not on the chunk's own parse, walk from P until the two meet
  if (tid == 0) {
    const int chunks = (m.len + kChunk - 1) / kChunk;
    int P = exit_at[0];
    for (int t = 1; t < chunks; ++t) {
      const int cs = t * kChunk, ce = min(cs + kChunk, m.len);
      if (P >= ce) {  // covered by a match of an earlier chunk
        for (int q = cs; q < ce; ++q) m.mark[q] = kNone;
        continue;
      }
      if (P == cs || is_start(m.mark[P])) {
        for (int q = cs; q < P; ++q) m.mark[q] = kNone;
        P = exit_at[t];
        continue;
      }
      int q = P;
      while (q < ce && !is_start(m.mark[q])) {
        uint16_t code;
        int d;
        q += token_at(m, q, &code, &d);
      }
      for (int r = cs; r < min(q, ce); ++r) m.mark[r] = kNone;
      for (int r = P; r < q;) {
        uint16_t code;
        int d;
        const int l = token_at(m, r, &code, &d);
        m.mark[r] = code;
        r += l;
      }
      P = q < ce ? exit_at[t] : q;
    }
  }
  __syncthreads();

  // tokens out, histogram, Adler-32 partial sums
  const unsigned long long tok_at = strip_at + o;
  unsigned long long s1 = 0, s2 = 0;
  for (int p = c0; p < c1; ++p) {
    const uint16_t v = m.mark[p];
    const unsigned int b = m.win[m.hist_at + p];
    s1 += b;
    s2 += static_cast<unsigned long long>(p) * b;
    if (v == kNone) {  // the byte after a match start holds the match's distance, written with the start
      if (p == 0 || m.mark[p - 1] < kMatch || m.mark[p - 1] == kNone) tok[tok_at + p] = kNone;
      continue;
    }
    tok[tok_at + p] = v;
    if (v < kMatch) {
      atomicAdd(&h_sm[v & 0xff], 1u);
    } else {
      int eb, ev, d = 0;
      match_len(m, p, &d);
      tok[tok_at + p + 1] = static_cast<uint16_t>(d - 1);
      atomicAdd(&h_sm[len_code(v - kMatch + 3, &eb, &ev)], 1u);
      atomicAdd(&h_sm[kNumLit + dist_code(d, &eb, &ev)], 1u);
    }
  }
  unsigned long long t1, t2;
  block_exclusive<kMatchThreads>(s1, &t1);
  block_exclusive<kMatchThreads>(s2, &t2);
  for (int i = tid; i < kNumSym; i += kMatchThreads) hist[static_cast<unsigned long long>(g) * kNumSym + i] = h_sm[i];
  if (tid == 0) {
    sums[2 * g] = t1;
    sums[2 * g + 1] = t2;
  }
}

// ---- huffman --------------------------------------------------------------------------------------------------------------
// Code lengths <= limit for the n counts f (at least two non-zero), written to len[] (0 for unused symbols).  One warp;
// scratch: sorted[n], w[2n], parent[2n], depth[2n] in shared memory.
__device__ void huff_lengths(const uint32_t* f, int n, int limit, uint8_t* len, int* sorted, uint32_t* w, int* parent,
                             int* depth) {
  const int lane = threadIdx.x & 31;
  int used = 0;
  for (int i = 0; i < n; ++i) used += f[i] > 0;
  for (int i = lane; i < n; i += 32) {  // ascending (count, symbol)
    len[i] = 0;
    if (f[i] == 0) continue;
    int r = 0;
    for (int j = 0; j < n; ++j) r += f[j] > 0 && (f[j] < f[i] || (f[j] == f[i] && j < i));
    sorted[r] = i;
  }
  __syncwarp();
  if (lane == 0) {
    // two queues: leaves 0..used-1 in order, internal nodes used.. as they are made (weights never decrease)
    for (int k = 0; k < used; ++k) w[k] = f[sorted[k]];
    int li = 0, ii = used, made = used;
    for (int step = 0; step < used - 1; ++step) {
      int pick[2];
      for (int c = 0; c < 2; ++c) {
        if (li < used && (ii >= made || w[li] <= w[ii]))
          pick[c] = li++;
        else
          pick[c] = ii++;
      }
      w[made] = w[pick[0]] + w[pick[1]];
      parent[pick[0]] = parent[pick[1]] = made;
      ++made;
    }
    depth[made - 1] = 0;
    for (int k = made - 2; k >= 0; --k) depth[k] = depth[parent[k]] + 1;
    int count[16] = {0};
    for (int k = 0; k < used; ++k) ++count[min(depth[k], limit)];
    // clamping made the code over-full by `excess` units of 2^-limit; every move below takes one away: a leaf at
    // depth b < limit goes one level down and a leaf from the last level becomes its sibling
    long long kraft = 0;
    for (int l = 1; l <= limit; ++l) kraft += static_cast<long long>(count[l]) << (limit - l);
    for (long long excess = kraft - (1ll << limit); excess > 0; --excess) {
      int b = limit - 1;
      while (count[b] == 0) --b;
      --count[b];
      count[b + 1] += 2;
      --count[limit];
    }
    // the longest codes to the rarest symbols
    int k = 0;
    for (int l = limit; l >= 1; --l)
      for (int c = 0; c < count[l]; ++c) len[sorted[k++]] = static_cast<uint8_t>(l);
  }
  __syncwarp();
}

// Canonical codes (RFC 1951 3.2.2), bit-reversed for LSB-first packing: (length << 16) | code
__device__ void canonical(const uint8_t* len, int n, uint32_t* out) {
  int count[16] = {0}, next[16];
  for (int i = 0; i < n; ++i) ++count[len[i]];
  count[0] = 0;
  int code = 0;
  for (int l = 1; l < 16; ++l) {
    code = (code + count[l - 1]) << 1;
    next[l] = code;
  }
  for (int i = 0; i < n; ++i) {
    const int l = len[i];
    if (!l) {
      out[i] = 0;
      continue;
    }
    const uint32_t c = static_cast<uint32_t>(next[l]++);
    uint32_t r = 0;
    for (int k = 0; k < l; ++k) r |= ((c >> k) & 1u) << (l - 1 - k);
    out[i] = (static_cast<uint32_t>(l) << 16) | r;
  }
}

struct BitWriter {  // serial, into a byte buffer in shared memory
  unsigned char* buf;
  int n = 0;
  __device__ void put(uint32_t v, int bits) {
    for (int b = 0; b < bits; ++b, ++n)
      if ((v >> b) & 1u) buf[n >> 3] |= static_cast<unsigned char>(1u << (n & 7));
  }
};

__device__ __forceinline__ int sym_extra_bits(int sym) {  // literal/length 0..285, then distance 286..315
  if (sym < 265 || sym == 285) return 0;
  if (sym < kNumLit) return (sym - 261) / 4;
  const int d = sym - kNumLit;
  return d < 4 ? 0 : d / 2 - 1;
}

__device__ __forceinline__ int fixed_len(int sym) {
  if (sym >= kNumLit) return 5;
  return sym < 144 ? 8 : sym < 256 ? 9 : sym < 280 ? 7 : 8;
}

__constant__ uint8_t kClOrderDev[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

struct HuffSmem {
  uint32_t f[kNumSym];
  uint32_t clf[19];
  uint8_t len[kNumSym];
  uint8_t cl_len[19];
  int sorted[kNumLit];
  uint32_t w[2 * kNumLit];
  int parent[2 * kNumLit];
  int depth[2 * kNumLit];
  uint16_t rle[kNumSym];      // code-length symbol | extra << 5
  uint32_t cl_code[19];
  unsigned char header[kHeaderBytes];
  int type;
};

// One warp per block b (strip b / blocks, block b % blocks of it).  Out: type (0 stored, 1 fixed, 2 dynamic), the
// block's bits when coded, each segment's bit offset in its block, the 316 codes and the dynamic header.
__global__ void __launch_bounds__(32)
    deflate_huffman_kernel(const DeflateShape s, const uint32_t* __restrict__ hist, uint32_t* __restrict__ codes,
                           unsigned char* __restrict__ headers, int* __restrict__ type,
                           unsigned long long* __restrict__ bits, unsigned long long* __restrict__ seg_bit) {
  __shared__ HuffSmem sm;
  const int b = blockIdx.x, strip = b / s.blocks, j = b % s.blocks, lane = threadIdx.x;
  const unsigned long long n = strip_len(s, strip);
  const unsigned long long at = static_cast<unsigned long long>(j) * kBlock;
  if (at >= n) return;
  const unsigned long long blen = min_u64(static_cast<unsigned long long>(kBlock), n - at);
  const bool final = at + blen == n;
  const int g0 = strip * s.segs + j * kSegsPerBlock;
  const int nseg = static_cast<int>((blen + kSeg - 1) / kSeg);
  for (int i = lane; i < kNumSym; i += 32) {
    uint32_t v = 0;
    for (int q = 0; q < nseg; ++q) v += hist[static_cast<unsigned long long>(g0 + q) * kNumSym + i];
    sm.f[i] = v;
  }
  for (int i = lane; i < kHeaderBytes; i += 32) sm.header[i] = 0;
  __syncwarp();
  if (lane == 0) {
    sm.f[256] = 1;  // end of block
    // two codes at least in each tree, so that both are complete
    int lit_used = 0, dist_used = 0;
    for (int i = 0; i < kNumLit; ++i) lit_used += sm.f[i] > 0;
    for (int i = 0; i < kNumDist; ++i) dist_used += sm.f[kNumLit + i] > 0;
    if (lit_used < 2) sm.f[sm.f[0] ? 1 : 0] = 1;
    for (int i = 0; dist_used < 2; ++i)
      if (!sm.f[kNumLit + i]) {
        sm.f[kNumLit + i] = 1;
        ++dist_used;
      }
  }
  __syncwarp();
  uint32_t* f = sm.f;
  huff_lengths(f, kNumLit, 15, sm.len, sm.sorted, sm.w, sm.parent, sm.depth);
  huff_lengths(f + kNumLit, kNumDist, 15, sm.len + kNumLit, sm.sorted, sm.w, sm.parent, sm.depth);
  __syncwarp();
  int hlit = 0, hdist = 0, n_rle = 0;
  if (lane == 0) {
    hlit = 257;
    for (int i = 257; i < kNumLit; ++i)
      if (sm.len[i]) hlit = i + 1;
    hdist = 1;
    for (int i = 0; i < kNumDist; ++i)
      if (sm.len[kNumLit + i]) hdist = i + 1;
    // run-length code of the hlit + hdist lengths (16: repeat previous 3..6, 17: zeros 3..10, 18: zeros 11..138)
    const int total = hlit + hdist;
    for (int i = 0; i < 19; ++i) sm.clf[i] = 0;
    for (int i = 0; i < total;) {
      const int v = i < hlit ? sm.len[i] : sm.len[kNumLit + i - hlit];
      int run = 1;
      while (i + run < total && (i + run < hlit ? sm.len[i + run] : sm.len[kNumLit + i + run - hlit]) == v) ++run;
      if (v == 0 && run >= 3) {
        const int r = min(run, 138);
        sm.rle[n_rle++] = static_cast<uint16_t>(r >= 11 ? 18 | ((r - 11) << 5) : 17 | ((r - 3) << 5));
        ++sm.clf[r >= 11 ? 18 : 17];
        i += r;
      } else if (v != 0 && run >= 4) {
        sm.rle[n_rle++] = static_cast<uint16_t>(v);
        ++sm.clf[v];
        const int r = min(run - 1, 6);
        sm.rle[n_rle++] = static_cast<uint16_t>(16 | ((r - 3) << 5));
        ++sm.clf[16];
        i += 1 + r;
      } else {
        sm.rle[n_rle++] = static_cast<uint16_t>(v);
        ++sm.clf[v];
        i += 1;
      }
    }
    int cl_used = 0;
    for (int i = 0; i < 19; ++i) cl_used += sm.clf[i] > 0;
    for (int i = 0; cl_used < 2; ++i)
      if (!sm.clf[i]) {
        sm.clf[i] = 1;
        ++cl_used;
      }
  }
  __syncwarp();
  huff_lengths(sm.clf, 19, 7, sm.cl_len, sm.sorted, sm.w, sm.parent, sm.depth);
  if (lane == 0) {
    int hclen = 19;
    while (hclen > 4 && sm.cl_len[kClOrderDev[hclen - 1]] == 0) --hclen;
    canonical(sm.cl_len, 19, sm.cl_code);
    BitWriter hw{sm.header};
    hw.put(final ? 5u : 4u, 3);  // BFINAL, BTYPE = 10
    hw.put(hlit - 257, 5);
    hw.put(hdist - 1, 5);
    hw.put(hclen - 4, 4);
    for (int i = 0; i < hclen; ++i) hw.put(sm.cl_len[kClOrderDev[i]], 3);
    for (int i = 0; i < n_rle; ++i) {
      const int sym = sm.rle[i] & 31, extra = sm.rle[i] >> 5;
      hw.put(sm.cl_code[sym] & 0xffffu, static_cast<int>(sm.cl_code[sym] >> 16));
      if (sym == 16) hw.put(extra, 2);
      if (sym == 17) hw.put(extra, 3);
      if (sym == 18) hw.put(extra, 7);
    }
    // the cost of each choice; the histograms of the tokens themselves (no padding counts)
    unsigned long long dyn = hw.n, fix = 3;
    unsigned long long seg_dyn[kSegsPerBlock], seg_fix[kSegsPerBlock];
    for (int q = 0; q < nseg; ++q) {
      seg_dyn[q] = seg_fix[q] = 0;
      const uint32_t* hq = hist + static_cast<unsigned long long>(g0 + q) * kNumSym;
      for (int i = 0; i < kNumSym; ++i) {
        const unsigned long long c = hq[i];
        if (!c) continue;
        seg_dyn[q] += c * (sm.len[i] + sym_extra_bits(i));
        seg_fix[q] += c * (fixed_len(i) + sym_extra_bits(i));
      }
    }
    unsigned long long dyn_total = dyn + sm.len[256], fix_total = fix + 7;
    for (int q = 0; q < nseg; ++q) {
      dyn_total += seg_dyn[q];
      fix_total += seg_fix[q];
    }
    const unsigned long long stored = 8 * blen + 40;
    const int t = (dyn_total <= fix_total ? dyn_total : fix_total) > stored ? 0 : dyn_total <= fix_total ? 2 : 1;
    type[b] = t;
    sm.type = t;
    bits[b] = t == 2 ? dyn_total : t == 1 ? fix_total : 0;
    unsigned long long off = t == 2 ? dyn : 3;
    for (int q = 0; q < nseg; ++q) {
      seg_bit[g0 + q] = off;
      off += t == 2 ? seg_dyn[q] : seg_fix[q];
    }
  }
  __syncwarp();
  if (lane == 0) {
    canonical(sm.len, kNumLit, codes + static_cast<unsigned long long>(b) * kNumSym);
    canonical(sm.len + kNumLit, kNumDist, codes + static_cast<unsigned long long>(b) * kNumSym + kNumLit);
    if (sm.type == 1) {  // RFC 1951 3.2.6: the canonical code of 288 literal/length and 32 distance symbols
      uint32_t* c = codes + static_cast<unsigned long long>(b) * kNumSym;
      for (int i = 0; i < kNumSym; ++i) {
        const uint32_t v = i >= kNumLit ? i - kNumLit : i < 144 ? 0x30 + i : i < 256 ? 0x190 + i - 144
                                                      : i < 280 ? i - 256 : 0xc0 + i - 280;
        const int l = fixed_len(i);
        uint32_t r = 0;
        for (int k = 0; k < l; ++k) r |= ((v >> k) & 1u) << (l - 1 - k);
        c[i] = (static_cast<uint32_t>(l) << 16) | r;
      }
    }
  }
  for (int i = lane; i < kHeaderBytes; i += 32) headers[static_cast<unsigned long long>(b) * kHeaderBytes + i] = sm.header[i];
}

// ---- layout ---------------------------------------------------------------------------------------------------------------
// One thread per strip: the bit position of each block in the strip's Deflate data, the strip's byte length (zlib
// header, data, Adler-32) and its Adler-32
__global__ void __launch_bounds__(128)
    deflate_layout_kernel(const DeflateShape s, const int* __restrict__ type, const unsigned long long* __restrict__ bits,
                          const unsigned long long* __restrict__ sums, unsigned long long* __restrict__ blk_pos,
                          unsigned long long* __restrict__ strip_bytes, uint32_t* __restrict__ adler) {
  const int strip = blockIdx.x * blockDim.x + threadIdx.x;
  if (strip >= s.n_strips) return;
  const unsigned long long n = strip_len(s, strip);
  const int nb = static_cast<int>((n + kBlock - 1) / kBlock);
  unsigned long long P = 0;
  for (int j = 0; j < nb; ++j) {
    const int b = strip * s.blocks + j;
    blk_pos[b] = P;
    if (type[b] == 0) {
      const unsigned long long blen = min_u64(static_cast<unsigned long long>(kBlock), n - static_cast<unsigned long long>(j) * kBlock);
      P = ((P + 3 + 7) & ~7ull) + 32 + 8 * blen;
    } else {
      P += bits[b];
    }
  }
  strip_bytes[strip] = 2 + (P + 7) / 8 + 4;
  const int ns = static_cast<int>((n + kSeg - 1) / kSeg);
  unsigned long long a = 1, bb = n % kAdlerMod;
  for (int q = 0; q < ns; ++q) {
    const int g = strip * s.segs + q;
    adler_add_segment(n, static_cast<unsigned long long>(q) * kSeg, sums[2 * g], sums[2 * g + 1], &a, &bb);
  }
  adler[strip] = static_cast<uint32_t>((bb << 16) | a);
}

// ---- pack -----------------------------------------------------------------------------------------------------------------
// LSB-first bit writer over 32-bit words; the first and the last word may be shared with a neighbour
struct BitSink {
  uint32_t* words;
  unsigned long long w;
  unsigned long long acc;
  int n;  // bits in acc (the low n of them; the first ones belong to earlier writers and are 0)
  bool shared;
  __device__ __forceinline__ BitSink(uint32_t* out, unsigned long long pos)
      : words(out), w(pos >> 5), acc(0), n(static_cast<int>(pos & 31)), shared(n != 0) {}
  __device__ __forceinline__ void put(uint32_t v, int len) {  // len 0..32
    acc |= static_cast<unsigned long long>(v & (len == 32 ? 0xffffffffu : (1u << len) - 1u)) << n;
    n += len;
    if (n >= 32) {
      const uint32_t x = static_cast<uint32_t>(acc);
      if (shared)
        atomicAdd(words + w, x);  // disjoint bits: the sum is the OR
      else
        words[w] = x;
      shared = false;
      ++w;
      acc >>= 32;
      n -= 32;
    }
  }
  __device__ __forceinline__ void finish() {
    if (n > 0) atomicAdd(words + w, static_cast<uint32_t>(acc));
  }
};

// One CTA per segment.  Every thread codes the tokens that start in its chunk at the bit offset the block scan gives it.
__global__ void __launch_bounds__(kMatchThreads)
    deflate_pack_kernel(const DeflateShape s, const unsigned char* __restrict__ pred, const uint16_t* __restrict__ tok,
                        const uint32_t* __restrict__ codes, const unsigned char* __restrict__ headers,
                        const int* __restrict__ type, const unsigned long long* __restrict__ bits,
                        const unsigned long long* __restrict__ seg_bit, const unsigned long long* __restrict__ blk_pos,
                        const unsigned long long* __restrict__ strip_off, uint32_t* __restrict__ words) {
  __shared__ uint32_t code_sm[kNumSym];
  const int g = blockIdx.x, strip = g / s.segs, k = g % s.segs, tid = threadIdx.x;
  const unsigned long long n = strip_len(s, strip);
  const unsigned long long o = static_cast<unsigned long long>(k) * kSeg;
  if (o >= n) return;
  const int j = k / kSegsPerBlock, kb = k % kSegsPerBlock;
  const int b = strip * s.blocks + j;
  const int t = type[b];
  const unsigned long long blen = min_u64(static_cast<unsigned long long>(kBlock), n - static_cast<unsigned long long>(j) * kBlock);
  const bool final = static_cast<unsigned long long>(j) * kBlock + blen == n;
  const int len = static_cast<int>(min_u64(static_cast<unsigned long long>(kSeg), n - o));
  const unsigned long long strip_at = static_cast<unsigned long long>(strip) * s.rps * s.row_bytes;
  const unsigned long long block_bit = 8 * (strip_off[strip] + 2) + blk_pos[b];
  const int c0 = min(tid * kChunk, len), c1 = min(c0 + kChunk, len);
  const unsigned char* data = pred + strip_at + o;
  if (t == 0) {  // stored: BFINAL, 00, pad to a byte, LEN, NLEN, the bytes
    const unsigned long long data_bit = ((block_bit + 3 + 7) & ~7ull) + 32;
    if (kb == 0 && tid == 0) {
      BitSink h(words, block_bit);
      h.put(final ? 1u : 0u, 3);
      h.finish();
      BitSink l(words, data_bit - 32);
      l.put(static_cast<uint32_t>(blen) | (static_cast<uint32_t>(~blen & 0xffffu) << 16), 32);
      l.finish();
    }
    if (c0 < c1) {
      BitSink o2(words, data_bit + 8ull * (static_cast<unsigned long long>(kb) * kSeg + c0));
      for (int p = c0; p < c1; ++p) o2.put(data[p], 8);
      o2.finish();
    }
    return;
  }
  const uint32_t* cb = codes + static_cast<unsigned long long>(b) * kNumSym;
  for (int i = tid; i < kNumSym; i += kMatchThreads) code_sm[i] = cb[i];
  __syncthreads();
  const uint16_t* tk = tok + strip_at + o;
  unsigned long long mine = 0;
  for (int p = c0; p < c1; ++p) {
    const uint16_t v = tk[p];
    if (!is_start(v)) continue;
    if (v < kMatch) {
      mine += code_sm[v & 0xff] >> 16;
    } else {
      int eb, ev, db, dv;
      const int lc = len_code(v - kMatch + 3, &eb, &ev);
      const int dc = dist_code(tk[p + 1] + 1, &db, &dv);
      mine += (code_sm[lc] >> 16) + eb + (code_sm[kNumLit + dc] >> 16) + db;
    }
  }
  unsigned long long total;
  const unsigned long long before = block_exclusive<kMatchThreads>(mine, &total);
  if (mine) {
    BitSink out(words, block_bit + seg_bit[g] + before);
    for (int p = c0; p < c1; ++p) {
      const uint16_t v = tk[p];
      if (!is_start(v)) continue;
      if (v < kMatch) {
        const uint32_t c = code_sm[v & 0xff];
        out.put(c & 0xffffu, static_cast<int>(c >> 16));
      } else {
        int eb, ev, db, dv;
        const uint32_t lc = code_sm[len_code(v - kMatch + 3, &eb, &ev)];
        const uint32_t dc = code_sm[kNumLit + dist_code(tk[p + 1] + 1, &db, &dv)];
        out.put(lc & 0xffffu, static_cast<int>(lc >> 16));
        out.put(static_cast<uint32_t>(ev), eb);
        out.put(dc & 0xffffu, static_cast<int>(dc >> 16));
        out.put(static_cast<uint32_t>(dv), db);
      }
    }
    out.finish();
  }
  if (tid == 0 && kb == 0) {  // the block's header
    BitSink h(words, block_bit);
    if (t == 1) {
      h.put(final ? 3u : 2u, 3);  // BFINAL, BTYPE = 01
    } else {
      const unsigned char* hb = headers + static_cast<unsigned long long>(b) * kHeaderBytes;
      const unsigned long long hbits = seg_bit[g];
      for (unsigned long long i = 0; i < hbits; i += 8)
        h.put(hb[i >> 3], static_cast<int>(min_u64(8ull, hbits - i)));
    }
    h.finish();
  }
  if (tid == 0 && static_cast<unsigned long long>(k + 1) * kSeg >= static_cast<unsigned long long>(j) * kBlock + blen) {
    BitSink e(words, block_bit + bits[b] - (code_sm[256] >> 16));  // end of block
    e.put(code_sm[256] & 0xffffu, static_cast<int>(code_sm[256] >> 16));
    e.finish();
  }
}

// ---- frame ----------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void put_byte(uint32_t* words, unsigned long long i, unsigned int v) {
  atomicAdd(words + (i >> 2), v << (8 * static_cast<int>(i & 3)));
}

__global__ void __launch_bounds__(128)
    deflate_frame_kernel(const DeflateShape s, const unsigned long long* __restrict__ strip_off,
                         const uint32_t* __restrict__ adler, uint32_t* __restrict__ words,
                         uint32_t* __restrict__ strip_bytes) {
  const int strip = blockIdx.x * blockDim.x + threadIdx.x;
  if (strip >= s.n_strips) return;
  const unsigned long long at = strip_off[strip], end = strip_off[strip + 1];
  put_byte(words, at, 0x78);  // CM 8, CINFO 7 (32 KB window); FLEVEL 0, FCHECK: 0x7801 % 31 == 0
  put_byte(words, at + 1, 0x01);
  for (int q = 0; q < 4; ++q) put_byte(words, end - 4 + q, (adler[strip] >> (24 - 8 * q)) & 0xffu);
  strip_bytes[strip] = static_cast<uint32_t>(end - at);
}

// ---- host side ------------------------------------------------------------------------------------------------------------
unsigned long long strip_bound(unsigned long long n) { return n + 5 * ((n + kBlock - 1) / kBlock) + 6; }

size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

}  // namespace

int deflate_params(int32_t w, int32_t h, int format, int32_t rps, DeflateParams* p, bool predictor) {
  if (w <= 0 || h <= 0 || rps <= 0 || (!predictor && format == AMB_RASTER_F32)) return AMB_ERR_INVALID_ARGUMENT;
  DeflateShape& s = p->s;
  switch (format) {
    case AMB_RASTER_F32: s.spp = 1; s.bps = 4; break;
    case AMB_RASTER_GRAY8:
    case AMB_RASTER_MASK8: s.spp = 1; s.bps = 1; break;
    case AMB_RASTER_BGR8: s.spp = 3; s.bps = 1; break;
    default: return AMB_ERR_INVALID_ARGUMENT;
  }
  s.predict = predictor ? 1 : 0;
  s.img = nullptr;
  s.stride = 0;
  s.w = w;
  s.h = h;
  s.row_bytes = static_cast<unsigned long long>(w) * s.spp * s.bps;
  s.rps = std::min(rps, h);
  s.n_strips = (h + s.rps - 1) / s.rps;
  const unsigned long long full = s.row_bytes * s.rps;
  if (strip_bound(full) > 0xffffffffull || (full + kSeg - 1) / kSeg * s.n_strips > 0x7fffffffull)
    return AMB_ERR_UNSUPPORTED;
  s.segs = static_cast<int32_t>((full + kSeg - 1) / kSeg);
  s.blocks = static_cast<int32_t>((full + kBlock - 1) / kBlock);
  const int seg_max = static_cast<int>(std::min<unsigned long long>(kSeg, full));
  const int hist_max = static_cast<int>(std::min<unsigned long long>(kWindow, static_cast<unsigned long long>(s.segs - 1) * kSeg));
  s.win_bytes = (hist_max + seg_max + 15) & ~15;
  s.prev_bytes = (2 * seg_max + 15) & ~15;
  p->n_bytes = s.row_bytes * h;
  const unsigned long long last = s.row_bytes * (h - static_cast<unsigned long long>(s.n_strips - 1) * s.rps);
  p->bound = strip_bound(full) * (s.n_strips - 1) + strip_bound(last);
  return AMB_OK;
}

int deflate_encode(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, DeflateParams p, void* host_out,
                   size_t capacity, size_t* size, uint32_t* strip_bytes) {
  DeflateShape& s = p.s;
  s.img = d_img;
  s.stride = row_stride;
  cudaStream_t st = ctx->stream;
  const unsigned long long G = static_cast<unsigned long long>(s.n_strips) * s.segs;
  const unsigned long long B = static_cast<unsigned long long>(s.n_strips) * s.blocks;
  const unsigned long long S = s.n_strips;
  // scratch: predicted bytes, tokens, per segment histogram / sums / bit offset, per block codes / header / type / bits /
  // position, per strip lengths -> offsets / Adler-32 / uint32 lengths, the scan spine
  const size_t sz[] = {align256(p.n_bytes), align256(2 * p.n_bytes), align256(G * kNumSym * 4), align256(G * 16),
                       align256(G * 8), align256(B * kNumSym * 4), align256(B * kHeaderBytes), align256(B * 4),
                       align256(B * 8), align256(B * 8), align256((S + 1) * 8), align256(S * 4), align256(S * 4),
                       align256(((S + kScanTile - 1) / kScanTile + 1) * 8)};
  size_t total_scratch = 0;
  for (size_t v : sz) total_scratch += v;
  AMB_CUDA(ctx, ctx->deflate_scratch.reserve(total_scratch));
  unsigned char* at = ctx->deflate_scratch.as<unsigned char>();
  void* part[sizeof(sz) / sizeof(sz[0])];
  for (size_t i = 0; i < sizeof(sz) / sizeof(sz[0]); ++i) {
    part[i] = at;
    at += sz[i];
  }
  unsigned char* pred = static_cast<unsigned char*>(part[0]);
  uint16_t* tok = static_cast<uint16_t*>(part[1]);
  uint32_t* hist = static_cast<uint32_t*>(part[2]);
  unsigned long long* sums = static_cast<unsigned long long*>(part[3]);
  unsigned long long* seg_bit = static_cast<unsigned long long*>(part[4]);
  uint32_t* codes = static_cast<uint32_t*>(part[5]);
  unsigned char* headers = static_cast<unsigned char*>(part[6]);
  int* type = static_cast<int*>(part[7]);
  unsigned long long* bits = static_cast<unsigned long long*>(part[8]);
  unsigned long long* blk_pos = static_cast<unsigned long long*>(part[9]);
  unsigned long long* strip_off = static_cast<unsigned long long*>(part[10]);
  uint32_t* adler = static_cast<uint32_t*>(part[11]);
  uint32_t* lens32 = static_cast<uint32_t*>(part[12]);
  unsigned long long* spine = static_cast<unsigned long long*>(part[13]);

  const unsigned long long pred_blocks = std::min((p.n_bytes + 255) / 256, 1ull << 20);
  deflate_predict_kernel<<<static_cast<unsigned int>(pred_blocks), 256, 0, st>>>(s, p.n_bytes, pred);
  const size_t smem = static_cast<size_t>(s.win_bytes) + s.prev_bytes + (4 << kHashBits);  // the marks reuse the hash heads
  AMB_CUDA(ctx, cudaFuncSetAttribute(deflate_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     static_cast<int>(smem)));
  deflate_match_kernel<<<static_cast<unsigned int>(G), kMatchThreads, smem, st>>>(s, pred, tok, hist, sums);
  deflate_huffman_kernel<<<static_cast<unsigned int>(B), 32, 0, st>>>(s, hist, codes, headers, type, bits, seg_bit);
  deflate_layout_kernel<<<static_cast<unsigned int>((S + 127) / 128), 128, 0, st>>>(s, type, bits, sums, blk_pos,
                                                                                     strip_off, adler);
  scan_u64(strip_off, S, spine, st);
  AMB_CUDA(ctx, cudaGetLastError());
  unsigned long long n_out = 0;
  int rc = read_u64(ctx, strip_off + S, &n_out);
  if (rc != AMB_OK) return rc;
  *size = static_cast<size_t>(n_out);
  if (capacity < n_out) return AMB_ERR_SIZE_MISMATCH;

  const size_t word_bytes = static_cast<size_t>((n_out + 7) & ~3ull);
  AMB_CUDA(ctx, ctx->deflate_words.reserve(word_bytes));
  uint32_t* words = ctx->deflate_words.as<uint32_t>();
  AMB_CUDA(ctx, cudaMemsetAsync(words, 0, word_bytes, st));
  deflate_pack_kernel<<<static_cast<unsigned int>(G), kMatchThreads, 0, st>>>(s, pred, tok, codes, headers, type, bits,
                                                                             seg_bit, blk_pos, strip_off, words);
  deflate_frame_kernel<<<static_cast<unsigned int>((S + 127) / 128), 128, 0, st>>>(s, strip_off, adler, words, lens32);
  AMB_CUDA(ctx, cudaGetLastError());
  rc = staged_d2h(ctx, host_out, words, static_cast<size_t>(n_out), st);
  if (rc != AMB_OK) return rc;
  return staged_d2h(ctx, strip_bytes, lens32, static_cast<size_t>(S) * 4, st);
}

}  // namespace amb

using namespace amb;

extern "C" {

size_t amb_deflate_max_size(int32_t width, int32_t height, int format, int32_t rows_per_strip) {
  DeflateParams p;
  if (deflate_params(width, height, format, rows_per_strip, &p) != AMB_OK) return 0;
  return static_cast<size_t>(p.bound);
}

int amb_deflate_strips_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                              int format, int32_t rows_per_strip, void* host_out, size_t capacity, size_t* size,
                              uint32_t* strip_bytes) {
  if (!ctx || !d_image || !host_out || !size || !strip_bytes) return AMB_ERR_INVALID_ARGUMENT;
  DeflateParams p;
  const int st = deflate_params(width, height, format, rows_per_strip, &p);
  if (st != AMB_OK) return st;
  const size_t row = static_cast<size_t>(p.s.row_bytes);
  if (row_stride < row) return AMB_ERR_INVALID_ARGUMENT;
  if (p.s.bps == 4 && ((reinterpret_cast<uintptr_t>(d_image) & 3) || (row_stride & 3))) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return deflate_encode(ctx, static_cast<const unsigned char*>(d_image), row_stride, p, host_out, capacity, size,
                        strip_bytes);
}

int amb_export_deflate_strips(amb_ctx* ctx, int layer, int format, int32_t rows_per_strip, void* host_out,
                              size_t capacity, size_t* size, uint32_t* strip_bytes) {
  if (!ctx || !host_out || !size || !strip_bytes || layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  DeflateParams p;
  const int st = deflate_params(ctx->geom.rows, ctx->col_end - ctx->col_begin, format, rows_per_strip, &p);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t stride = static_cast<size_t>(p.s.row_bytes);
  AMB_CUDA(ctx, ctx->raster_band.reserve(static_cast<size_t>(p.n_bytes)));
  const int rc = amb_export_raster_device(ctx, layer, format, ctx->raster_band.ptr);
  if (rc != AMB_OK) return rc;
  return deflate_encode(ctx, ctx->raster_band.as<unsigned char>(), stride, p, host_out, capacity, size, strip_bytes);
}

}  // extern "C"
