// deflate_decode.cu — the chunks of a Deflate-compressed (or uncompressed) TIFF band inflated, unpredicted and converted
// to float32 on the device (convention in include/aerial_mapper_b200.h, amb_tiff_decode_device; the TIFF is parsed by
// the caller).  Only the chunks that intersect the window asked for are copied and decoded, in groups whose scratch
// stays under kGroupBudget:
//   inflate    one warp per zlib stream.  Every lane runs the same bit reader over the stream (the loads are
//              broadcasts), so every lane knows every symbol without a shuffle; the lanes share the work that has width:
//              building each block's canonical decode tables in shared memory (ballot ranks for the symbol sort, one
//              lane per table entry run), the stored-block and match copies (an overlapping match of distance d < 32
//              in ceil(len / d) rounds of d bytes) and the Adler-32, summed per lane and combined with the segment
//              formula of deflate_encode.h.  Output past the chunk's expected bytes goes to a 32 KB ring per stream,
//              so back-references and the Adler-32 still see it.  Every read of the stream is checked against the
//              stream's length, every write against its region, every distance against the bytes already out.
//   unpredict  one CTA per chunk row that meets the window: the predictor's prefix sum modulo the sample (predictor
//              2) or the byte (predictor 3, over the row's byte planes, then the planes gathered back into samples)
//              with block_scan.inc's block scan, the band selected, converted to float32 and stored at (r - r0, c - c0);
//              uncompressed chunks take this kernel straight from the file's bytes (predictor 3 sums them into
//              scratch of their own: chunks may share bytes of the file).
#include <algorithm>
#include <cstring>
#include <vector>

#include "deflate_encode.h"

namespace amb {
namespace {

#include "block_scan.inc"

constexpr int kInflateWarps = 4;                    // streams per CTA
constexpr int kUnpredictThreads = 256;
constexpr unsigned long long kRing = 32768;         // bytes of the window kept past a stream's expected bytes
constexpr size_t kGroupBudget = size_t(1) << 30;
constexpr unsigned kFull = 0xffffffffu;

__constant__ uint16_t kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                      31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t kDistBase[30] = {1,   2,   3,   4,   5,   7,    9,    13,   17,   25,   33,   49,    65,    97,    129,
                                       193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
__constant__ uint8_t kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// A canonical Huffman code: count[l] codes of length l, the symbols in code order, and a table of the next LB bits
// (read LSB first) -> (symbol << 4) | length for codes of at most LB bits; 0: a longer code, or none
template <int LB, int NSYM>
struct Huff {
  uint32_t count[16];
  uint16_t sym[NSYM];
  uint16_t lut[1 << LB];
};

struct InflateSmem {
  Huff<10, 288> lit;
  Huff<8, 32> dist;    // also the code-length code of a dynamic block header
  uint8_t lens[320];
};

struct InflateJob {
  unsigned long long src, src_len;   // the stream in the group's file buffer
  unsigned long long out, cap;       // its region of expected bytes in the inflated buffer
  unsigned long long ring;           // its 32 KB ring in the inflated buffer
};

// LSB-first reader of one stream; bytes past its end read as 0 and are caught by over()
struct Bits {
  const unsigned char* p;
  unsigned long long n, next, buf;
  int nb;
  __device__ __forceinline__ void seek(unsigned long long byte) {
    next = byte;
    buf = 0;
    nb = 0;
  }
  __device__ __forceinline__ void fill() {
    while (nb <= 56) {
      const unsigned long long b = next < n ? p[next] : 0ull;
      buf |= b << nb;
      nb += 8;
      ++next;
    }
  }
  __device__ __forceinline__ uint32_t get(int k) {  // 0 <= k <= 32
    fill();
    const uint32_t v = static_cast<uint32_t>(buf & ((1ull << k) - 1));
    buf >>= k;
    nb -= k;
    return v;
  }
  __device__ __forceinline__ unsigned long long consumed() const { return next * 8 - nb; }
  __device__ __forceinline__ bool over() const { return consumed() > n * 8; }
};

__device__ __forceinline__ uint32_t reverse_bits(uint32_t v, int l) {
  uint32_t r = 0;
  for (int k = 0; k < l; ++k) r |= ((v >> k) & 1u) << (l - 1 - k);
  return r;
}

// Builds h from lens[0, n) with zlib's acceptance (inftrees.c): an over-subscribed set fails; an incomplete one fails
// unless it is a literal / distance code of a single length-1 code; an empty literal / distance code builds (every
// symbol then fails to decode), an empty code-length code fails.  Warp-collective; the result is warp-uniform.
template <int LB, int NSYM>
__device__ bool build_huff(Huff<LB, NSYM>& h, const uint8_t* lens, int n, bool codes) {
  const int lane = threadIdx.x & 31;
  if (lane < 16) h.count[lane] = 0;
  for (int i = lane; i < (1 << LB); i += 32) h.lut[i] = 0;
  __syncwarp();
  for (int s = lane; s < n; s += 32)
    if (lens[s]) atomicAdd(&h.count[lens[s]], 1u);
  __syncwarp();
  int left = 1, maxlen = 0;
  uint32_t offs = 0, code = 0, prev = 0, my_offs = 0, my_code = 0;
  for (int l = 1; l <= 15; ++l) {
    const uint32_t c = h.count[l];
    code = (code + prev) << 1;
    if (lane == l) {
      my_offs = offs;
      my_code = code;
    }
    offs += c;
    prev = c;
    left = (left << 1) - static_cast<int>(c);
    if (left < 0) break;
    if (c) maxlen = l;
  }
  if (left < 0) return false;
  if (maxlen == 0) {
    if (codes) return false;
  } else if (left > 0 && (codes || maxlen != 1)) {
    return false;
  }
  // the symbols in code order: lane l holds the next free position of length l
  const uint32_t offs0 = my_offs;
  for (int base = 0; base < n; base += 32) {
    const int s = base + lane;
    const int l = s < n ? lens[s] : 0;
    uint32_t rank = 0, batch = 0;
    for (int L = 1; L <= 15; ++L) {
      const uint32_t m = __ballot_sync(kFull, l == L);
      if (l == L) rank = __popc(m & ((1u << lane) - 1u));
      if (lane == L) batch = __popc(m);
    }
    const uint32_t start = __shfl_sync(kFull, my_offs, l);
    if (l) h.sym[start + rank] = static_cast<uint16_t>(s);
    my_offs += batch;
  }
  __syncwarp();
  for (uint32_t base = 0; base < offs; base += 32) {
    const uint32_t p = base + lane;
    const int s = p < offs ? h.sym[p] : 0;
    const int l = p < offs ? lens[s] : 0;
    const uint32_t o = __shfl_sync(kFull, offs0, l), fc = __shfl_sync(kFull, my_code, l);
    if (l && l <= LB) {
      const uint32_t rev = reverse_bits(fc + (p - o), l);
      for (uint32_t k = rev; k < (1u << LB); k += 1u << l) h.lut[k] = static_cast<uint16_t>((s << 4) | l);
    }
  }
  __syncwarp();
  return true;
}

// The next symbol of h, or -1 for a code h does not hold (puff.c's canonical walk past the table)
template <int LB, int NSYM>
__device__ __forceinline__ int decode_sym(const Huff<LB, NSYM>& h, Bits& br) {
  br.fill();
  const uint32_t e = h.lut[br.buf & ((1u << LB) - 1u)];
  if (e) {
    br.buf >>= (e & 15u);
    br.nb -= static_cast<int>(e & 15u);
    return static_cast<int>(e >> 4);
  }
  int code = 0, first = 0, index = 0;
  for (int len = 1; len <= 15; ++len) {
    code |= static_cast<int>((br.buf >> (len - 1)) & 1ull);
    const int c = static_cast<int>(h.count[len]);
    if (code - first < c) {
      br.buf >>= len;
      br.nb -= len;
      return h.sym[index + (code - first)];
    }
    index += c;
    first = (first + c) << 1;
    code <<= 1;
  }
  return -1;
}

// The output of one stream: [0, cap) in its region, past that in its ring; Adler-32 sums of the bytes this lane wrote
struct Out {
  unsigned char* region;
  unsigned char* ring;
  unsigned long long cap;
  unsigned long long s, w;
  __device__ __forceinline__ unsigned char* at(unsigned long long pos) const {
    return pos < cap ? region + pos : ring + (pos & (kRing - 1));
  }
  __device__ __forceinline__ void put(unsigned long long pos, unsigned int b) {
    *at(pos) = static_cast<unsigned char>(b);
    s += b;
    w += pos * b;
    if (w >> 60) w %= kAdlerMod;
  }
};

enum : int { kOk = 0, kBad = 1 };

__device__ int inflate_stream(InflateSmem& sm, const unsigned char* src, unsigned long long n, Out& out,
                              unsigned long long* total) {
  const int lane = threadIdx.x & 31;
  if (n < 2) return kBad;
  const uint32_t cmf = src[0], flg = src[1];
  if ((cmf * 256u + flg) % 31u != 0 || (cmf & 15u) != 8u || (cmf >> 4) + 8u > 15u || (flg & 0x20u)) return kBad;
  Bits br{src, n, 0, 0, 0};
  br.seek(2);
  unsigned long long pos = 0;
  bool fixed_loaded = false, last = false;
  while (!last) {
    last = br.get(1) != 0;
    const uint32_t type = br.get(2);
    if (br.over()) return kBad;
    if (type == 0) {  // stored
      br.get(br.nb & 7);
      const uint32_t len = br.get(16), nlen = br.get(16);
      if (br.over() || len != (nlen ^ 0xffffu)) return kBad;
      const unsigned long long at = br.consumed() / 8;
      if (at + len > n) return kBad;
      for (uint32_t i = lane; i < len; i += 32) out.put(pos + i, src[at + i]);
      __syncwarp();
      pos += len;
      br.seek(at + len);
      continue;
    }
    if (type == 3) return kBad;
    if (type == 1) {
      if (!fixed_loaded) {
        for (int s = lane; s < 288; s += 32) sm.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        __syncwarp();
        build_huff(sm.lit, sm.lens, 288, false);
        for (int s = lane; s < 32; s += 32) sm.lens[s] = 5;
        __syncwarp();
        build_huff(sm.dist, sm.lens, 32, false);
        fixed_loaded = true;
      }
    } else {  // dynamic
      fixed_loaded = false;
      const int nlen = static_cast<int>(br.get(5)) + 257, ndist = static_cast<int>(br.get(5)) + 1;
      const int ncode = static_cast<int>(br.get(4)) + 4;
      if (nlen > 286 || ndist > 30) return kBad;
      if (lane < 19) sm.lens[lane] = 0;
      __syncwarp();
      for (int k = 0; k < ncode; ++k) {
        const uint32_t v = br.get(3);
        if (lane == 0) sm.lens[kClOrder[k]] = static_cast<uint8_t>(v);
      }
      __syncwarp();
      if (br.over() || !build_huff(sm.dist, sm.lens, 19, true)) return kBad;
      const int all = nlen + ndist;
      int idx = 0, prev = 0;
      while (idx < all) {
        const int sym = decode_sym(sm.dist, br);
        if (sym < 0) return kBad;
        int rep = 1, v = sym;
        if (sym == 16) {
          if (idx == 0) return kBad;
          v = prev;
          rep = 3 + static_cast<int>(br.get(2));
        } else if (sym == 17) {
          v = 0;
          rep = 3 + static_cast<int>(br.get(3));
        } else if (sym == 18) {
          v = 0;
          rep = 11 + static_cast<int>(br.get(7));
        }
        if (br.over() || idx + rep > all) return kBad;
        for (int k = lane; k < rep; k += 32) sm.lens[idx + k] = static_cast<uint8_t>(v);
        idx += rep;
        prev = v;
      }
      __syncwarp();
      if (sm.lens[256] == 0) return kBad;
      if (!build_huff(sm.lit, sm.lens, nlen, false)) return kBad;
      if (!build_huff(sm.dist, sm.lens + nlen, ndist, false)) return kBad;
    }
    for (;;) {
      const int sym = decode_sym(sm.lit, br);
      if (sym < 0 || br.over()) return kBad;
      if (sym < 256) {
        if (lane == 0) out.put(pos, static_cast<unsigned int>(sym));
        ++pos;
        continue;
      }
      if (sym == 256) break;
      if (sym >= 286) return kBad;
      const uint32_t len = kLenBase[sym - 257] + br.get(kLenExtra[sym - 257]);
      const int dsym = decode_sym(sm.dist, br);
      if (dsym < 0 || dsym >= 30) return kBad;
      const uint32_t dist = kDistBase[dsym] + br.get(kDistExtra[dsym]);
      if (br.over() || dist > pos) return kBad;
      __syncwarp();  // the literals lane 0 wrote are visible to every lane
      const uint32_t c = dist < 32u ? dist : 32u;
      for (uint32_t done = 0; done < len; done += c) {  // a round reads only bytes written before it
        const uint32_t i = done + lane;
        const bool copy = lane < c && i < len;
        const unsigned int b = copy ? *out.at(pos + i - dist) : 0u;
        __syncwarp();  // every read of the round before any write: in the ring a read and another lane's write of the
                       // same round can share a slot (distances within 31 of 32768)
        if (copy) out.put(pos + i, b);
        __syncwarp();
      }
      pos += len;
    }
  }
  // the Adler-32, big-endian, at the next byte boundary
  br.get(br.nb & 7);
  const unsigned long long at = br.consumed() / 8;
  if (at + 4 > n) return kBad;
  const uint32_t want = (static_cast<uint32_t>(src[at]) << 24) | (static_cast<uint32_t>(src[at + 1]) << 16) |
                        (static_cast<uint32_t>(src[at + 2]) << 8) | src[at + 3];
  unsigned long long s = out.s % kAdlerMod, w = out.w % kAdlerMod;
  for (int o = 16; o; o >>= 1) {
    s += __shfl_xor_sync(kFull, s, o);
    w += __shfl_xor_sync(kFull, w, o);
  }
  unsigned long long a = 1, b = pos % kAdlerMod;
  adler_add_segment(pos, 0, s, w, &a, &b);
  *total = pos;
  return static_cast<uint32_t>((b << 16) | a) == want ? kOk : kBad;
}

__global__ void __launch_bounds__(32 * kInflateWarps)
    inflate_kernel(const InflateJob* __restrict__ jobs, uint32_t n_jobs, const unsigned char* __restrict__ files,
                   unsigned char* __restrict__ inflated, int* __restrict__ status) {
  __shared__ InflateSmem smem[kInflateWarps];
  const int warp = threadIdx.x >> 5;
  const uint32_t j = blockIdx.x * kInflateWarps + warp;
  if (j >= n_jobs) return;
  const InflateJob job = jobs[j];
  Out out{inflated + job.out, inflated + job.ring, job.cap, 0, 0};
  unsigned long long total = 0;
  const int st = inflate_stream(smem[warp], files + job.src, job.src_len, out, &total);
  if ((threadIdx.x & 31) == 0) status[j] = st == kOk && total >= job.cap ? kOk : kBad;
}

// ---- unpredict + convert ---------------------------------------------------------------------------------------------
struct UnpredictShape {
  int32_t cols, spp, band, item, sample, predictor;
  int32_t r0, c0, c1;        // the window: image rows from r0, columns [c0, c1)
  int32_t width;
  unsigned long long stride; // floats between the band's rows
};

struct RowJob {
  unsigned long long at;     // the row's bytes in `inflated` (or `files` when raw)
  unsigned long long sum;    // predictor 3: where its summed bytes go in `inflated` (at itself unless raw)
  int32_t r, c;              // its image row and the chunk's first column
  int32_t raw;
  int32_t pad;
};

__device__ __forceinline__ unsigned long long load_le(const unsigned char* p, int item) {
  unsigned long long v = 0;
  for (int k = 0; k < item; ++k) v |= static_cast<unsigned long long>(p[k]) << (8 * k);
  return v;
}

__device__ __forceinline__ float to_f32(unsigned long long v, int sample) {
  switch (sample) {
    case AMB_SAMPLE_U8: return static_cast<float>(static_cast<uint32_t>(v & 0xffu));
    case AMB_SAMPLE_I16: return static_cast<float>(static_cast<int16_t>(static_cast<uint16_t>(v)));
    case AMB_SAMPLE_U16: return static_cast<float>(static_cast<uint32_t>(v & 0xffffu));
    case AMB_SAMPLE_I32: return static_cast<float>(static_cast<int32_t>(static_cast<uint32_t>(v)));
    case AMB_SAMPLE_F32: return __uint_as_float(static_cast<uint32_t>(v));
    default: return __double2float_rn(__longlong_as_double(static_cast<long long>(v)));
  }
}

__global__ void __launch_bounds__(kUnpredictThreads)
    unpredict_kernel(const UnpredictShape s, const RowJob* __restrict__ jobs, unsigned char* __restrict__ files,
                     unsigned char* __restrict__ inflated, float* __restrict__ out) {
  const RowJob job = jobs[blockIdx.x];
  unsigned char* row = (job.raw ? files : inflated) + job.at;
  float* dst = out + static_cast<unsigned long long>(job.r - s.r0) * s.stride;
  const int lo = max(s.c0, job.c), hi = min(min(s.c1, s.width), job.c + s.cols);  // image columns to store
  const int tid = threadIdx.x;
  const unsigned long long width_mask = s.item == 8 ? ~0ull : (1ull << (8 * s.item)) - 1;
  if (s.predictor == 1) {
    for (int c = lo + tid; c < hi; c += kUnpredictThreads) {
      const unsigned long long k = static_cast<unsigned long long>(c - job.c) * s.spp + s.band;
      dst[c - s.c0] = to_f32(load_le(row + k * s.item, s.item), s.sample);
    }
    return;
  }
  if (s.predictor == 2) {  // samples of the band, summed modulo the sample type
    unsigned long long carry = 0;
    for (int base = 0; base < s.cols; base += kUnpredictThreads) {
      const int q = base + tid;
      const unsigned long long x =
          q < s.cols ? load_le(row + (static_cast<unsigned long long>(q) * s.spp + s.band) * s.item, s.item) : 0ull;
      unsigned long long tile;
      const unsigned long long v = (carry + block_exclusive<kUnpredictThreads>(x, &tile) + x) & width_mask;
      const int c = job.c + q;
      if (q < s.cols && c >= lo && c < hi) dst[c - s.c0] = to_f32(v, s.sample);
      carry += tile;
    }
    return;
  }
  // predictor 3: the band's bytes along the row's planes, summed mod 256 into the row's own scratch (never the file's
  // bytes, which another chunk may share), then gathered big-endian
  const int L = s.cols * s.item;
  unsigned char* sum = inflated + job.sum;
  unsigned long long carry = 0;
  for (int base = 0; base < L; base += kUnpredictThreads) {
    const int q = base + tid;
    const unsigned long long k = static_cast<unsigned long long>(q) * s.spp + s.band;
    const unsigned long long x = q < L ? row[k] : 0ull;
    unsigned long long tile;
    const unsigned long long v = carry + block_exclusive<kUnpredictThreads>(x, &tile) + x;
    if (q < L) sum[k] = static_cast<unsigned char>(v);
    carry += tile;
  }
  __syncthreads();
  for (int c = lo + tid; c < hi; c += kUnpredictThreads) {
    unsigned long long v = 0;
    for (int k = 0; k < s.item; ++k)
      v = (v << 8) | sum[(static_cast<unsigned long long>(k) * s.cols + (c - job.c)) * s.spp + s.band];
    dst[c - s.c0] = to_f32(v, s.sample);
  }
}

int sample_bytes(int sample) {
  switch (sample) {
    case AMB_SAMPLE_U8: return 1;
    case AMB_SAMPLE_I16:
    case AMB_SAMPLE_U16: return 2;
    case AMB_SAMPLE_I32:
    case AMB_SAMPLE_F32: return 4;
    case AMB_SAMPLE_F64: return 8;
    default: return 0;
  }
}

struct ChunkRect {
  int32_t r, c, rows, cols;  // image row and column of its corner, its rows and columns of data
};

ChunkRect chunk_rect(const amb_tiff_layout& L, uint32_t k) {
  if (L.tiled) {
    const uint32_t across = static_cast<uint32_t>((L.width + L.chunk_width - 1) / L.chunk_width);
    return ChunkRect{static_cast<int32_t>(k / across) * L.chunk_height, static_cast<int32_t>(k % across) * L.chunk_width,
                     L.chunk_height, L.chunk_width};
  }
  const int32_t r = static_cast<int32_t>(k) * L.chunk_height;
  return ChunkRect{r, 0, std::min(L.chunk_height, L.height - r), L.width};
}

size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

// One group of chunks (indices into the layout, all meeting the window): copied, inflated, unpredicted into `out`.
// Returns AMB_ERR_CORRUPT_DATA if a chunk does not inflate.
int decode_group(amb_ctx* ctx, const unsigned char* file, const amb_tiff_layout& L, const std::vector<uint32_t>& chunks,
                 int32_t r0, int32_t r1, int32_t c0, int32_t c1, float* out, size_t stride) {
  cudaStream_t st = ctx->stream;
  const bool raw = L.compression == 1;
  const unsigned long long row_bytes =
      static_cast<unsigned long long>(L.chunk_width) * L.spp * sample_bytes(L.sample);
  // the chunks' file ranges, those that touch or overlap merged into spans copied in one piece: only bytes of the
  // window's chunks cross PCIe
  std::vector<uint32_t> order(chunks);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return L.offsets[a] < L.offsets[b]; });
  struct Span {
    unsigned long long begin, end, dev;
  };
  std::vector<Span> spans;
  for (size_t k = 0; k < order.size(); ++k) {
    const unsigned long long b = L.offsets[order[k]], e = b + L.byte_counts[order[k]];
    if (spans.empty() || b > spans.back().end) {  // only touching or overlapping chunks share a copy
      const unsigned long long dev = spans.empty() ? 0 : align256(spans.back().dev + spans.back().end - spans.back().begin);
      spans.push_back(Span{b, e, dev});
    } else {
      spans.back().end = std::max(spans.back().end, e);
    }
  }
  const unsigned long long file_bytes = spans.empty() ? 0 : spans.back().dev + spans.back().end - spans.back().begin;
  AMB_CUDA(ctx, ctx->tiff_files.reserve(file_bytes + 256));
  unsigned char* d_files = ctx->tiff_files.as<unsigned char>();
  for (const Span& s : spans) {
    const int rc = staged_h2d(ctx, d_files + s.dev, file + s.begin, s.end - s.begin, st);
    if (rc != AMB_OK) return rc;
  }
  auto dev_offset = [&](uint32_t k) {  // chunk k's first byte in the group's file buffer
    const unsigned long long b = L.offsets[k];
    const Span& s = *(std::upper_bound(spans.begin(), spans.end(), b,
                                       [](unsigned long long v, const Span& x) { return v < x.begin; }) - 1);
    return s.dev + (b - s.begin);
  };
  std::vector<InflateJob> infl;
  std::vector<RowJob> rows;
  unsigned long long infl_bytes = 0;
  for (uint32_t k : chunks) {
    const ChunkRect cr = chunk_rect(L, k);
    const unsigned long long at = dev_offset(k);
    unsigned long long data = at;
    if (!raw) {
      const unsigned long long cap = row_bytes * static_cast<unsigned long long>(cr.rows);
      infl.push_back(InflateJob{at, L.byte_counts[k], infl_bytes, cap, 0});
      data = infl_bytes;
      infl_bytes += align256(cap);
    }
    const int32_t first = std::max(r0, cr.r), last = std::min(r1, cr.r + cr.rows);
    unsigned long long sum = data;  // predictor 3 sums in place in the chunk's own inflated bytes
    if (raw && L.predictor == 3) {  // an uncompressed chunk's rows are summed into scratch of their own
      sum = infl_bytes - static_cast<unsigned long long>(first - cr.r) * row_bytes;
      infl_bytes += align256(static_cast<unsigned long long>(last - first) * row_bytes);
    }
    for (int32_t r = first; r < last; ++r) {
      const unsigned long long off = static_cast<unsigned long long>(r - cr.r) * row_bytes;
      rows.push_back(RowJob{data + off, sum + off, r, cr.c, raw ? 1 : 0, 0});
    }
  }
  for (InflateJob& j : infl) {
    j.ring = infl_bytes;
    infl_bytes += kRing;
  }
  AMB_CUDA(ctx, ctx->tiff_inflated.reserve(infl_bytes + 256));
  const size_t meta_bytes = align256(infl.size() * sizeof(InflateJob)) + align256(rows.size() * sizeof(RowJob)) +
                            align256(infl.size() * sizeof(int));
  AMB_CUDA(ctx, ctx->tiff_meta.reserve(meta_bytes + 256));
  unsigned char* mp = ctx->tiff_meta.as<unsigned char>();
  InflateJob* d_infl = reinterpret_cast<InflateJob*>(mp);
  RowJob* d_rows = reinterpret_cast<RowJob*>(mp + align256(infl.size() * sizeof(InflateJob)));
  int* d_status = reinterpret_cast<int*>(mp + align256(infl.size() * sizeof(InflateJob)) +
                                         align256(rows.size() * sizeof(RowJob)));
  if (!infl.empty()) {
    AMB_CUDA(ctx, cudaMemcpyAsync(d_infl, infl.data(), infl.size() * sizeof(InflateJob), cudaMemcpyHostToDevice, st));
    const uint32_t n = static_cast<uint32_t>(infl.size());
    inflate_kernel<<<(n + kInflateWarps - 1) / kInflateWarps, 32 * kInflateWarps, 0, st>>>(
        d_infl, n, d_files, ctx->tiff_inflated.as<unsigned char>(), d_status);
    AMB_CUDA(ctx, cudaGetLastError());
  }
  if (!rows.empty()) {
    AMB_CUDA(ctx, cudaMemcpyAsync(d_rows, rows.data(), rows.size() * sizeof(RowJob), cudaMemcpyHostToDevice, st));
    UnpredictShape s;
    s.cols = L.chunk_width;
    s.spp = L.spp;
    s.band = L.band;
    s.item = sample_bytes(L.sample);
    s.sample = L.sample;
    s.predictor = L.predictor;
    s.r0 = r0;
    s.c0 = c0;
    s.c1 = c1;
    s.width = L.width;
    s.stride = stride;
    unpredict_kernel<<<static_cast<unsigned int>(rows.size()), kUnpredictThreads, 0, st>>>(
        s, d_rows, d_files, ctx->tiff_inflated.as<unsigned char>(), out);
    AMB_CUDA(ctx, cudaGetLastError());
  }
  std::vector<int> status(infl.size(), kOk);
  if (!infl.empty())
    AMB_CUDA(ctx, cudaMemcpyAsync(status.data(), d_status, infl.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  AMB_CUDA(ctx, cudaStreamSynchronize(st));
  for (int v : status)
    if (v != kOk) return AMB_ERR_CORRUPT_DATA;
  return AMB_OK;
}

}  // namespace

int tiff_layout_check(const amb_tiff_layout* L, size_t bytes) {
  if (!L || !L->offsets || !L->byte_counts || L->width < 1 || L->height < 1 || L->chunk_width < 1 ||
      L->chunk_height < 1 || L->spp < 1 || L->band < 0 || L->band >= L->spp || sample_bytes(L->sample) == 0)
    return AMB_ERR_INVALID_ARGUMENT;
  const bool is_float = L->sample == AMB_SAMPLE_F32 || L->sample == AMB_SAMPLE_F64;
  if ((L->compression != 1 && L->compression != 8 && L->compression != 32946) ||
      (L->predictor != 1 && L->predictor != 2 && L->predictor != 3) || (L->predictor == 2 && is_float) ||
      (L->predictor == 3 && !is_float))
    return AMB_ERR_INVALID_ARGUMENT;
  if (!L->tiled && L->chunk_width != L->width) return AMB_ERR_INVALID_ARGUMENT;
  const unsigned long long down = (static_cast<unsigned long long>(L->height) + L->chunk_height - 1) / L->chunk_height;
  const unsigned long long across =
      L->tiled ? (static_cast<unsigned long long>(L->width) + L->chunk_width - 1) / L->chunk_width : 1;
  if (L->n_chunks != down * across) return AMB_ERR_INVALID_ARGUMENT;
  const unsigned long long chunk = static_cast<unsigned long long>(L->chunk_width) * L->spp *
                                   sample_bytes(L->sample) * static_cast<unsigned long long>(L->chunk_height);
  if (chunk > (1ull << 32)) return AMB_ERR_INVALID_ARGUMENT;
  for (uint32_t k = 0; k < L->n_chunks; ++k)
    if (L->offsets[k] > bytes || L->byte_counts[k] > bytes - L->offsets[k]) return AMB_ERR_INVALID_ARGUMENT;
  return AMB_OK;
}

int tiff_decode_window(amb_ctx* ctx, const unsigned char* file, const amb_tiff_layout& L, int32_t r0, int32_t r1,
                       int32_t c0, int32_t c1, float* out, size_t stride) {
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const unsigned long long row_bytes = static_cast<unsigned long long>(L.chunk_width) * L.spp * sample_bytes(L.sample);
  std::vector<uint32_t> group;
  size_t used = 0;
  for (uint32_t k = 0; k < L.n_chunks; ++k) {
    const ChunkRect cr = chunk_rect(L, k);
    if (cr.r >= r1 || cr.r + cr.rows <= r0 || cr.c >= c1 || cr.c + cr.cols <= c0) continue;
    const unsigned long long expected = row_bytes * static_cast<unsigned long long>(cr.rows);
    if (L.compression == 1 && L.byte_counts[k] < expected) return AMB_ERR_CORRUPT_DATA;
    const size_t need = L.byte_counts[k] + (L.compression != 1 ? align256(expected) + kRing
                                                                 : L.predictor == 3 ? align256(expected) : 0) + 512;
    if (!group.empty() && used + need > kGroupBudget) {
      const int rc = decode_group(ctx, file, L, group, r0, r1, c0, c1, out, stride);
      if (rc != AMB_OK) return rc;
      group.clear();
      used = 0;
    }
    group.push_back(k);
    used += need;
  }
  if (group.empty()) return AMB_OK;
  return decode_group(ctx, file, L, group, r0, r1, c0, c1, out, stride);
}

}  // namespace amb

using namespace amb;

extern "C" {

int amb_tiff_decode_device(amb_ctx* ctx, const void* file, size_t bytes, const amb_tiff_layout* layout, int32_t r0,
                           int32_t r1, int32_t c0, int32_t c1, float* d_band, size_t row_stride) {
  if (!ctx || !file || !d_band || (reinterpret_cast<uintptr_t>(d_band) & 3) != 0) return AMB_ERR_INVALID_ARGUMENT;
  const int rc = tiff_layout_check(layout, bytes);
  if (rc != AMB_OK) return rc;
  if (r0 < 0 || r1 > layout->height || r0 >= r1 || c0 < 0 || c1 > layout->width || c0 >= c1 || row_stride % 4 != 0 ||
      row_stride < 4 * static_cast<size_t>(c1 - c0))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  // into the context's scratch first: a corrupt chunk leaves the caller's band untouched
  const size_t w = static_cast<size_t>(c1 - c0), h = static_cast<size_t>(r1 - r0);
  AMB_CUDA(ctx, ctx->raster_band.reserve(w * h * sizeof(float)));
  const int st = tiff_decode_window(ctx, static_cast<const unsigned char*>(file), *layout, r0, r1, c0, c1,
                                    ctx->raster_band.as<float>(), w);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaMemcpy2DAsync(d_band, row_stride, ctx->raster_band.ptr, w * sizeof(float), w * sizeof(float), h,
                                  cudaMemcpyDeviceToDevice, ctx->stream));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return AMB_OK;
}

}  // extern "C"
