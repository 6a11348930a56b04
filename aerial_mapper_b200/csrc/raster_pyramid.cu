// raster_pyramid.cu — the tiles of a Cloud-Optimized GeoTIFF of a raster in device memory: the overview pyramid, every
// level cut into T x T tiles, and the tiles compressed by the Deflate encoder (convention in include/aerial_mapper_b200.h,
// amb_cog_tiles_device).  Three steps:
//   reduce  level k -> level k + 1, one block per output row, one thread per 16 bytes of it (4 F32, 16 GRAY8 / MASK8 or
//           16 BGR8 pixels in 48 bytes): the 2 x 2 children of each pixel from two input rows, loads coalesced along the
//           rows, 16-byte stores where the output piece is whole.  Levels 1.. are kept with rows padded to 16 bytes.
//   tile    every level into its tiles, one block (32 x 8 threads) per tile: 16-byte pieces of the tile rows, the bytes
//           outside the level zero.  All tiles of all levels go into one buffer, smallest level first,
//           each level's tiles row-major, so the buffer is a raster T pixels wide and n_tiles * T rows high.
//   deflate that raster compressed by deflate_encode (deflate_encode.cu) in strips of T rows: strip k is tile k.
// The JPEG tiles (amb_cog_jpeg_tiles_device) encode the stacked raster instead as one JPEG image with a restart interval
// per tile, split into one abbreviated stream per tile (jpeg_encode.cu).  The 1-bit mask tiles (amb_cog_mask_tiles_device)
// pack the stacked MASK8 tiles to bits (mask_pack_kernel) and deflate them without a predictor.
// One-dimensional grids with grid-stride loops over rows and tiles; offsets are 64-bit.
#include <algorithm>

#include "deflate_encode.h"
#include "jpeg_encode.h"

namespace amb {
namespace {

constexpr int kMaxLevels = 32;
constexpr int kReduceThreads = 256;

__host__ __device__ constexpr int cog_bpp(int fmt) { return fmt == AMB_RASTER_F32 ? 4 : fmt == AMB_RASTER_BGR8 ? 3 : 1; }

__device__ __forceinline__ bool nan_bits(uint32_t b) { return (b & 0x7fffffffu) > 0x7f800000u; }

// ---- reduce -------------------------------------------------------------------------------------------------------------
// One output pixel from its m present children c[0..m) in the order (0,0), (0,1), (1,0), (1,1).  F32: the mean of the
// non-NaN children in IEEE double, every operation rounded; a NaN result (no such child, or +inf and -inf among them) is
// the quiet NaN 0x7FC00000.  GRAY8 / BGR8: the rounded mean of each byte.  MASK8: the maximum.
template <int FMT>
__device__ __forceinline__ uint32_t reduce_children(const uint32_t* c, int m) {
  if (FMT == AMB_RASTER_F32) {
    double s = 0.0;
    int n = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < m && !nan_bits(c[k])) {
        const double v = static_cast<double>(__uint_as_float(c[k]));
        s = n == 0 ? v : __dadd_rn(s, v);
        ++n;
      }
    if (n == 0) return 0x7fc00000u;
    const uint32_t b = __float_as_uint(__double2float_rn(__ddiv_rn(s, static_cast<double>(n))));
    return nan_bits(b) ? 0x7fc00000u : b;
  } else if (FMT == AMB_RASTER_MASK8) {
    uint32_t v = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (k < m) v = max(v, c[k]);
    return v;
  } else {
    constexpr int CH = FMT == AMB_RASTER_BGR8 ? 3 : 1;
    const uint32_t half = static_cast<uint32_t>(m) >> 1;
    uint32_t out = 0;
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      uint32_t s = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k < m) s += (c[k] >> (8 * ch)) & 0xffu;
      out |= ((s + half) / static_cast<uint32_t>(m)) << (8 * ch);
    }
    return out;
  }
}

template <int FMT>
__device__ __forceinline__ uint32_t load_pixel(const unsigned char* row, long long x) {
  if (FMT == AMB_RASTER_F32) return __ldg(reinterpret_cast<const uint32_t*>(row) + x);
  if (FMT == AMB_RASTER_BGR8)
    return __ldg(row + 3 * x) | (static_cast<uint32_t>(__ldg(row + 3 * x + 1)) << 8) |
           (static_cast<uint32_t>(__ldg(row + 3 * x + 2)) << 16);
  return __ldg(row + x);
}

// Output pixels [x0, x0 + npx) (npx <= PX) of a row from its input rows r0 and r1 (has_r1: r1 is inside the level),
// written to out: 16-byte stores when the piece is whole (dst rows and pieces are 16-byte aligned), else byte stores.
template <int FMT, int PX>
__device__ __forceinline__ void reduce_piece(const unsigned char* r0, const unsigned char* r1, bool has_r1, int32_t sw,
                                             long long x0, int npx, unsigned char* out) {
  constexpr int BPP = cog_bpp(FMT);
  constexpr int NW = PX * BPP / 4;  // 32-bit words of the piece
  uint32_t word[NW];
#pragma unroll
  for (int i = 0; i < NW; ++i) word[i] = 0;
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    if (p < npx) {
      const long long cx = 2 * (x0 + p);
      const bool has_c1 = cx + 1 < sw;
      uint32_t c[4];
      int m = 0;
      c[m++] = load_pixel<FMT>(r0, cx);
      if (has_c1) c[m++] = load_pixel<FMT>(r0, cx + 1);
      if (has_r1) {
        c[m++] = load_pixel<FMT>(r1, cx);
        if (has_c1) c[m++] = load_pixel<FMT>(r1, cx + 1);
      }
      const uint32_t v = reduce_children<FMT>(c, m);
#pragma unroll
      for (int q = 0; q < BPP; ++q) {
        const int b = p * BPP + q;  // byte of the piece
        word[b >> 2] |= ((v >> (8 * q)) & 0xffu) << (8 * (b & 3));
      }
    }
  }
  if (npx == PX) {
#pragma unroll
    for (int q = 0; q < NW / 4; ++q)
      reinterpret_cast<uint4*>(out)[q] = make_uint4(word[4 * q], word[4 * q + 1], word[4 * q + 2], word[4 * q + 3]);
  } else {
#pragma unroll
    for (int b = 0; b < NW * 4; ++b)
      if (b < npx * BPP) out[b] = static_cast<unsigned char>(word[b >> 2] >> (8 * (b & 3)));
  }
}

// dst (dw x dh, rows dst_stride bytes apart, 16-byte aligned) = the reduction of src (sw x sh, rows src_stride apart);
// block b makes rows y = b, b + gridDim.x, ...; thread t of it output pixels [PX x, PX x + PX) for x = t, t + blockDim.x ...
template <int FMT>
__global__ void __launch_bounds__(kReduceThreads)
    pyramid_reduce_kernel(const unsigned char* __restrict__ src, unsigned long long src_stride, int32_t sw, int32_t sh,
                          unsigned char* __restrict__ dst, unsigned long long dst_stride, int32_t dw, int32_t dh) {
  constexpr int PX = FMT == AMB_RASTER_F32 ? 4 : 16;  // pixels per thread: 16 or 48 bytes, whole 16-byte stores
  for (int y = blockIdx.x; y < dh; y += gridDim.x) {
    const unsigned char* r0 = src + static_cast<unsigned long long>(2 * static_cast<long long>(y)) * src_stride;
    const bool has_r1 = 2 * static_cast<long long>(y) + 1 < sh;
    unsigned char* row = dst + static_cast<unsigned long long>(y) * dst_stride;
    for (long long x0 = static_cast<long long>(threadIdx.x) * PX; x0 < dw; x0 += static_cast<long long>(blockDim.x) * PX)
      reduce_piece<FMT, PX>(r0, r0 + src_stride, has_r1, sw, x0, static_cast<int>(min(static_cast<long long>(PX), dw - x0)),
                            row + static_cast<unsigned long long>(x0) * cog_bpp(FMT));
  }
}

// ---- tile -----------------------------------------------------------------------------------------------------------------
// The level (rows of row_bytes bytes, `stride` apart) into tiles_x x tiles_y tiles of T rows of tile_row bytes (a
// multiple of 16), tile (ty, tx) at dst + (ty * tiles_x + tx) * T rows.  Block b makes tiles b, b + gridDim.x, ...:
// threadIdx.y picks the tile rows, threadIdx.x the 16-byte pieces of a row; bytes past the level's right or bottom edge
// are zero.
__global__ void __launch_bounds__(256)
    pyramid_tile_kernel(const unsigned char* __restrict__ src, unsigned long long stride, unsigned long long row_bytes,
                        int32_t h, int32_t T, int32_t tile_row, int32_t tiles_x, int32_t n_tiles,
                        uint4* __restrict__ dst) {
  const int pieces = tile_row >> 4;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {  // n_tiles * T < 2^31 (cog_plan)
    const int ty = tile / tiles_x, tx = tile - ty * tiles_x;         // once per tile
    const unsigned long long xb = static_cast<unsigned long long>(tx) * tile_row;  // the tile's first byte in a level row
    for (int r = threadIdx.y; r < T; r += blockDim.y) {
      const long long y = static_cast<long long>(ty) * T + r;
      const unsigned char* row = src + static_cast<unsigned long long>(y) * stride;
      uint4* out = dst + (static_cast<unsigned long long>(tile) * T + r) * pieces;
      for (int q = threadIdx.x; q < pieces; q += blockDim.x) {
        const unsigned long long b = xb + 16ull * q;
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (y < h && b < row_bytes) {
          if (b + 16 <= row_bytes && (reinterpret_cast<uintptr_t>(row + b) & 15) == 0) {
            v = __ldg(reinterpret_cast<const uint4*>(row + b));
          } else {
            uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
            for (int i = 0; i < 16; ++i)
              if (b + i < row_bytes) w[i >> 2] |= static_cast<uint32_t>(__ldg(row + b + i)) << (8 * (i & 3));
            v = make_uint4(w[0], w[1], w[2], w[3]);
          }
        }
        out[q] = v;
      }
    }
  }
}

// ---- mask ------------------------------------------------------------------------------------------------------------------
// The stacked MASK8 tiles (n pieces of 16 bytes) at 1 bit per pixel, most significant bit first, 1 where the byte is not
// 0: piece i becomes bytes 2i and 2i + 1.  A tile row is T / 16 whole pieces (16 | T), so rows of T / 8 bytes.
__global__ void __launch_bounds__(256)
    mask_pack_kernel(const uint4* __restrict__ src, unsigned long long n, uint16_t* __restrict__ dst) {
  for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const uint4 v = __ldg(src + i);
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    uint32_t bits = 0;  // pixel q at bit 15 - q
#pragma unroll
    for (int q = 0; q < 16; ++q) bits |= (((w[q >> 2] >> (8 * (q & 3))) & 0xffu) != 0u ? 1u : 0u) << (15 - q);
    dst[i] = static_cast<uint16_t>((bits >> 8) | ((bits & 0xffu) << 8));  // little-endian: pixels 0..7 in the first byte
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------------
struct CogPlan {
  int32_t n_levels;
  int32_t w[kMaxLevels], h[kMaxLevels];
  int32_t tiles_x[kMaxLevels], tiles_y[kMaxLevels];
  long long first_tile[kMaxLevels];  // in file order: the smallest level first
  unsigned long long level_at[kMaxLevels], level_pitch[kMaxLevels];  // levels 1..: offset and row pitch in cog_levels
  unsigned long long level_bytes;    // all of cog_levels
  long long n_tiles;
  int32_t tile, bpp;
  DeflateParams deflate;             // the stacked tiles: tile wide, n_tiles * tile high, strips of tile rows
  JpegParams jpeg;                   // ... or one JPEG image with a restart interval per tile
};

// The levels alone: AMB_OK or AMB_ERR_INVALID_ARGUMENT
int cog_levels(int32_t w, int32_t h, int32_t tile, CogPlan* p) {
  if (w <= 0 || h <= 0 || tile < 16 || tile > 4096 || tile % 16 != 0) return AMB_ERR_INVALID_ARGUMENT;
  p->tile = tile;
  p->n_levels = 1;
  p->w[0] = w;
  p->h[0] = h;
  for (int k = 0; p->w[k] > tile || p->h[k] > tile; ++k) {  // ceil(w / 2) without overflow; at most 28 levels
    p->w[k + 1] = p->w[k] / 2 + (p->w[k] & 1);
    p->h[k + 1] = p->h[k] / 2 + (p->h[k] & 1);
    ++p->n_levels;
  }
  return AMB_OK;
}

// The levels, their tiles and the scratch layout: AMB_OK, AMB_ERR_INVALID_ARGUMENT or AMB_ERR_UNSUPPORTED (more tile
// rows than an int32 counts)
int cog_grid(int32_t w, int32_t h, int format, int32_t tile, CogPlan* p) {
  int st = cog_levels(w, h, tile, p);
  if (st != AMB_OK) return st;
  if (format < AMB_RASTER_F32 || format > AMB_RASTER_MASK8) return AMB_ERR_INVALID_ARGUMENT;
  p->bpp = cog_bpp(format);
  long long n = 0;
  for (int k = p->n_levels - 1; k >= 0; --k) {
    p->tiles_x[k] = (p->w[k] - 1) / tile + 1;
    p->tiles_y[k] = (p->h[k] - 1) / tile + 1;
    p->first_tile[k] = n;
    n += static_cast<long long>(p->tiles_x[k]) * p->tiles_y[k];
  }
  p->n_tiles = n;
  if (n * tile > 0x7fffffffll) return AMB_ERR_UNSUPPORTED;
  unsigned long long at = 0;
  p->level_at[0] = p->level_pitch[0] = 0;
  for (int k = 1; k < p->n_levels; ++k) {
    p->level_pitch[k] = (static_cast<unsigned long long>(p->w[k]) * p->bpp + 15) & ~15ull;
    p->level_at[k] = at;
    at += (p->level_pitch[k] * p->h[k] + 255) & ~255ull;
  }
  p->level_bytes = at;
  return AMB_OK;
}

// AMB_OK, AMB_ERR_INVALID_ARGUMENT or AMB_ERR_UNSUPPORTED (more tile rows than an int32 counts, or what deflate_params
// cannot take)
int cog_plan(int32_t w, int32_t h, int format, int32_t tile, CogPlan* p) {
  const int st = cog_grid(w, h, format, tile, p);
  if (st != AMB_OK) return st;
  return deflate_params(tile, static_cast<int32_t>(p->n_tiles * tile), format, tile, &p->deflate);
}

// JPEG tiles of a GRAY8 or BGR8 raster: AMB_OK, AMB_ERR_INVALID_ARGUMENT (format, sizes, tile side) or
// AMB_ERR_UNSUPPORTED (quality, sampling, too many tile rows)
int cog_plan_jpeg(int32_t w, int32_t h, int format, int32_t tile, int quality, int sampling, CogPlan* p) {
  if (format != AMB_RASTER_GRAY8 && format != AMB_RASTER_BGR8) return AMB_ERR_INVALID_ARGUMENT;
  const int st = cog_grid(w, h, format, tile, p);
  if (st != AMB_OK) return st;
  return jpeg_tile_params(tile, p->n_tiles, format == AMB_RASTER_BGR8 ? 3 : 1, quality, sampling, &p->jpeg);
}

// 1-bit mask tiles of a MASK8 raster: the packed tiles T / 8 bytes wide, deflated without a predictor
int cog_plan_mask(int32_t w, int32_t h, int32_t tile, CogPlan* p) {
  const int st = cog_grid(w, h, AMB_RASTER_MASK8, tile, p);
  if (st != AMB_OK) return st;
  return deflate_params(tile / 8, static_cast<int32_t>(p->n_tiles * tile), AMB_RASTER_MASK8, tile, &p->deflate, false);
}

template <int FMT>
void launch_reduce(const unsigned char* src, unsigned long long src_stride, int32_t sw, int32_t sh, unsigned char* dst,
                   unsigned long long dst_stride, int32_t dw, int32_t dh, int grid_cap, cudaStream_t st) {
  constexpr int PX = FMT == AMB_RASTER_F32 ? 4 : 16;
  const long long pieces = (static_cast<long long>(dw) + PX - 1) / PX;
  const int threads = static_cast<int>(std::min<long long>(kReduceThreads, (pieces + 31) / 32 * 32));
  const int grid = std::min(dh, grid_cap);
  pyramid_reduce_kernel<FMT><<<grid, threads, 0, st>>>(src, src_stride, sw, sh, dst, dst_stride, dw, dh);
}

// The pyramid of the raster at d_img and its stacked tiles in ctx->cog_tiles (followed by `extra` bytes of scratch)
int cog_stack(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, int format, const CogPlan& p,
              size_t extra) {
  cudaStream_t st = ctx->stream;
  const int T = p.tile;
  const unsigned long long tile_row = static_cast<unsigned long long>(T) * p.bpp;
  AMB_CUDA(ctx, ctx->cog_levels.reserve(std::max<unsigned long long>(p.level_bytes, 1)));
  AMB_CUDA(ctx, ctx->cog_tiles.reserve(static_cast<size_t>(p.n_tiles) * T * tile_row + extra));
  unsigned char* levels = ctx->cog_levels.as<unsigned char>();
  uint4* tiles = ctx->cog_tiles.as<uint4>();
  const int cap = ctx->num_sms * 16;  // grid-stride launches: blocks per kernel
  for (int k = 0; k < p.n_levels; ++k) {
    const unsigned char* src = k == 0 ? d_img : levels + p.level_at[k];
    const unsigned long long stride = k == 0 ? row_stride : p.level_pitch[k];
    if (k > 0) {
      const unsigned char* up = k == 1 ? d_img : levels + p.level_at[k - 1];
      const unsigned long long up_stride = k == 1 ? row_stride : p.level_pitch[k - 1];
      unsigned char* dst = levels + p.level_at[k];
      switch (format) {
        case AMB_RASTER_F32:
          launch_reduce<AMB_RASTER_F32>(up, up_stride, p.w[k - 1], p.h[k - 1], dst, stride, p.w[k], p.h[k], cap, st);
          break;
        case AMB_RASTER_GRAY8:
          launch_reduce<AMB_RASTER_GRAY8>(up, up_stride, p.w[k - 1], p.h[k - 1], dst, stride, p.w[k], p.h[k], cap, st);
          break;
        case AMB_RASTER_BGR8:
          launch_reduce<AMB_RASTER_BGR8>(up, up_stride, p.w[k - 1], p.h[k - 1], dst, stride, p.w[k], p.h[k], cap, st);
          break;
        default:
          launch_reduce<AMB_RASTER_MASK8>(up, up_stride, p.w[k - 1], p.h[k - 1], dst, stride, p.w[k], p.h[k], cap, st);
          break;
      }
    }
    const int n = p.tiles_x[k] * p.tiles_y[k];
    pyramid_tile_kernel<<<std::min(n, cap), dim3(32, 8), 0, st>>>(
        src, stride, static_cast<unsigned long long>(p.w[k]) * p.bpp, p.h[k], T, static_cast<int32_t>(tile_row),
        p.tiles_x[k], n, tiles + p.first_tile[k] * T * (tile_row / 16));
  }
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

int cog_encode(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, int format, const CogPlan& p,
               void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes) {
  const int rc = cog_stack(ctx, d_img, row_stride, format, p, 0);
  if (rc != AMB_OK) return rc;
  return deflate_encode(ctx, ctx->cog_tiles.as<unsigned char>(), static_cast<size_t>(p.tile) * p.bpp, p.deflate,
                        host_out, capacity, size, tile_bytes);
}

int cog_encode_jpeg(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, int format, const CogPlan& p,
                    void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes) {
  const int rc = cog_stack(ctx, d_img, row_stride, format, p, 0);
  if (rc != AMB_OK) return rc;
  return jpeg_tiles_encode(ctx, ctx->cog_tiles.as<unsigned char>(), static_cast<size_t>(p.tile) * p.bpp, p.jpeg,
                           host_out, capacity, size, tile_bytes);
}

int cog_encode_mask(amb_ctx* ctx, const unsigned char* d_img, size_t row_stride, const CogPlan& p, void* host_out,
                    size_t capacity, size_t* size, uint32_t* tile_bytes) {
  const size_t stacked = static_cast<size_t>(p.n_tiles) * p.tile * p.tile;  // MASK8 bytes; the packed bits follow
  const int rc = cog_stack(ctx, d_img, row_stride, AMB_RASTER_MASK8, p, stacked / 8);
  if (rc != AMB_OK) return rc;
  const unsigned long long pieces = stacked / 16;
  unsigned char* packed = ctx->cog_tiles.as<unsigned char>() + stacked;
  const int grid = static_cast<int>(std::min<unsigned long long>((pieces + 255) / 256, ctx->num_sms * 16ull));
  mask_pack_kernel<<<grid, 256, 0, ctx->stream>>>(ctx->cog_tiles.as<uint4>(), pieces,
                                                  reinterpret_cast<uint16_t*>(packed));
  AMB_CUDA(ctx, cudaGetLastError());
  return deflate_encode(ctx, packed, static_cast<size_t>(p.tile / 8), p.deflate, host_out, capacity, size, tile_bytes);
}

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" {

int amb_cog_layout(int32_t width, int32_t height, int32_t tile, int32_t* n_levels, int32_t* level_w, int32_t* level_h) {
  if (!n_levels || !level_w || !level_h) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_levels(width, height, tile, &p);
  if (st != AMB_OK) return st;
  *n_levels = p.n_levels;
  for (int k = 0; k < p.n_levels; ++k) {
    level_w[k] = p.w[k];
    level_h[k] = p.h[k];
  }
  return AMB_OK;
}

size_t amb_cog_max_size(int32_t width, int32_t height, int format, int32_t tile) {
  CogPlan p;
  if (cog_plan(width, height, format, tile, &p) != AMB_OK) return 0;
  return static_cast<size_t>(p.deflate.bound);
}

int amb_cog_tiles_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride, int format,
                         int32_t tile, void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes) {
  if (!ctx || !d_image || !host_out || !size || !tile_bytes) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_plan(width, height, format, tile, &p);
  if (st != AMB_OK) return st;
  if (row_stride < static_cast<size_t>(width) * p.bpp) return AMB_ERR_INVALID_ARGUMENT;
  if (p.bpp == 4 && ((reinterpret_cast<uintptr_t>(d_image) & 3) || (row_stride & 3))) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return cog_encode(ctx, static_cast<const unsigned char*>(d_image), row_stride, format, p, host_out, capacity, size,
                    tile_bytes);
}

int amb_export_cog_tiles(amb_ctx* ctx, int layer, int format, int32_t tile, void* host_out, size_t capacity,
                         size_t* size, uint32_t* tile_bytes) {
  if (!ctx || !host_out || !size || !tile_bytes || layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_plan(ctx->geom.rows, ctx->col_end - ctx->col_begin, format, tile, &p);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t stride = static_cast<size_t>(ctx->geom.rows) * p.bpp;
  AMB_CUDA(ctx, ctx->raster_band.reserve(stride * static_cast<size_t>(ctx->col_end - ctx->col_begin)));
  const int rc = amb_export_raster_device(ctx, layer, format, ctx->raster_band.ptr);
  if (rc != AMB_OK) return rc;
  return cog_encode(ctx, ctx->raster_band.as<unsigned char>(), stride, format, p, host_out, capacity, size, tile_bytes);
}

size_t amb_cog_jpeg_max_size(int32_t width, int32_t height, int format, int32_t tile, int quality, int sampling) {
  CogPlan p;
  if (cog_plan_jpeg(width, height, format, tile, quality, sampling, &p) != AMB_OK) return 0;
  return static_cast<size_t>(jpeg_tiles_bound(p.jpeg));
}

int amb_cog_jpeg_tables(int channels, int quality, void* out, size_t capacity, size_t* size) {
  if (!out || !size) return AMB_ERR_INVALID_ARGUMENT;
  if ((channels != 1 && channels != 3) || quality < 1 || quality > 100) return AMB_ERR_UNSUPPORTED;
  const std::vector<unsigned char> t = jpeg_tables_stream(channels, quality);
  *size = t.size();
  if (capacity < t.size()) return AMB_ERR_SIZE_MISMATCH;
  std::copy(t.begin(), t.end(), static_cast<unsigned char*>(out));
  return AMB_OK;
}

int amb_cog_jpeg_tiles_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                              int format, int32_t tile, int quality, int sampling, void* host_out, size_t capacity,
                              size_t* size, uint32_t* tile_bytes) {
  if (!ctx || !d_image || !host_out || !size || !tile_bytes) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_plan_jpeg(width, height, format, tile, quality, sampling, &p);
  if (st != AMB_OK) return st;
  if (row_stride < static_cast<size_t>(width) * p.bpp) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return cog_encode_jpeg(ctx, static_cast<const unsigned char*>(d_image), row_stride, format, p, host_out, capacity,
                         size, tile_bytes);
}

int amb_export_cog_jpeg_tiles(amb_ctx* ctx, int layer, int format, int32_t tile, int quality, int sampling,
                              void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes) {
  if (!ctx || !host_out || !size || !tile_bytes || layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_plan_jpeg(ctx->geom.rows, ctx->col_end - ctx->col_begin, format, tile, quality, sampling, &p);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t stride = static_cast<size_t>(ctx->geom.rows) * p.bpp;
  AMB_CUDA(ctx, ctx->raster_band.reserve(stride * static_cast<size_t>(ctx->col_end - ctx->col_begin)));
  const int rc = amb_export_raster_device(ctx, layer, format, ctx->raster_band.ptr);
  if (rc != AMB_OK) return rc;
  return cog_encode_jpeg(ctx, ctx->raster_band.as<unsigned char>(), stride, format, p, host_out, capacity, size,
                         tile_bytes);
}

size_t amb_cog_mask_max_size(int32_t width, int32_t height, int32_t tile) {
  CogPlan p;
  if (cog_plan_mask(width, height, tile, &p) != AMB_OK) return 0;
  return static_cast<size_t>(p.deflate.bound);
}

int amb_cog_mask_tiles_device(amb_ctx* ctx, const void* d_mask, int32_t width, int32_t height, size_t row_stride,
                              int32_t tile, void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes) {
  if (!ctx || !d_mask || !host_out || !size || !tile_bytes) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_plan_mask(width, height, tile, &p);
  if (st != AMB_OK) return st;
  if (row_stride < static_cast<size_t>(width)) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return cog_encode_mask(ctx, static_cast<const unsigned char*>(d_mask), row_stride, p, host_out, capacity, size,
                         tile_bytes);
}

int amb_export_cog_mask_tiles(amb_ctx* ctx, int layer, int32_t tile, void* host_out, size_t capacity, size_t* size,
                              uint32_t* tile_bytes) {
  if (!ctx || !host_out || !size || !tile_bytes || layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  CogPlan p;
  const int st = cog_plan_mask(ctx->geom.rows, ctx->col_end - ctx->col_begin, tile, &p);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t stride = static_cast<size_t>(ctx->geom.rows);
  AMB_CUDA(ctx, ctx->raster_band.reserve(stride * static_cast<size_t>(ctx->col_end - ctx->col_begin)));
  const int rc = amb_export_raster_device(ctx, layer, AMB_RASTER_MASK8, ctx->raster_band.ptr);
  if (rc != AMB_OK) return rc;
  return cog_encode_mask(ctx, ctx->raster_band.as<unsigned char>(), stride, p, host_out, capacity, size, tile_bytes);
}

}  // extern "C"
