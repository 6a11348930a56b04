// raster_export.cu — a layer slab as a north-up, row-major raster band ("next" row N4; convention in
// include/aerial_mapper_b200.h): pixel (r, c) of the band is cell (rows - 1 - c, r) of the slab, converted to one of the
// amb_raster_format pixel formats.
//
// Output pixel p = r * rows + c reads slab element r * rows + (rows - 1 - c): each image row is one layer column read
// backwards.  The kernel walks the OUTPUT in tiles of 256 pieces of W bytes (16, or 48 for BGR8), tile starts 16-byte
// aligned in the destination:
//   load   consecutive threads take consecutive pixels of the tile (coalesced reversed loads), convert them and put their
//          bytes into a shared-memory image of the tile — any byte offset, so a destination that is not a multiple of the
//          pixel size needs no special case
//   store  every thread writes its piece with 16-byte stores; the pieces that the band's first bytes (up to the first
//          16-byte boundary of the destination) and its last bytes cut are written byte by byte
// 32-bit cell indices: a slab holds fewer than 2^32 cells (amb_create).
#include <cmath>

#include "amb_context.h"

namespace amb {
namespace {

constexpr int kRasterThreads = 256;

// floor(n / d) for 32-bit n by one 64 x 32-bit multiply-high (m = ceil(2^64 / d), exact for every 32-bit n and d >= 2;
// Lemire, Kaser & Kurz 2019); m = 0 stands for d = 1
struct RowDiv {
  uint64_t m;
  __device__ __forceinline__ uint32_t div(uint32_t n) const {
    if (m == 0) return n;
    const uint64_t lo = (m & 0xffffffffull) * n;
    const uint64_t hi = (m >> 32) * n + (lo >> 32);
    return static_cast<uint32_t>(hi >> 32);
  }
};

__host__ __device__ constexpr int raster_bpp(int fmt) { return fmt == AMB_RASTER_F32 ? 4 : fmt == AMB_RASTER_BGR8 ? 3 : 1; }

__device__ __forceinline__ bool is_nan_bits(uint32_t bits) { return (bits & 0x7fffffffu) > 0x7f800000u; }

// OpenCV saturate_cast<uchar>(float): cvRound (round half to even; NaN and anything outside int32 give INT_MIN), then
// clamp to [0, 255]
__device__ __forceinline__ uint32_t gray8(float v) {
  if (!(v < 2147483648.0f)) return 0u;  // NaN, +inf, >= 2^31
  const float r = rintf(v);
  return r >= 255.0f ? 255u : r > 0.0f ? static_cast<uint32_t>(r) : 0u;
}

// bytes of one pixel into the shared tile at byte offset o (parts outside [0, TW) belong to a neighbouring tile)
template <int FMT, int TW>
__device__ __forceinline__ void put_pixel(unsigned char* tile, long long o, uint32_t bits) {
  if (FMT == AMB_RASTER_F32) {
    if ((o & 3) == 0 && o >= 0 && o + 4 <= TW) {
      *reinterpret_cast<uint32_t*>(tile + o) = bits;
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (o + q >= 0 && o + q < TW) tile[o + q] = static_cast<unsigned char>(bits >> (8 * q));
    }
  } else if (FMT == AMB_RASTER_BGR8) {
    const uint32_t v = is_nan_bits(bits) ? 0u : bits;  // 0x00RRGGBB -> B, G, R
#pragma unroll
    for (int q = 0; q < 3; ++q)
      if (o + q >= 0 && o + q < TW) tile[o + q] = static_cast<unsigned char>(v >> (8 * q));
  } else if (o >= 0 && o < TW) {
    tile[o] = static_cast<unsigned char>(FMT == AMB_RASTER_GRAY8 ? gray8(__uint_as_float(bits))
                                                                : (is_nan_bits(bits) ? 0u : 255u));
  }
}

// Tiles k = 0 .. n_tiles-1 cover band bytes [base + k * TW, base + (k + 1) * TW) clipped to [0, total); base is chosen so
// that dst + base is 16-byte aligned.
template <int FMT>
__global__ void __launch_bounds__(kRasterThreads)
    raster_export_kernel(const float* __restrict__ layer, uint32_t rows, RowDiv rdiv, unsigned char* __restrict__ dst,
                         long long base, unsigned long long total, unsigned long long n_tiles) {
  constexpr int BPP = raster_bpp(FMT);
  constexpr int W = FMT == AMB_RASTER_BGR8 ? 48 : 16;    // bytes per thread: a whole number of pixels and of 16-byte stores
  constexpr int TW = kRasterThreads * W;
  constexpr int MAXM = (TW / BPP + 2 + kRasterThreads - 1) / kRasterThreads;  // pixels per thread, cut pixels included
  __shared__ __align__(16) unsigned char tile[TW];
  for (unsigned long long k = blockIdx.x; k < n_tiles; k += gridDim.x) {
    const long long b0 = base + static_cast<long long>(k) * TW;
    const unsigned long long lo = b0 < 0 ? 0ull : static_cast<unsigned long long>(b0);
    const unsigned long long hi = static_cast<unsigned long long>(b0 + TW) < total ? static_cast<unsigned long long>(b0 + TW) : total;
    const uint32_t p_lo = static_cast<uint32_t>(lo / BPP);
    const uint32_t n_pix = static_cast<uint32_t>((hi - 1) / BPP + 1 - p_lo);
    uint32_t bits[MAXM];  // all loads of the tile in flight before the first conversion
#pragma unroll
    for (int m = 0; m < MAXM; ++m) {
      const uint32_t t = threadIdx.x + m * kRasterThreads;
      bits[m] = 0u;
      if (t < n_pix) {
        const uint32_t p = p_lo + t;
        const uint32_t r = rdiv.div(p), c = p - r * rows;
        bits[m] = __float_as_uint(__ldg(layer + (r * rows + (rows - 1u - c))));
      }
    }
#pragma unroll
    for (int m = 0; m < MAXM; ++m) {
      const uint32_t t = threadIdx.x + m * kRasterThreads;
      if (t < n_pix) put_pixel<FMT, TW>(tile, static_cast<long long>(p_lo + t) * BPP - b0, bits[m]);
    }
    __syncthreads();
    const long long s = b0 + static_cast<long long>(threadIdx.x) * W;  // this thread's piece of the band
    const unsigned char* src = tile + threadIdx.x * W;
    if (s >= static_cast<long long>(lo) && static_cast<unsigned long long>(s + W) <= hi) {
#pragma unroll
      for (int q = 0; q < W / 16; ++q)
        reinterpret_cast<uint4*>(dst + s)[q] = reinterpret_cast<const uint4*>(src)[q];
    } else {
      for (int q = 0; q < W; ++q)
        if (s + q >= static_cast<long long>(lo) && static_cast<unsigned long long>(s + q) < hi) dst[s + q] = src[q];
    }
    __syncthreads();  // the tile is refilled by the next iteration
  }
}

bool raster_args_ok(int layer, int format) {
  return layer >= 0 && layer < AMB_NUM_LAYERS && format >= AMB_RASTER_F32 && format <= AMB_RASTER_MASK8;
}

// Enqueue the export of the slab of `layer` into device memory `dst` on the context's stream.
int export_raster_enqueue(amb_ctx* ctx, int layer, int format, unsigned char* dst) {
  int st = ensure_layer(ctx, layer);
  if (st != AMB_OK) return st;
  const uint32_t rows = static_cast<uint32_t>(ctx->geom.rows);
  const unsigned long long total = static_cast<unsigned long long>(ctx->slab_cells()) * raster_bpp(format);
  const int tw = kRasterThreads * (format == AMB_RASTER_BGR8 ? 48 : 16);
  const long long head =
      std::min<long long>((16 - static_cast<long long>(reinterpret_cast<uintptr_t>(dst) & 15)) & 15, total);
  const long long base = head > 0 ? head - tw : 0;
  const unsigned long long n_tiles = (total - base + tw - 1) / tw;
  const RowDiv rdiv{rows > 1 ? ~0ull / rows + 1 : 0ull};
  const int grid = static_cast<int>(std::min<unsigned long long>(n_tiles, static_cast<unsigned long long>(ctx->num_sms) * 8));
  const float* src = ctx->layers[layer];
  switch (format) {
    case AMB_RASTER_F32:
      raster_export_kernel<AMB_RASTER_F32><<<grid, kRasterThreads, 0, ctx->stream>>>(src, rows, rdiv, dst, base, total, n_tiles);
      break;
    case AMB_RASTER_GRAY8:
      raster_export_kernel<AMB_RASTER_GRAY8><<<grid, kRasterThreads, 0, ctx->stream>>>(src, rows, rdiv, dst, base, total, n_tiles);
      break;
    case AMB_RASTER_BGR8:
      raster_export_kernel<AMB_RASTER_BGR8><<<grid, kRasterThreads, 0, ctx->stream>>>(src, rows, rdiv, dst, base, total, n_tiles);
      break;
    default:
      raster_export_kernel<AMB_RASTER_MASK8><<<grid, kRasterThreads, 0, ctx->stream>>>(src, rows, rdiv, dst, base, total, n_tiles);
      break;
  }
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" {

int amb_raster_geotransform(const amb_geometry* g, double gt[6]) {
  if (!g || !gt || g->rows <= 0 || g->cols <= 0 || !(g->resolution > 0.0)) return AMB_ERR_INVALID_ARGUMENT;
  gt[0] = g->pos_x - 0.5 * g->length_x;  // west edge: column c = 0 is cell row i = rows - 1
  gt[1] = g->resolution;
  gt[2] = 0.0;
  gt[3] = g->pos_y + 0.5 * g->length_y;  // north edge: image row r = 0 is cell column j = 0
  gt[4] = 0.0;
  gt[5] = -g->resolution;
  return AMB_OK;
}

int amb_export_raster_device(amb_ctx* ctx, int layer, int format, void* device_band) {
  if (!ctx || !device_band || !raster_args_ok(layer, format)) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return export_raster_enqueue(ctx, layer, format, static_cast<unsigned char*>(device_band));
}

int amb_export_raster(amb_ctx* ctx, int layer, int format, void* host_band) {
  if (!ctx || !host_band || !raster_args_ok(layer, format)) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t bytes = ctx->slab_cells() * static_cast<size_t>(raster_bpp(format));
  AMB_CUDA(ctx, ctx->raster_band.reserve(bytes));
  const int st = export_raster_enqueue(ctx, layer, format, ctx->raster_band.as<unsigned char>());
  if (st != AMB_OK) return st;
  return staged_d2h(ctx, host_band, ctx->raster_band.ptr, bytes, ctx->stream);
}

}  // extern "C"
