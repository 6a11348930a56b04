// raster_import.cu — a north-up float32 raster resampled into a layer slab (convention in include/aerial_mapper_b200.h,
// amb_resample): the inverse of raster_export.cu, with nearest or bilinear resampling when the grids differ.
//
// The map-to-raster mapping is separable: x depends on the cell row i only, y on the column j only.  The host computes
// one table per axis in IEEE double (source index, fraction of the next index, -1 where uncovered) and the window of
// raster rows and columns they reference; the kernel does no division, only the blend:
//   threads run along i (the slab's contiguous axis: coalesced stores), each thread reads its i entry once and walks
//   kImportCols columns, issuing every load of those columns before the first store.  In the aligned case cell i + 1
//   reads raster column c - 1: contiguous, reversed loads.
// The blend is double, every operation rounded (__dmul_rn / __dadd_rn), so the result does not depend on contraction;
// a tap of weight 0 is never read, and untouched cells issue no store.
#include <algorithm>
#include <cmath>
#include <vector>

#include "amb_context.h"

namespace amb {
namespace {

constexpr int kImportThreads = 256;
constexpr int kImportCols = 8;        // columns per thread
constexpr double kSnap = 0x1p-20;     // fractions closer than this to 0 or 1 snap to the pixel

// one axis entry: source column (i table) or row (j table), -1 where the cell is outside the raster, and the weight of
// the next source index (0 for NEAREST and for snapped fractions)
struct ImportTap {
  double f;
  int32_t k;
  int32_t pad;
};

__device__ __forceinline__ bool no_data(float v, int has_nodata, float nodata) {
  return v != v || (has_nodata && v == nodata);
}

// (1 - f) a + f b with f != 0, g = 1 - f
__device__ __forceinline__ double lerp_rn(double g, double f, double a, double b) {
  return __dadd_rn(__dmul_rn(g, a), __dmul_rn(f, b));
}

// band: row r at band + r * stride (floats); slab: rows x ncols, column-major; tables: itab[rows], jtab[ncols].  Block b
// covers rows [256 (b % row_blocks), + 256) and columns [kImportCols (b / row_blocks), + kImportCols) (a 1-D grid: at most
// rows * ncols / 2048 < 2^21 blocks)
template <int RESAMPLE>
__global__ void __launch_bounds__(kImportThreads)
    raster_import_kernel(const float* __restrict__ band, long long stride, const ImportTap* __restrict__ itab,
                         const ImportTap* __restrict__ jtab, uint32_t rows, uint32_t ncols, uint32_t row_blocks,
                         float* __restrict__ layer, int has_nodata, float nodata) {
  const uint32_t i = (blockIdx.x % row_blocks) * kImportThreads + threadIdx.x;
  const uint32_t j0 = (blockIdx.x / row_blocks) * kImportCols;
  if (i >= rows) return;
  const int32_t c = __ldg(&itab[i].k);
  if (c < 0) return;
  const double fx = __ldg(&itab[i].f);
  const double gx = __dadd_rn(1.0, -fx);
  if (RESAMPLE == AMB_RESAMPLE_NEAREST) {
    float v[kImportCols];
    bool ok[kImportCols];
#pragma unroll
    for (int q = 0; q < kImportCols; ++q) {
      const uint32_t j = j0 + q;
      const int32_t r = j < ncols ? __ldg(&jtab[j].k) : -1;
      ok[q] = r >= 0;
      v[q] = ok[q] ? __ldg(band + (static_cast<long long>(r) * stride + c)) : 0.0f;
    }
#pragma unroll
    for (int q = 0; q < kImportCols; ++q)
      if (ok[q] && !no_data(v[q], has_nodata, nodata)) layer[static_cast<size_t>(j0 + q) * rows + i] = v[q];
  } else {
    float p[kImportCols][4];  // taps (r0, c0), (r0, c0 + 1), (r0 + 1, c0), (r0 + 1, c0 + 1); weight 0: not read
    double fy[kImportCols];
    bool ok[kImportCols];
#pragma unroll
    for (int q = 0; q < kImportCols; ++q) {
      const uint32_t j = j0 + q;
      const int32_t r = j < ncols ? __ldg(&jtab[j].k) : -1;
      ok[q] = r >= 0;
      fy[q] = ok[q] ? __ldg(&jtab[j].f) : 0.0;
      const float* a = band + (static_cast<long long>(ok[q] ? r : 0) * stride + c);
      p[q][0] = ok[q] ? __ldg(a) : 0.0f;
      p[q][1] = ok[q] && fx != 0.0 ? __ldg(a + 1) : 0.0f;
      p[q][2] = ok[q] && fy[q] != 0.0 ? __ldg(a + stride) : 0.0f;
      p[q][3] = ok[q] && fx != 0.0 && fy[q] != 0.0 ? __ldg(a + stride + 1) : 0.0f;
    }
#pragma unroll
    for (int q = 0; q < kImportCols; ++q) {
      if (!ok[q]) continue;
      const bool wx = fx != 0.0, wy = fy[q] != 0.0;
      if (no_data(p[q][0], has_nodata, nodata) || (wx && no_data(p[q][1], has_nodata, nodata)) ||
          (wy && (no_data(p[q][2], has_nodata, nodata) || (wx && no_data(p[q][3], has_nodata, nodata)))))
        continue;
      double h = wx ? lerp_rn(gx, fx, p[q][0], p[q][1]) : static_cast<double>(p[q][0]);
      if (wy) {
        const double h1 = wx ? lerp_rn(gx, fx, p[q][2], p[q][3]) : static_cast<double>(p[q][2]);
        h = lerp_rn(__dadd_rn(1.0, -fy[q]), fy[q], h, h1);
      }
      layer[static_cast<size_t>(j0 + q) * rows + i] = __double2float_rn(h);
    }
  }
}

bool gt_ok(const double* gt) {
  if (!gt) return false;
  for (int k = 0; k < 6; ++k)
    if (!std::isfinite(gt[k])) return false;
  return gt[2] == 0.0 && gt[4] == 0.0 && gt[1] > 0.0 && gt[5] < 0.0;
}

bool import_args_ok(int layer, int32_t width, int32_t height, size_t row_stride, const double* gt, int resample) {
  return layer >= 0 && layer < AMB_NUM_LAYERS && width > 0 && height > 0 && row_stride % 4 == 0 &&
         row_stride >= 4 * static_cast<size_t>(width) && gt_ok(gt) &&
         (resample == AMB_RESAMPLE_NEAREST || resample == AMB_RESAMPLE_BILINEAR);
}

// position q along one axis of a raster of n pixels with origin o and step d
ImportTap axis_tap(double q, double o, double d, int32_t n, int resample) {
  ImportTap t{0.0, -1, 0};
  const double u = (q - o) / d;
  if (!(u >= 0.0 && u < static_cast<double>(n))) return t;
  if (resample == AMB_RESAMPLE_NEAREST) {
    t.k = static_cast<int32_t>(std::floor(u));
    return t;
  }
  const double s = std::min(std::max(u - 0.5, 0.0), static_cast<double>(n - 1));
  double k = std::floor(s);
  double f = s - k;
  if (f < kSnap) {
    f = 0.0;
  } else if (f > 1.0 - kSnap) {
    k += 1.0;
    f = 0.0;
  }
  t.k = static_cast<int32_t>(k);
  t.f = f;
  return t;
}

// taps[0, rows): the i table; taps[rows, rows + n): the j table of columns [col_begin, col_end).  The positions are
// amb_geometry_position's own, so they are the cells' positions bit for bit.
void import_tables(const amb_geometry& g, int32_t col_begin, int32_t col_end, int32_t width, int32_t height,
                   const double* gt, int resample, std::vector<ImportTap>* taps) {
  taps->resize(static_cast<size_t>(g.rows) + static_cast<size_t>(col_end - col_begin));
  double x, y;
  for (int32_t i = 0; i < g.rows; ++i) {
    amb_geometry_position(&g, i, col_begin, &x, &y);
    (*taps)[i] = axis_tap(x, gt[0], gt[1], width, resample);
  }
  for (int32_t j = col_begin; j < col_end; ++j) {
    amb_geometry_position(&g, 0, j, &x, &y);
    (*taps)[static_cast<size_t>(g.rows) + (j - col_begin)] = axis_tap(y, gt[3], gt[5], height, resample);
  }
}

// [lo, hi] of the source indices an axis table reads (a fraction > 0 reads k + 1 too); false if nothing is covered
bool axis_window(const ImportTap* t, size_t n, int32_t* lo, int32_t* hi) {
  *lo = INT32_MAX;
  *hi = -1;
  for (size_t k = 0; k < n; ++k)
    if (t[k].k >= 0) {
      *lo = std::min(*lo, t[k].k);
      *hi = std::max(*hi, t[k].k + (t[k].f != 0.0 ? 1 : 0));
    }
  return *hi >= 0;
}

// The stripe's tables for a width x height raster and the window of raster columns [c_lo, c_hi] and rows [r_lo, r_hi]
// they read, the tables rebased to the window's corner; false if the raster does not overlap the stripe
bool import_window(const amb_ctx* ctx, int32_t width, int32_t height, const double* gt, int resample,
                   std::vector<ImportTap>* taps, int32_t* c_lo, int32_t* c_hi, int32_t* r_lo, int32_t* r_hi) {
  import_tables(ctx->geom, ctx->col_begin, ctx->col_end, width, height, gt, resample, taps);
  const size_t rows = static_cast<size_t>(ctx->geom.rows);
  if (!axis_window(taps->data(), rows, c_lo, c_hi) || !axis_window(taps->data() + rows, taps->size() - rows, r_lo, r_hi))
    return false;
  for (size_t k = 0; k < taps->size(); ++k)
    if ((*taps)[k].k >= 0) (*taps)[k].k -= k < rows ? *c_lo : *r_lo;
  return true;
}

// Enqueue the tables' upload and the kernel on the context's stream; band rows are `stride` floats apart.
int import_enqueue(amb_ctx* ctx, int layer, const float* band, long long stride, const std::vector<ImportTap>& taps,
                   int has_nodata, float nodata, int resample) {
  int st = ensure_layer(ctx, layer);
  if (st != AMB_OK) return st;
  wait_layer_copy(ctx, layer);
  // the tables travel through the context's pinned per-call staging (see HostStage), so back-to-back asynchronous
  // imports do not wait for the driver's pageable staging
  const size_t bytes = taps.size() * sizeof(ImportTap);
  const int turn = static_cast<int>(ctx->stage_turn++ & 1u);
  HostStage& stage = ctx->stages[turn];
  cudaEvent_t& stage_event = ctx->stage_events[turn];
  if (!stage_event) AMB_CUDA(ctx, cudaEventCreateWithFlags(&stage_event, cudaEventDisableTiming));
  AMB_CUDA(ctx, cudaEventSynchronize(stage_event));
  AMB_CUDA(ctx, stage.reserve(bytes + 64));
  stage.used = 0;
  ImportTap* staged = stage.take<ImportTap>(taps.size());
  std::memcpy(staged, taps.data(), bytes);
  AMB_CUDA(ctx, ctx->raster_taps.reserve(bytes));
  AMB_CUDA(ctx, cudaMemcpyAsync(ctx->raster_taps.ptr, staged, bytes, cudaMemcpyHostToDevice, ctx->stream));
  AMB_CUDA(ctx, cudaEventRecord(stage_event, ctx->stream));
  const uint32_t rows = static_cast<uint32_t>(ctx->geom.rows);
  const uint32_t ncols = static_cast<uint32_t>(ctx->col_end - ctx->col_begin);
  const ImportTap* itab = ctx->raster_taps.as<ImportTap>();
  const uint32_t row_blocks = (rows + kImportThreads - 1) / kImportThreads;
  const uint32_t grid = row_blocks * ((ncols + kImportCols - 1) / kImportCols);
  if (resample == AMB_RESAMPLE_NEAREST)
    raster_import_kernel<AMB_RESAMPLE_NEAREST><<<grid, kImportThreads, 0, ctx->stream>>>(
        band, stride, itab, itab + rows, rows, ncols, row_blocks, ctx->layers[layer], has_nodata, nodata);
  else
    raster_import_kernel<AMB_RESAMPLE_BILINEAR><<<grid, kImportThreads, 0, ctx->stream>>>(
        band, stride, itab, itab + rows, rows, ncols, row_blocks, ctx->layers[layer], has_nodata, nodata);
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" {

int amb_raster_import_tables(const amb_geometry* geom, int32_t col_begin, int32_t col_end, int32_t width,
                             int32_t height, const double gt[6], int resample, int32_t* src_col, double* fx,
                             int32_t* src_row, double* fy) {
  if (!geom || !src_col || !fx || !src_row || !fy || geom->rows <= 0 || geom->cols <= 0 ||
      !(geom->resolution > 0.0) || col_begin < 0 || col_end > geom->cols || col_begin >= col_end ||
      !import_args_ok(0, width, height, 4 * static_cast<size_t>(width), gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  std::vector<ImportTap> taps;
  import_tables(*geom, col_begin, col_end, width, height, gt, resample, &taps);
  for (int32_t i = 0; i < geom->rows; ++i) {
    src_col[i] = taps[i].k;
    fx[i] = taps[i].f;
  }
  for (int32_t k = 0; k < col_end - col_begin; ++k) {
    src_row[k] = taps[static_cast<size_t>(geom->rows) + k].k;
    fy[k] = taps[static_cast<size_t>(geom->rows) + k].f;
  }
  return AMB_OK;
}

int amb_import_raster_device(amb_ctx* ctx, int layer, const float* device_band, int32_t width, int32_t height,
                             size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample) {
  if (!ctx || !device_band || (reinterpret_cast<uintptr_t>(device_band) & 3) != 0 ||
      !import_args_ok(layer, width, height, row_stride, gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<ImportTap> taps;
  import_tables(ctx->geom, ctx->col_begin, ctx->col_end, width, height, gt, resample, &taps);
  int32_t c_lo, c_hi, r_lo, r_hi;
  const size_t rows = static_cast<size_t>(ctx->geom.rows);
  if (!axis_window(taps.data(), rows, &c_lo, &c_hi) ||
      !axis_window(taps.data() + rows, taps.size() - rows, &r_lo, &r_hi))
    return AMB_OK;  // no overlap with the stripe
  return import_enqueue(ctx, layer, device_band, static_cast<long long>(row_stride / 4), taps, has_nodata, nodata,
                        resample);
}

int amb_import_raster(amb_ctx* ctx, int layer, const float* host_band, int32_t width, int32_t height,
                      size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample) {
  if (!ctx || !host_band || !import_args_ok(layer, width, height, row_stride, gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<ImportTap> taps;
  int32_t c_lo, c_hi, r_lo, r_hi;
  if (!import_window(ctx, width, height, gt, resample, &taps, &c_lo, &c_hi, &r_lo, &r_hi))
    return AMB_OK;  // no overlap with the stripe
  // only the window crosses PCIe, packed: the tables index it from its corner
  const size_t win_w = static_cast<size_t>(c_hi - c_lo + 1), win_h = static_cast<size_t>(r_hi - r_lo + 1);
  AMB_CUDA(ctx, ctx->raster_band.reserve(win_w * win_h * sizeof(float)));
  const StagedRect rect{ctx->raster_band.as<unsigned char>(), win_w * sizeof(float),
                        reinterpret_cast<const unsigned char*>(host_band) + static_cast<size_t>(r_lo) * row_stride +
                            static_cast<size_t>(c_lo) * sizeof(float),
                        row_stride, win_w * sizeof(float), win_h};
  int st = staged_h2d_rects(ctx, &rect, 1, ctx->stream);
  if (st != AMB_OK) return st;
  st = import_enqueue(ctx, layer, ctx->raster_band.as<float>(), static_cast<long long>(win_w), taps, has_nodata, nodata,
                      resample);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the caller's band (pinned: read by the DMA) may be reused
  return AMB_OK;
}

int amb_import_tiff(amb_ctx* ctx, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                    const double gt[6], int has_nodata, float nodata, int resample) {
  if (!ctx || !file || tiff_layout_check(layout, bytes) != AMB_OK ||
      !import_args_ok(layer, layout->width, layout->height, 4 * static_cast<size_t>(layout->width), gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<ImportTap> taps;
  int32_t c_lo, c_hi, r_lo, r_hi;
  if (!import_window(ctx, layout->width, layout->height, gt, resample, &taps, &c_lo, &c_hi, &r_lo, &r_hi))
    return AMB_OK;  // no overlap with the stripe
  // only the window's chunks are copied and decoded, into the window band the tables index from its corner
  const size_t win_w = static_cast<size_t>(c_hi - c_lo + 1), win_h = static_cast<size_t>(r_hi - r_lo + 1);
  AMB_CUDA(ctx, ctx->raster_band.reserve(win_w * win_h * sizeof(float)));
  int st = tiff_decode_window(ctx, static_cast<const unsigned char*>(file), *layout, r_lo, r_hi + 1, c_lo, c_hi + 1,
                              ctx->raster_band.as<float>(), win_w);
  if (st != AMB_OK) return st;
  st = import_enqueue(ctx, layer, ctx->raster_band.as<float>(), static_cast<long long>(win_w), taps, has_nodata, nodata,
                      resample);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return AMB_OK;
}

}  // extern "C"
