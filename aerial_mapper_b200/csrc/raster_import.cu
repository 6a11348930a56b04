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
// Longitude/latitude rasters into UTM maps (amb_import_*_lonlat, below) are not separable: the same block shape, but
// every cell inverse-projects its own position and takes its taps with the same axis_tap and blend.
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

// The bilinear blend of taps p = (r0, c0), (r0, c0 + 1), (r0 + 1, c0), (r0 + 1, c0 + 1), of which only those of non-zero
// weight were read (gx = 1 - fx); false, and *h unset, if a tap it reads is no-data
__device__ __forceinline__ bool blend(const float p[4], double fx, double gx, double fy, int has_nodata, float nodata,
                                      float* h) {
  const bool wx = fx != 0.0, wy = fy != 0.0;
  if (no_data(p[0], has_nodata, nodata) || (wx && no_data(p[1], has_nodata, nodata)) ||
      (wy && (no_data(p[2], has_nodata, nodata) || (wx && no_data(p[3], has_nodata, nodata)))))
    return false;
  double v = wx ? lerp_rn(gx, fx, p[0], p[1]) : static_cast<double>(p[0]);
  if (wy) {
    const double v1 = wx ? lerp_rn(gx, fx, p[2], p[3]) : static_cast<double>(p[2]);
    v = lerp_rn(__dadd_rn(1.0, -fy), fy, v, v1);
  }
  *h = __double2float_rn(v);
  return true;
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
      float h;
      if (ok[q] && blend(p[q], fx, gx, fy[q], has_nodata, nodata, &h)) layer[static_cast<size_t>(j0 + q) * rows + i] = h;
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

// position q along one axis of a raster of n pixels with origin o and step d: the host's per-axis tables and the
// longitude/latitude kernel's per-cell taps (one IEEE subtraction, one IEEE division: nothing to contract)
__host__ __device__ inline ImportTap axis_tap(double q, double o, double d, int32_t n, int resample) {
  ImportTap t{0.0, -1, 0};
  const double u = (q - o) / d;
  if (!(u >= 0.0 && u < static_cast<double>(n))) return t;
  if (resample == AMB_RESAMPLE_NEAREST) {
    t.k = static_cast<int32_t>(floor(u));
    return t;
  }
  double s = u - 0.5;  // min(max(u - 0.5, 0), n - 1)
  s = s < 0.0 ? 0.0 : s;
  s = static_cast<double>(n - 1) < s ? static_cast<double>(n - 1) : s;
  double k = floor(s);
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

// ---- longitude/latitude rasters into UTM maps (amb_import_raster_lonlat*) ----
// Inverse transverse Mercator as Krüger's series of order 6 in n (Karney 2011, eqs 11, 15, 36):
//   xi = (N - FN) / (k0 A),  eta = (E - FE) / (k0 A)
//   xi' = xi - sum_k beta_k sin(2k xi) cosh(2k eta),  eta' = eta - sum_k beta_k cos(2k xi) sinh(2k eta)
//   lambda = lambda0 + atan2(sinh eta', cos xi'),  tan(chi) = sin xi' / hypot(sinh eta', cos xi')  (conformal latitude)
// and the geodetic latitude from tan(chi) by two Newton steps on tau = tan(phi) (Karney 2011, eqs 7-9, 19-21).  eta depends
// on the cell row i only (easting), xi on the column j only (northing): a prologue kernel tabulates both axes' harmonics,
// and a cell costs two 6-term dot products plus the non-separable part.
constexpr int kTmOrder = 6;
constexpr double kRadToDeg = 57.295779513082320876798154814105;  // 180 / pi

// i table (row i): eta, beta_k cosh(2k eta), beta_k sinh(2k eta); j table (column j): xi, sin(2k xi), cos(2k xi)
struct TmAxis {
  double v;
  double a[kTmOrder];
  double b[kTmOrder];
};

struct TmParams {
  double lon0;   // central meridian, degrees
  double fn;     // false northing
  double k0A;    // k0 * rectifying radius
  double e, e2m; // eccentricity, 1 - e^2
  double beta[kTmOrder];
};

// WGS84 UTM zone of an EPSG code (32601-32660 north, 32701-32760 south); false for any other code
bool tm_params(int32_t epsg, TmParams* p) {
  const bool north = epsg >= 32601 && epsg <= 32660, south = epsg >= 32701 && epsg <= 32760;
  if (!north && !south) return false;
  const int zone = epsg % 100;
  const double f = 1.0 / 298.257223563, n = f / (2.0 - f), e2 = f * (2.0 - f);
  p->lon0 = 6.0 * zone - 183.0;
  p->fn = south ? 10000000.0 : 0.0;
  const double n2 = n * n;
  p->k0A = 0.9996 * 6378137.0 / (1.0 + n) * (1.0 + n2 * (1.0 / 4.0 + n2 * (1.0 / 64.0 + n2 * (1.0 / 256.0))));
  p->e = std::sqrt(e2);
  p->e2m = 1.0 - e2;
  // Karney 2011, eq 36: beta_k as polynomials in n (Horner from n^6 down to the lowest power)
  static const double c[kTmOrder][kTmOrder] = {
      {1.0 / 2, -2.0 / 3, 37.0 / 96, -1.0 / 360, -81.0 / 512, 96199.0 / 604800},
      {0, 1.0 / 48, 1.0 / 15, -437.0 / 1440, 46.0 / 105, -1118711.0 / 3870720},
      {0, 0, 17.0 / 480, -37.0 / 840, -209.0 / 4480, 5569.0 / 90720},
      {0, 0, 0, 4397.0 / 161280, -11.0 / 504, -830251.0 / 7257600},
      {0, 0, 0, 0, 4583.0 / 161280, -108847.0 / 3991680},
      {0, 0, 0, 0, 0, 20648693.0 / 638668800}};
  for (int k = 0; k < kTmOrder; ++k) {
    double v = 0.0;
    for (int m = kTmOrder - 1; m >= 0; --m) v = v * n + c[k][m];
    p->beta[k] = v * n;
  }
  return true;
}

// one entry of the axis tables: row i (easting x) or column j (northing y)
__host__ __device__ inline void tm_row(double x, const TmParams& p, TmAxis* a) {
  a->v = (x - 500000.0) / p.k0A;
  for (int k = 0; k < kTmOrder; ++k) {
    a->a[k] = p.beta[k] * cosh(2.0 * (k + 1) * a->v);
    a->b[k] = p.beta[k] * sinh(2.0 * (k + 1) * a->v);
  }
}
__host__ __device__ inline void tm_col(double y, const TmParams& p, TmAxis* a) {
  a->v = (y - p.fn) / p.k0A;
  for (int k = 0; k < kTmOrder; ++k) {
    a->a[k] = sin(2.0 * (k + 1) * a->v);
    a->b[k] = cos(2.0 * (k + 1) * a->v);
  }
}

// The stripe's axis tables on the host (host libm), for the window only: t[0, rows) for the rows i, t[rows, rows + n)
// for the columns [col_begin, col_end), at the cells' positions as amb_geometry_position gives them
void tm_tables(const amb_geometry& g, int32_t col_begin, int32_t col_end, const TmParams& p, std::vector<TmAxis>* t) {
  t->resize(static_cast<size_t>(g.rows) + static_cast<size_t>(col_end - col_begin));
  double x, y;
  for (int32_t i = 0; i < g.rows; ++i) {
    amb_geometry_position(&g, i, col_begin, &x, &y);
    tm_row(x, p, &(*t)[i]);
  }
  for (int32_t j = col_begin; j < col_end; ++j) {
    amb_geometry_position(&g, 0, j, &x, &y);
    tm_col(y, p, &(*t)[static_cast<size_t>(g.rows) + (j - col_begin)]);
  }
}

// The same tables on the device, which the kernels read: one thread per entry, positions by amb_geometry_position's
// expression with every operation rounded (no contraction), so they are its bits
__global__ void __launch_bounds__(kImportThreads)
    tm_tables_kernel(amb_geometry g, int32_t col_begin, uint32_t rows, uint32_t ncols, TmParams p,
                     TmAxis* __restrict__ t) {
  const uint32_t k = blockIdx.x * kImportThreads + threadIdx.x;
  if (k >= rows + ncols) return;
  if (k < rows) {
    const double x0 = __dadd_rn(g.pos_x, __dadd_rn(__dmul_rn(0.5, g.length_x), -__dmul_rn(0.5, g.resolution)));
    tm_row(__dadd_rn(x0, __dmul_rn(g.resolution, -static_cast<double>(k))), p, &t[k]);
  } else {
    const double y0 = __dadd_rn(g.pos_y, __dadd_rn(__dmul_rn(0.5, g.length_y), -__dmul_rn(0.5, g.resolution)));
    const int32_t j = col_begin + static_cast<int32_t>(k - rows);
    tm_col(__dadd_rn(y0, __dmul_rn(g.resolution, -static_cast<double>(j))), p, &t[k]);
  }
}

// x y + z rounded once, on the device and on the host alike
__host__ __device__ inline double fma_rn(double x, double y, double z) {
#ifdef __CUDA_ARCH__
  return __fma_rn(x, y, z);
#else
  return std::fma(x, y, z);
#endif
}

struct LonLat {
  double lon, lat;  // degrees
};

// (lon, lat) of the cell at row entry ti and column entry tj.  The two series are explicit fused multiply-adds and the
// rest is one function that is not inlined, so the import kernels and the positions hook compute the same bits, and the
// hook returns the very positions the imports resample at.
__host__ __device__ __noinline__ LonLat tm_geodetic(double xip, double etap, double lon0, double e, double e2m) {
  const double s = sin(xip), c = cos(xip), sh = sinh(etap);
  const double taup = s / sqrt(sh * sh + c * c);  // tan(chi)
  double tau = taup / e2m;
  for (int it = 0; it < 2; ++it) {
    const double tau1 = sqrt(1.0 + tau * tau);
    const double sig = sinh(e * atanh(e * tau / tau1));
    const double taupa = sqrt(1.0 + sig * sig) * tau - sig * tau1;  // tan(chi) of tau
    tau += (taup - taupa) * (1.0 + e2m * tau * tau) / (e2m * tau1 * sqrt(1.0 + taupa * taupa));
  }
  return LonLat{lon0 + atan2(sh, c) * kRadToDeg, atan(tau) * kRadToDeg};
}

__host__ __device__ inline LonLat tm_lonlat(const TmAxis& ti, const TmAxis& tj, double lon0, double e, double e2m) {
  double xip = tj.v, etap = ti.v;
  for (int k = 0; k < kTmOrder; ++k) {
    xip = fma_rn(-tj.a[k], ti.a[k], xip);
    etap = fma_rn(-tj.b[k], ti.b[k], etap);
  }
  return tm_geodetic(xip, etap, lon0, e, e2m);
}

constexpr int kLonLatPositions = 2;  // the kernel's third mode: write (lon, lat), read no raster

struct LonLatArgs {
  double lon0, e, e2m;
  double gt0, gt1, gt3, gt5;  // the raster's geotransform
  int32_t width, height;      // the raster's pixels
  int32_t win_c0, win_r0, win_w, win_h;  // the copied window: band[0][0] is pixel (win_r0, win_c0)
  int has_nodata;
  float nodata;
};

// One thread per cell along i, kImportCols columns per thread, the block shape of raster_import_kernel.  MODE: NEAREST
// or BILINEAR resample into `layer` (a tap outside the window sets *outside and leaves the cell), or kLonLatPositions:
// (lon, lat) of cell (i, j) at lonlat[2 ((j - col_begin) rows + i)].
template <int MODE>
__global__ void __launch_bounds__(kImportThreads)
    raster_lonlat_kernel(const float* __restrict__ band, long long stride, const TmAxis* __restrict__ itab,
                         const TmAxis* __restrict__ jtab, uint32_t rows, uint32_t ncols, uint32_t row_blocks,
                         LonLatArgs a, float* __restrict__ layer, double* __restrict__ lonlat,
                         unsigned int* __restrict__ outside) {
  const uint32_t i = (blockIdx.x % row_blocks) * kImportThreads + threadIdx.x;
  const uint32_t j0 = (blockIdx.x / row_blocks) * kImportCols;
  if (i >= rows) return;
  const TmAxis ti = itab[i];
  for (int q = 0; q < kImportCols; ++q) {
    const uint32_t j = j0 + q;
    if (j >= ncols) return;
    const LonLat ll = tm_lonlat(ti, jtab[j], a.lon0, a.e, a.e2m);
    const double lon = ll.lon, lat = ll.lat;
    const size_t cell = static_cast<size_t>(j) * rows + i;
    if (MODE == kLonLatPositions) {
      lonlat[2 * cell] = lon;
      lonlat[2 * cell + 1] = lat;
      continue;
    }
    const ImportTap tx = axis_tap(lon, a.gt0, a.gt1, a.width, MODE);
    const ImportTap ty = axis_tap(lat, a.gt3, a.gt5, a.height, MODE);
    if (tx.k < 0 || ty.k < 0) continue;
    const int32_t c = tx.k - a.win_c0, r = ty.k - a.win_r0;
    if (c < 0 || r < 0 || c + (tx.f != 0.0) >= a.win_w || r + (ty.f != 0.0) >= a.win_h) {
      *outside = 1u;  // the host's window missed a tap: the call fails rather than read past the copy
      continue;
    }
    const float* p0 = band + (static_cast<long long>(r) * stride + c);
    if (MODE == AMB_RESAMPLE_NEAREST) {
      const float v = __ldg(p0);
      if (!no_data(v, a.has_nodata, a.nodata)) layer[cell] = v;
      continue;
    }
    const float p[4] = {__ldg(p0), tx.f != 0.0 ? __ldg(p0 + 1) : 0.0f, ty.f != 0.0 ? __ldg(p0 + stride) : 0.0f,
                        tx.f != 0.0 && ty.f != 0.0 ? __ldg(p0 + stride + 1) : 0.0f};
    float h;
    if (blend(p, tx.f, __dadd_rn(1.0, -tx.f), ty.f, a.has_nodata, a.nodata, &h)) layer[cell] = h;
  }
}

bool valid_epsg(int32_t epsg) {
  TmParams p;
  return tm_params(epsg, &p);
}

// Pixel window [c_lo, c_hi] x [r_lo, r_hi] of a width x height raster that holds every tap of the stripe's cells.  u
// and v are affine in longitude and latitude; longitude and the isometric latitude (monotone in latitude) are harmonic
// functions of (northing, easting), as the real and imaginary parts of an analytic map, so their extremes over the
// stripe's rectangle lie on its boundary.  A cell at u reads pixels in [floor(u - 1/2), floor(u - 1/2) + 1] under either
// method, so the window is that range at the boundary's extremes, one pixel wider on each side for the host's libm
// against the device's (and for extremes between two boundary cells), clamped to the raster.  0: the raster misses the
// stripe; 1: window set; AMB_ERR_INVALID_ARGUMENT: a boundary cell has no finite position.
int tm_window(const amb_geometry& g, int32_t col_begin, const std::vector<TmAxis>& t, const TmParams& p, int32_t width,
              int32_t height, const double* gt, int32_t* win) {
  const size_t rows = static_cast<size_t>(g.rows), ncols = t.size() - rows;
  double u_lo = INFINITY, u_hi = -INFINITY, v_lo = INFINITY, v_hi = -INFINITY;
  bool finite = true;
  auto visit = [&](size_t i, size_t j) {
    const LonLat ll = tm_lonlat(t[i], t[rows + j], p.lon0, p.e, p.e2m);
    const double u = (ll.lon - gt[0]) / gt[1], v = (ll.lat - gt[3]) / gt[5];
    finite = finite && std::isfinite(u) && std::isfinite(v);
    u_lo = std::min(u_lo, u);
    u_hi = std::max(u_hi, u);
    v_lo = std::min(v_lo, v);
    v_hi = std::max(v_hi, v);
  };
  for (size_t j = 0; j < ncols; ++j) {
    visit(0, j);
    visit(rows - 1, j);
  }
  for (size_t i = 0; i < rows; ++i) {
    visit(i, 0);
    visit(i, ncols - 1);
  }
  if (!finite) return AMB_ERR_INVALID_ARGUMENT;
  if (!(u_hi >= -1.0 && u_lo < width + 1.0 && v_hi >= -1.0 && v_lo < height + 1.0)) return 0;
  auto lo = [](double q) { return static_cast<int32_t>(std::max(std::floor(q - 0.5) - 1.0, 0.0)); };
  auto hi = [](double q, int32_t n) {
    return static_cast<int32_t>(std::min(std::floor(q - 0.5) + 2.0, static_cast<double>(n - 1)));
  };
  win[0] = lo(u_lo);
  win[1] = hi(u_hi, width);
  win[2] = lo(v_lo);
  win[3] = hi(v_hi, height);
  return 1;
}

// The stripe's window (see tm_window) from host tables: AMB_OK with *overlap, or an error status
int lonlat_plan(const amb_ctx* ctx, int32_t epsg, int32_t width, int32_t height, const double* gt, TmParams* p,
                std::vector<TmAxis>* t, int32_t* win, bool* overlap) {
  if (!tm_params(epsg, p)) return AMB_ERR_INVALID_ARGUMENT;
  tm_tables(ctx->geom, ctx->col_begin, ctx->col_end, *p, t);
  const int st = tm_window(ctx->geom, ctx->col_begin, *t, *p, width, height, gt, win);
  if (st < 0) return st;
  *overlap = st == 1;
  return AMB_OK;
}

// Enqueue the tables' build and the kernel on the context's stream.  band: the window win (c_lo, c_hi, r_lo, r_hi) of a
// width x height raster, rows `stride` floats apart (NULL for kLonLatPositions).  With `check`, waits for the kernel and
// fails if it met a tap outside the window.
int lonlat_enqueue(amb_ctx* ctx, int mode, int layer, const float* band, long long stride, const int32_t* win,
                   int32_t width, int32_t height, const double* gt, const TmParams& p, int has_nodata, float nodata,
                   double* lonlat, bool check) {
  int st = ensure_counters(ctx);
  if (st != AMB_OK) return st;
  if (mode != kLonLatPositions) {
    st = ensure_layer(ctx, layer);
    if (st != AMB_OK) return st;
    wait_layer_copy(ctx, layer);
  }
  const uint32_t rows = static_cast<uint32_t>(ctx->geom.rows);
  const uint32_t ncols = static_cast<uint32_t>(ctx->col_end - ctx->col_begin);
  AMB_CUDA(ctx, ctx->raster_taps.reserve((static_cast<size_t>(rows) + ncols) * sizeof(TmAxis)));
  TmAxis* itab = ctx->raster_taps.as<TmAxis>();
  tm_tables_kernel<<<(rows + ncols + kImportThreads - 1) / kImportThreads, kImportThreads, 0, ctx->stream>>>(
      ctx->geom, ctx->col_begin, rows, ncols, p, itab);
  unsigned int* outside = ctx->counters.as<unsigned int>() + CTR_LONLAT_OUTSIDE;
  AMB_CUDA(ctx, cudaMemsetAsync(outside, 0, sizeof(unsigned int), ctx->stream));
  LonLatArgs a{p.lon0, p.e, p.e2m, 0.0, 1.0, 0.0, -1.0, width, height, 0, 0, 0, 0, has_nodata, nodata};
  if (gt) {
    a.gt0 = gt[0];
    a.gt1 = gt[1];
    a.gt3 = gt[3];
    a.gt5 = gt[5];
    a.win_c0 = win[0];
    a.win_w = win[1] - win[0] + 1;
    a.win_r0 = win[2];
    a.win_h = win[3] - win[2] + 1;
  }
  const uint32_t row_blocks = (rows + kImportThreads - 1) / kImportThreads;
  const uint32_t grid = row_blocks * ((ncols + kImportCols - 1) / kImportCols);
  float* dst = mode == kLonLatPositions ? nullptr : ctx->layers[layer];
  if (mode == AMB_RESAMPLE_NEAREST)
    raster_lonlat_kernel<AMB_RESAMPLE_NEAREST><<<grid, kImportThreads, 0, ctx->stream>>>(
        band, stride, itab, itab + rows, rows, ncols, row_blocks, a, dst, lonlat, outside);
  else if (mode == AMB_RESAMPLE_BILINEAR)
    raster_lonlat_kernel<AMB_RESAMPLE_BILINEAR><<<grid, kImportThreads, 0, ctx->stream>>>(
        band, stride, itab, itab + rows, rows, ncols, row_blocks, a, dst, lonlat, outside);
  else
    raster_lonlat_kernel<kLonLatPositions><<<grid, kImportThreads, 0, ctx->stream>>>(
        band, stride, itab, itab + rows, rows, ncols, row_blocks, a, dst, lonlat, outside);
  AMB_CUDA(ctx, cudaGetLastError());
  if (!check) return AMB_OK;
  unsigned int missed = 0;
  AMB_CUDA(ctx, cudaMemcpyAsync(&missed, outside, sizeof(missed), cudaMemcpyDeviceToHost, ctx->stream));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (missed) {
    ctx->last_error = "amb_import_*_lonlat: a tap fell outside the raster window the host computed";
    return AMB_ERR_UNSUPPORTED;
  }
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

int amb_lonlat_import_window(const amb_geometry* geom, int32_t col_begin, int32_t col_end, int32_t map_epsg,
                             int32_t width, int32_t height, const double gt[6], int32_t window[4]) {
  TmParams p;
  if (!geom || !window || geom->rows <= 0 || geom->cols <= 0 || !(geom->resolution > 0.0) || col_begin < 0 ||
      col_end > geom->cols || col_begin >= col_end || !tm_params(map_epsg, &p) ||
      !import_args_ok(0, width, height, 4 * static_cast<size_t>(width), gt, AMB_RESAMPLE_NEAREST))
    return AMB_ERR_INVALID_ARGUMENT;
  std::vector<TmAxis> t;
  tm_tables(*geom, col_begin, col_end, p, &t);
  const int st = tm_window(*geom, col_begin, t, p, width, height, gt, window);
  if (st < 0) return st;
  if (st == 0) window[0] = window[1] = window[2] = window[3] = -1;
  return AMB_OK;
}

int amb_lonlat_positions_device(amb_ctx* ctx, int32_t map_epsg, double* d_lonlat) {
  TmParams p;
  if (!ctx || !d_lonlat || (reinterpret_cast<uintptr_t>(d_lonlat) & 7) != 0 || !tm_params(map_epsg, &p))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return lonlat_enqueue(ctx, kLonLatPositions, 0, nullptr, 0, nullptr, 0, 0, nullptr, p, 0, 0.0f, d_lonlat, false);
}

int amb_import_raster_lonlat_device(amb_ctx* ctx, int layer, const float* device_band, int32_t width, int32_t height,
                                    size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample,
                                    int32_t map_epsg) {
  TmParams p;
  if (!ctx || !device_band || (reinterpret_cast<uintptr_t>(device_band) & 3) != 0 || !tm_params(map_epsg, &p) ||
      !import_args_ok(layer, width, height, row_stride, gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  // the band is read in place: no host window, its window is the whole raster, which holds every tap by the coverage
  // rule; a raster that misses the stripe costs one launch and writes nothing
  const int32_t whole[4] = {0, width - 1, 0, height - 1};
  return lonlat_enqueue(ctx, resample, layer, device_band, static_cast<long long>(row_stride / 4), whole, width, height,
                        gt, p, has_nodata, nodata, nullptr, false);
}

int amb_import_raster_lonlat(amb_ctx* ctx, int layer, const float* host_band, int32_t width, int32_t height,
                             size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample,
                             int32_t map_epsg) {
  if (!ctx || !host_band || !valid_epsg(map_epsg) || !import_args_ok(layer, width, height, row_stride, gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  TmParams p;
  std::vector<TmAxis> t;
  int32_t win[4];
  bool overlap;
  int st = lonlat_plan(ctx, map_epsg, width, height, gt, &p, &t, win, &overlap);
  if (st != AMB_OK || !overlap) return st;
  const size_t win_w = static_cast<size_t>(win[1] - win[0] + 1), win_h = static_cast<size_t>(win[3] - win[2] + 1);
  AMB_CUDA(ctx, ctx->raster_band.reserve(win_w * win_h * sizeof(float)));
  const StagedRect rect{ctx->raster_band.as<unsigned char>(), win_w * sizeof(float),
                        reinterpret_cast<const unsigned char*>(host_band) + static_cast<size_t>(win[2]) * row_stride +
                            static_cast<size_t>(win[0]) * sizeof(float),
                        row_stride, win_w * sizeof(float), win_h};
  st = staged_h2d_rects(ctx, &rect, 1, ctx->stream);
  if (st != AMB_OK) return st;
  // synchronous: the caller's band (pinned: read by the DMA) may be reused, and the window check is read back
  return lonlat_enqueue(ctx, resample, layer, ctx->raster_band.as<float>(), static_cast<long long>(win_w), win, width,
                        height, gt, p, has_nodata, nodata, nullptr, true);
}

int amb_import_tiff_lonlat(amb_ctx* ctx, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                           const double gt[6], int has_nodata, float nodata, int resample, int32_t map_epsg) {
  if (!ctx || !file || !valid_epsg(map_epsg) || tiff_layout_check(layout, bytes) != AMB_OK ||
      !import_args_ok(layer, layout->width, layout->height, 4 * static_cast<size_t>(layout->width), gt, resample))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  TmParams p;
  std::vector<TmAxis> t;
  int32_t win[4];
  bool overlap;
  int st = lonlat_plan(ctx, map_epsg, layout->width, layout->height, gt, &p, &t, win, &overlap);
  if (st != AMB_OK || !overlap) return st;
  const size_t win_w = static_cast<size_t>(win[1] - win[0] + 1), win_h = static_cast<size_t>(win[3] - win[2] + 1);
  AMB_CUDA(ctx, ctx->raster_band.reserve(win_w * win_h * sizeof(float)));
  st = tiff_decode_window(ctx, static_cast<const unsigned char*>(file), *layout, win[2], win[3] + 1, win[0], win[1] + 1,
                          ctx->raster_band.as<float>(), win_w);
  if (st != AMB_OK) return st;
  return lonlat_enqueue(ctx, resample, layer, ctx->raster_band.as<float>(), static_cast<long long>(win_w), win,
                        layout->width, layout->height, gt, p, has_nodata, nodata, nullptr, true);
}

}  // extern "C"
