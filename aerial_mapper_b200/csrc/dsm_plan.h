// dsm_plan.h — the launch plan, the sorted-point record, the exact-arithmetic and bucket-window device helpers and the
// warp-aggregated append shared by the DSM kernels (dsm_kernels.cu) and the adaptive OrthoFromPcl pass
// (pcl_adaptive_kernels.cu).
#ifndef AMB_DSM_PLAN_H_
#define AMB_DSM_PLAN_H_

#include <cuda_runtime.h>

#include <cfloat>
#include <cstddef>

#include "approx_math.h"
#include "halo_push.h"
namespace amb {
namespace dsmk {

constexpr int kMaxThresholds = 32;
constexpr int kMaxHalfWidth = 128;  // cells; window half-width limit (sqrt(threshold)/resolution)

struct PointRec {  // 32 bytes, one DRAM sector
  double x, y, z;
  // low word: original index (or the caller's global point id, < 2^32) — the canonical-order key;
  // high word: the point's fine bin as computed ONCE by the scatter kernel, (bi << 4) | (bj & 15), so that the tile
  // gather bins its window with integer arithmetic only (bj's upper bits follow from the bucket row the record is in)
  unsigned long long idx;
};
__host__ __device__ inline unsigned int rec_id(unsigned long long idx_word) { return static_cast<unsigned int>(idx_word); }
__host__ __device__ inline unsigned int rec_code(unsigned long long idx_word) { return static_cast<unsigned int>(idx_word >> 32); }

struct DsmPlan {
  int rows, cols_slab, col_begin;
  int W;          // window half-width (cells) of the primary threshold
  int P;          // reach (cells) of the largest retry threshold
  int Pa;         // apron of the bin grid (cells): P rounded up to a multiple of B
  int B, Bshift;  // bucket edge in cells (power of two) and its log2
  int BR, BC;     // fine bin grid (cells): bin (bi, bj) <-> cell (bi - Pa, gj0 + bj)
  int KR, KC;     // bucket grid
  int gj0;        // global column of bin column 0 (a multiple of TJ minus Pa: tiles align to GLOBAL columns)
  int tile_j0;    // global tile index of the first tile column of this stripe
  int mode;       // 0: dsm::Dsm (retry thresholds, coincident point = error); 1: ortho::OrthoFromPcl (no retry,
                  //    a zero-distance point is a "perfect match", ortho-from-pcl.cc:90-96)
  double base_x, base_y;  // cell centre of index 0: pos + (0.5*length - 0.5*res)   (grid_map getPosition)
  double res, inv_res;
  double shift_x, shift_y;  // dsm.cc:42-43: x -= center_northing, y -= center_easting
  double thr0;
  int n_thr;
  double thr[kMaxThresholds];
  short hw[kMaxHalfWidth + 1];  // half-width along i of the primary window at |dj|
  // FP32 gather (dsm_gather_f32.inc)
  float thr_f;          // (float)thr0 — an int, exact
  float eps_f;          // |d2_f32 - d2_reference| <= eps_f for every pair a tile can stage (see dsm_run)
  double zrange_limit;  // tiles whose staged heights span more than this go to the all-FP64 kernel
  float hdelta;         // |(dx_f, dy_f) - (dx, dy)| <= hdelta + u |(dx_f, dy_f)| for every staged pair (height bound)
  float hden_max;       // hdelta sqrt(den) (1 + 3u) + u <= 0.01  <=>  den <= hden_max
};

__device__ __forceinline__ double cell_x(const DsmPlan& p, int i) {
  // position = (mapPosition + offset) + resolution * (-(double)index); un-contracted like the CPU
  return __dadd_rn(p.base_x, __dmul_rn(p.res, -static_cast<double>(i)));
}
__device__ __forceinline__ double cell_y(const DsmPlan& p, int j_global) {
  return __dadd_rn(p.base_y, __dmul_rn(p.res, -static_cast<double>(j_global)));
}

// Fine bin (= nearest cell centre) of a shifted point; false if it lies outside the bin grid of this slab, i.e.
// cannot reach any of its cells.  An off-by-one at a cell edge is harmless: membership is re-decided exactly by
// d2 and every window carries half a cell of slack (see half_widths()).
// (explicit fma: the two-level binning evaluates the column twice — once per pass — and must get the same bin)
__device__ __forceinline__ double fine_bin_col(const DsmPlan& p, double py) {
  return floor(fma(p.base_y - py, p.inv_res, 0.5)) - static_cast<double>(p.gj0);
}
__device__ __forceinline__ bool fine_bin(const DsmPlan& p, double px, double py, int* bi, int* bj) {
  const double fi = floor(fma(p.base_x - px, p.inv_res, 0.5)) + static_cast<double>(p.Pa);
  const double fj = fine_bin_col(p, py);
  if (!(fi >= 0.0 && fi < static_cast<double>(p.BR) && fj >= 0.0 && fj < static_cast<double>(p.BC))) return false;
  *bi = static_cast<int>(fi);
  *bj = static_cast<int>(fj);
  return true;
}

// Buckets overlapping fine bins [bi - P, bi + P] x [bj - P, bj + P] (clamped to the bin grid).  Bucket row kj of the
// window is one contiguous record range, [G[kj * KR + kbi0], G[kj * KR + kbi1 + 1]).
struct BucketWindow {
  int kbi0, kbi1, kbj0, kbj1;
};
__device__ __forceinline__ BucketWindow bucket_window(const DsmPlan& p, int bi, int bj, int P) {
  return {max(bi - P, 0) >> p.Bshift, min(bi + P, p.BR - 1) >> p.Bshift, max(bj - P, 0) >> p.Bshift,
          min(bj + P, p.BC - 1) >> p.Bshift};
}

// Smallest d2 from (qx, qy) to the records of a bucket window, reduced over the warp (every lane calls it).  The minimum
// does not depend on the visiting order, so the records are read in bucket order.
__device__ __forceinline__ double window_min_d2(const DsmPlan& p, const unsigned int* G, const PointRec* rec,
                                                const BucketWindow& w, double qx, double qy, int lane) {
  double dmin = DBL_MAX;
  for (int kj = w.kbj0; kj <= w.kbj1; ++kj) {
    const size_t row = static_cast<size_t>(kj) * p.KR;
    const unsigned int lo = G[row + w.kbi0];
    const unsigned int hi = G[row + w.kbi1 + 1];
    for (unsigned int k = lo + lane; k < hi; k += 32) {
      const double2 v = __ldg(reinterpret_cast<const double2*>(rec + k));
      const double dx = qx - v.x;
      const double dy = qy - v.y;
      dmin = fmin(dmin, __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));  // L2_Adaptor, un-contracted
    }
  }
  for (int o = 16; o > 0; o >>= 1) dmin = fmin(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
  return dmin;
}

// Warp-aggregated append (every lane of the warp calls it): the lanes with `take` store `value` to consecutive slots
// of `list` in lane order.
__device__ __forceinline__ void warp_append(bool take, unsigned int* counter, unsigned int* list, unsigned int value) {
  warp_reserve(take, counter, [&](unsigned int slot) { list[slot] = value; });
}

}  // namespace dsmk
}  // namespace amb
#endif  // AMB_DSM_PLAN_H_
