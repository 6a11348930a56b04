// pcl_adaptive_kernels.cu — ortho::Settings::use_adaptive_interpolation of ortho::OrthoFromPcl::process
// ("next" row N1, SURVEY.md §8f; reference aerial_mapper_ortho/src/ortho-from-pcl.cc:63-72):
//
//     if (use_adaptive_interpolation) { int lambda = 10;
//       while (result_set.size() == 0u) { tmp(lambda * interpolation_radius, ...); findNeighbors(tmp); lambda *= 10; } }
//
// i.e. a cell whose primary ball (d2 < radius) is empty takes the IDW over the first non-empty ball of the
// thresholds 10*r, 100*r, 1000*r, ... (squared metres, `int` arithmetic in the reference: defined while
// 10^k * r <= INT_MAX).  Every cell ends up with a value (the cloud is not empty, :23).
//
// Built on the regular OrthoFromPcl pass without touching its kernels:
//   prepare : the `ortho` slab is saved and filled with NaN (no IDW of finite intensities is NaN: a sentinel);
//   dsm_run : the regular one-radius pass (mode 1) writes every cell with a non-empty primary ball;
//   finish  : cells still NaN are listed (pcl_adaptive_list_kernel) and evaluated one warp per cell
//             (pcl_adaptive_cell_kernel) straight from the bucket records the pass left in HBM — per level the
//             smallest d2 over the window the threshold can reach, then the IDW over d2 < threshold, visiting
//             records through order[] (canonical order) exactly like dsm_cell_kernel does for the DSM's retry loop.
// On a stripe (a context owning columns [col_begin, col_end) that is passed the WHOLE cloud, as amb_multi does) the
// regular pass bins only what reaches the stripe, while a far threshold may need any point.  finish therefore bins the
// cloud again with the plan a whole-map context builds (same density, hence the same bucket edge; the same global
// bucket lattice, tile_j0 = 0) and maps the stripe's cells into that grid (plan.col_begin = the stripe's first column,
// gj0 = the whole map's): every cell visits the same buckets in the same order with the same lane split as in the
// whole-map run, so the stripe is bit-identical to those columns.  A whole-map context reuses the regular pass's bins.
// Restrictions (AMB_ERR_UNSUPPORTED, layer restored): every point must lie inside the map's bin grid (map + apron),
// because the binning drops what lies outside; radius growth beyond `int` range is undefined behaviour in the reference.
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>

#include "amb_context.h"
#include "dsm_plan.h"

namespace amb {

using namespace dsmk;

namespace {

constexpr int kMaxAdaptiveLevels = 10;

struct AdaptiveArgs {
  const unsigned int* G;
  const unsigned int* order;
  const PointRec* rec;
  float* ortho;
  const unsigned int* cell_list;
  const unsigned int* n_cells;  // device counter written by the list kernel
  unsigned int* unresolved;     // device flag: some cell found no neighbour within the last defined threshold
  int n_levels;
  double thr[kMaxAdaptiveLevels];  // (double)(10^k * radius), k = 1 ..
  int reach[kMaxAdaptiveLevels];   // window half-width in cells that threshold can reach
};

__global__ void __launch_bounds__(256) pcl_adaptive_list_kernel(const float* __restrict__ ortho, size_t cells,
                                                                unsigned int* __restrict__ cell_list,
                                                                unsigned int* __restrict__ n_cells) {
  // whole warps iterate together (the ballot needs every lane): round the trip count up to a warp multiple
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t cells_up = (cells + 31) & ~static_cast<size_t>(31);
  for (size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; c < cells_up; c += stride) {
    const bool empty = c < cells && ortho[c] != ortho[c];  // still the NaN sentinel
    warp_append(empty, n_cells, cell_list, static_cast<unsigned int>(c));
  }
}

__global__ void __launch_bounds__(256) pcl_adaptive_cell_kernel(const __grid_constant__ DsmPlan plan,
                                                                const __grid_constant__ AdaptiveArgs a) {
  const int lane = threadIdx.x & 31;
  const size_t n_cells = *a.n_cells;
  const size_t warps_total = static_cast<size_t>(gridDim.x) * (blockDim.x >> 5);  // 64-bit cursor: see dsm_cell_kernel
  for (size_t c = blockIdx.x * static_cast<size_t>(blockDim.x >> 5) + (threadIdx.x >> 5); c < n_cells; c += warps_total) {
    const unsigned int cell = a.cell_list[c];
    const int i = static_cast<int>(cell % static_cast<unsigned int>(plan.rows));
    const int jl = static_cast<int>(cell / static_cast<unsigned int>(plan.rows));
    const double qx = cell_x(plan, i);
    const double qy = cell_y(plan, plan.col_begin + jl);
    const int bi = i + plan.Pa, bj = plan.col_begin + jl - plan.gj0;

    // first threshold whose (strict) ball is non-empty (ortho-from-pcl.cc:66-71)
    int level = -1;
    for (int L = 0; L < a.n_levels; ++L) {
      const int P = a.reach[L];
      const double dmin = window_min_d2(plan, a.G, a.rec, bucket_window(plan, bi, bj, P), qx, qy, lane);
      if (dmin < a.thr[L]) {
        level = L;
        break;
      }
      const bool whole_grid = bi - P <= 0 && bi + P >= plan.BR - 1 && bj - P <= 0 && bj + P >= plan.BC - 1;
      if (whole_grid) {  // dmin is the distance to the nearest point of the cloud: larger windows see the same
        for (int M = L + 1; M < a.n_levels; ++M) {
          if (dmin < a.thr[M]) {
            level = M;
            break;
          }
        }
        break;
      }
    }
    if (level < 0) {
      if (lane == 0) atomicExch(a.unresolved, 1u);
      continue;
    }

    const double thr = a.thr[level];
    const BucketWindow w = bucket_window(plan, bi, bj, a.reach[level]);
    double num = 0.0, den = 0.0;
    for (int kj = w.kbj0; kj <= w.kbj1; ++kj) {
      const size_t row = static_cast<size_t>(kj) * plan.KR;
      const unsigned int lo = a.G[row + w.kbi0];
      const unsigned int hi = a.G[row + w.kbi1 + 1];
      for (unsigned int k = lo + lane; k < hi; k += 32) {
        const PointRec* pr = a.rec + __ldg(a.order + k);  // canonical order: the lanes' partial sums are fixed
        const double2 v = __ldg(reinterpret_cast<const double2*>(pr));
        const double dx = qx - v.x;
        const double dy = qy - v.y;
        const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        // d2 > 0: a zero-distance point would have made the primary ball non-empty, so it cannot occur here
        if (d2 < thr && d2 > 0.0) {
          const double pz = __ldg(reinterpret_cast<const double*>(pr) + 2);
          const double w = fast_rcp(d2);  // 1.0 / distances[i]            (ortho-from-pcl.cc:100)
          num = fma(pz, w, num);          // heights[i] / distances[i]     (:99)
          den += w;
        }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      num += __shfl_xor_sync(0xffffffffu, num, o);
      den += __shfl_xor_sync(0xffffffffu, den, o);
    }
    if (lane == 0) a.ortho[cell] = __double2float_rn(__ddiv_rn(num, den));  // :104-106
  }
}

}  // namespace

// Before the regular pass: the slab is saved to `*saved` (device memory the caller releases through
// pcl_adaptive_finish) and filled with the NaN sentinel.
int pcl_adaptive_prepare(amb_ctx* ctx, float** saved) {
  *saved = nullptr;
  int st = ensure_layer(ctx, AMB_LAYER_ORTHO);
  if (st != AMB_OK) return st;
  wait_layer_copy(ctx, AMB_LAYER_ORTHO);
  const size_t bytes = ctx->slab_cells() * sizeof(float);
  AMB_CUDA(ctx, cudaMalloc(saved, bytes));
  AMB_CUDA(ctx, cudaMemcpyAsync(*saved, ctx->layers[AMB_LAYER_ORTHO], bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  AMB_CUDA(ctx, cudaMemsetAsync(ctx->layers[AMB_LAYER_ORTHO], 0xff, bytes, ctx->stream));  // 0xffffffff: a NaN
  return AMB_OK;
}

// After the regular pass (`pass_status` = what dsm_run returned).  On any failure the slab gets its saved content back.
int pcl_adaptive_finish(amb_ctx* ctx, int pass_status, const double* d_xyz, const unsigned long long* d_ids,
                        const int* d_intensities, size_t n, int32_t interpolation_radius, float* saved) {
  const size_t cells = ctx->slab_cells();
  const size_t bytes = cells * sizeof(float);
  float* ortho = ctx->layers[AMB_LAYER_ORTHO];
  cudaStream_t s = ctx->stream;
  auto restore = [&](int status) {
    if (saved && ortho) {
      wait_layer_copy(ctx, AMB_LAYER_ORTHO);
      cudaMemcpyAsync(ortho, saved, bytes, cudaMemcpyDeviceToDevice, s);
      cudaStreamSynchronize(s);
    }
    if (saved) cudaFree(saved);
    return status;
  };
  if (pass_status != AMB_OK) return restore(pass_status);
  if (ctx->col_begin != 0 || ctx->col_end != ctx->geom.cols) {  // a stripe: the whole map's bins (see the file header)
    const int st = dsm_run(ctx, d_xyz, d_ids, n, interpolation_radius, 0.0, 0.0, 1, d_intensities, nullptr, nullptr, true);
    if (st != AMB_OK) return restore(st);
  }
  if (ctx->last_dsm_plan.size() != sizeof(DsmPlan)) return restore(AMB_ERR_INVALID_ARGUMENT);
  DsmPlan plan;
  std::memcpy(&plan, ctx->last_dsm_plan.data(), sizeof(plan));

  unsigned int* counters = ctx->counters.as<unsigned int>();  // see amb::CounterSlot
  unsigned int h_counters[16];
  if (cudaMemcpyAsync(h_counters, counters, sizeof(h_counters), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
      cudaStreamSynchronize(s) != cudaSuccess) {
    cudaGetLastError();
    return restore(AMB_ERR_CUDA);
  }
  if (static_cast<size_t>(h_counters[CTR_DSM_BINNED]) != n) {
    ctx->last_error = "adaptive interpolation needs every point inside the map's bin grid (map + apron)";
    return restore(AMB_ERR_UNSUPPORTED);
  }

  AdaptiveArgs a;
  std::memset(&a, 0, sizeof(a));
  a.G = ctx->bin_starts.as<unsigned int>();
  a.order = ctx->point_order.as<unsigned int>();
  a.rec = ctx->records.as<PointRec>();
  a.ortho = ortho;
  a.cell_list = ctx->empty_cells.as<unsigned int>();
  a.n_cells = counters + CTR_PCL_CELLS;
  a.unresolved = counters + CTR_PCL_UNRESOLVED;
  // thresholds (double)(lambda * interpolation_radius), lambda = 10, 100, ... in `int` (ortho-from-pcl.cc:64-70)
  long long lambda = 10;
  const double slack = 1e-6;
  while (a.n_levels < kMaxAdaptiveLevels && lambda * interpolation_radius <= static_cast<long long>(INT_MAX) &&
         lambda <= static_cast<long long>(INT_MAX)) {
    const double thr = static_cast<double>(static_cast<int>(lambda) * interpolation_radius);
    a.thr[a.n_levels] = thr;
    const double reach = std::floor(std::sqrt(thr) / ctx->geom.resolution + 0.5 + slack);
    a.reach[a.n_levels] = reach > 1.0e9 ? 1000000000 : static_cast<int>(reach);
    ++a.n_levels;
    lambda *= 10;
  }

  wait_layer_copy(ctx, AMB_LAYER_ORTHO);  // the regular pass may have started mirroring the layer to the host
  if (cudaMemsetAsync(counters + CTR_PCL_CELLS, 0, 2 * sizeof(unsigned int), s) != cudaSuccess) {
    cudaGetLastError();
    return restore(AMB_ERR_CUDA);
  }
  pcl_adaptive_list_kernel<<<ctx->num_sms * 8, 256, 0, s>>>(ortho, cells, ctx->empty_cells.as<unsigned int>(),
                                                            counters + CTR_PCL_CELLS);
  pcl_adaptive_cell_kernel<<<ctx->num_sms * 8, 256, 0, s>>>(plan, a);
  ctx->dsm_launches += 2;
  if (cudaGetLastError() != cudaSuccess ||
      cudaMemcpyAsync(h_counters, counters, sizeof(h_counters), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
      cudaStreamSynchronize(s) != cudaSuccess) {
    cudaGetLastError();
    return restore(AMB_ERR_CUDA);
  }
  if (h_counters[CTR_PCL_UNRESOLVED]) {
    ctx->last_error = "adaptive interpolation: no neighbour within 10^k * radius <= INT_MAX (undefined in the reference)";
    return restore(AMB_ERR_UNSUPPORTED);
  }
  ctx->last_cells_empty = static_cast<int64_t>(h_counters[CTR_PCL_CELLS]);
  cudaFree(saved);
  return mirror_layer(ctx, AMB_LAYER_ORTHO);  // the final layer (re)starts streaming to its host mirror
}

}  // namespace amb
