// dsm_kernels.cu — point cloud -> `elevation` layer on sm_90a.
//
// Replaces dsm::Dsm::process (reference aerial_mapper_dsm/src/dsm.cc:186-201): kd-tree build (:36-52) + one
// radius query and IDW per cell (:113-184).  The reference's result for a cell is
//     S   = { p : d2(p) < threshold }                 d2 = (qx-px)^2 + (qy-py)^2, un-contracted double
//     h   = (sum_S z/d2) / (sum_S 1/d2)                elevation(i,j) = (float)h
// with threshold = (double)interpolation_radius, or, when that set is empty, the first of the retry thresholds
// lambda_k*radius (dsm.cc:133-144) that yields a non-empty set.  Nothing in that definition needs a tree.
//
// Layout of the work
//   HBM:   points are sorted into COARSE buckets of BxB grid cells (B a power of two chosen so that a bucket holds
//          a few dozen points; 8x8 cells at the benchmark density), each bucket's records one contiguous run.  Every
//          32-byte record {x, y, z, index word} carries the point's fine bin (nearest cell), computed once.
//   SMEM:  a 32x32-cell tile loads the buckets overlapping its window (tile + apron), bins their points with
//          shared-memory atomics, orders every bin's points by original index, and gathers from there.
//
// Pipeline (all on the context's stream):
//   K1 dsm_partition_kernel      (dsm_partition.inc) bins every point once in double precision, counts the buckets
//                                (atomics resolve in L2) and groups each tile of 2048 points by coarse destination
//   K2 scan_*                    inclusive scan of the bucket counts -> bucket start offsets
//   K3 dsm_fine_scatter_kernel   (dsm_partition.inc) records into bucket order, one coarse destination at a time
//   K4 dsm_gather_kernel_f32     one tile per block: bucket runs -> bins in shared memory -> every thread owns a 1x4
//      dsm_gather_kernel         strip of cells and walks the strip's bin rows in one flattened loop.  FP32 sums with
//                                exact decisions (the default; Dsm only) or all FP64; cells it cannot decide exactly
//                                and every cell of a tile too dense for the stage go to the cell list
//   K5 dsm_mark_buckets_kernel   flags the buckets the listed cells can reach (Dsm; OrthoFromPcl orders every bucket
//      dsm_bucket_order_kernel   after K3): the visiting order of a flagged bucket's records by original index
//                                (canonical order: the IDW summation order — hence every output bit — is independent
//                                of atomic scheduling and of how the map is striped across GPUs)
//   K6 dsm_cell_kernel           one warp per listed cell: the expanding-radius retry (dsm.cc:133-144) and the cells
//                                handed over by K4, from the bucket records in HBM
// With amb_dsm_set_stream_chunks, K4-K6 run once per group of tile columns.
//
// Membership (d2 < threshold) is evaluated with __dmul_rn/__dadd_rn (no FMA contraction) in the reference's
// operation order, so neighbour sets and retry levels are bit-exact decisions.  Heights differ from the CPU only
// by the order of the double-precision summation and by z*(1/d2) replacing z/d2 (both O(1e-16) relative).
#include <cfloat>
#include <cmath>
#include <cstdlib>

#include "amb_context.h"
#include "dsm_plan.h"
#include "halo_push.h"

namespace amb {

using namespace dsmk;  // DsmPlan, PointRec, cell_x/cell_y, fine_bin, fast_rcp

std::vector<double> dsm_thresholds(int32_t interpolation_radius) {
  // dsm.cc:133-144: lambda = 1; while (empty) { search(lambda*radius); lambda *= 1.1; if (lambda*radius > 7) break; }
  std::vector<double> thr;
  double lambda = 1.0;
  while (true) {
    thr.push_back(lambda * interpolation_radius);
    lambda *= 1.1;
    if (lambda * interpolation_radius > 7.0) break;
  }
  return thr;
}

namespace {

constexpr int TI = 32;              // tile extent along i (rows, the contiguous axis of the layer)
constexpr int TJ = 32;              // tile extent along j
constexpr int kGatherThreads = 256;
constexpr int kStrip = 4;           // cells per thread in the gather kernel (adjacent along j)
constexpr int kScanChunk = 4096;    // elements per block in the scan kernels (256 threads x 16)
constexpr int kSortRegs = 4;        // bucket sort: records per lane held in registers (buckets up to 128 points)
static_assert(TJ == kStrip * (kGatherThreads / 32), "one warp per strip row of the tile");

// ---------------------------------------------------------------------------------------------------------------
// K2: inclusive scan (reduce / spine / apply).
__device__ __forceinline__ unsigned int block_exclusive_scan(unsigned int v, unsigned int* total) {
  // `total` must point to shared memory; valid after return.
  __shared__ unsigned int warp_sums[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = blockDim.x >> 5;
  unsigned int inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const unsigned int w = lane < nwarps ? warp_sums[lane] : 0u;
    unsigned int winc = w;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    warp_sums[lane] = winc - w;  // exclusive prefix of the warp totals
    if (lane == 31) *total = winc;
  }
  __syncthreads();
  const unsigned int r = warp_sums[warp] + inc - v;
  __syncthreads();  // warp_sums is reused by the next call
  return r;
}

__global__ void __launch_bounds__(256) scan_reduce_kernel(const uint4* __restrict__ in, size_t n_vec,
                                                          unsigned int* __restrict__ block_sums) {
  const size_t base = static_cast<size_t>(blockIdx.x) * (kScanChunk / 4);
  unsigned int s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const size_t v = base + k * 256 + threadIdx.x;
    if (v < n_vec) {
      const uint4 q = in[v];
      s += q.x + q.y + q.z + q.w;
    }
  }
  __shared__ unsigned int total;
  block_exclusive_scan(s, &total);
  if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) scan_spine_kernel(unsigned int* __restrict__ block_sums, int n) {
  __shared__ unsigned int total;
  __shared__ unsigned int carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int k = base + threadIdx.x;
    const unsigned int v = k < n ? block_sums[k] : 0u;
    const unsigned int ex = block_exclusive_scan(v, &total);
    const unsigned int carry = carry_s;
    if (k < n) block_sums[k] = ex + carry;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + total;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) scan_apply_kernel(uint4* __restrict__ data, size_t n_vec,
                                                         const unsigned int* __restrict__ block_sums) {
  // blocked arrangement: thread t owns 4 consecutive uint4 (16 values) so that the scan order is the array order
  const size_t base = static_cast<size_t>(blockIdx.x) * (kScanChunk / 4) + threadIdx.x * 4;
  uint4 q[4];
  unsigned int s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    q[k] = (base + k < n_vec) ? data[base + k] : make_uint4(0, 0, 0, 0);
    s += q[k].x + q[k].y + q[k].z + q[k].w;
  }
  __shared__ unsigned int total;
  unsigned int run = block_exclusive_scan(s, &total) + block_sums[blockIdx.x];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    q[k].x += run;
    q[k].y += q[k].x;
    q[k].z += q[k].y;
    q[k].w += q[k].z;
    run = q[k].w;
    if (base + k < n_vec) data[base + k] = q[k];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// K1 / K3: two-level binning
#include "dsm_partition.inc"

// K5: canonical order inside every bucket (ascending original index = what a stable sort would give), as an
// index array: order[s + r] = position of the bucket's r-th smallest original index.  Only the warp-per-cell
// kernel needs it (the tile kernel orders every cell's points in shared memory); writing 4 bytes per point
// instead of permuting the 32-byte records keeps this pass at one read of the records.
// One warp per bucket; every lane ranks its keys against all keys of the bucket (broadcast loads).
template <int R>
__device__ __forceinline__ void rank_bucket(const PointRec* __restrict__ rec, unsigned int* __restrict__ order,
                                            unsigned int* skeys, unsigned int s, unsigned int k, int lane) {
  // original indices are < 2^32 (n is checked on the host): compare their low words
  unsigned int key[R], rank[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const unsigned int q = lane + 32u * r;
    key[r] = q < k ? static_cast<unsigned int>(__ldg(&rec[s + q].idx)) : 0xffffffffu;
    rank[r] = 0;
    skeys[q] = key[r];  // slots >= k hold 0xffffffff: never smaller than a real key
  }
  __syncwarp();
  const unsigned int k4 = (k + 3u) >> 2;
  const uint4* sk4 = reinterpret_cast<const uint4*>(skeys);
  for (unsigned int q = 0; q < k4; ++q) {
    const uint4 o = sk4[q];  // broadcast
#pragma unroll
    for (int r = 0; r < R; ++r)
      rank[r] += (o.x < key[r] ? 1u : 0u) + (o.y < key[r] ? 1u : 0u) + (o.z < key[r] ? 1u : 0u) +
                 (o.w < key[r] ? 1u : 0u);
  }
  __syncwarp();
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const unsigned int q = lane + 32u * r;
    if (q < k) order[s + rank[r]] = s + q;
  }
}

// `flags` (one byte per bucket, or nullptr = every bucket): only the buckets the warp-per-cell kernel is going to read
// are ordered — dsm_mark_buckets_kernel sets the bytes from the cell list after the gather, this kernel clears them.
// At the benchmark density ~30 % of the buckets are touched by a listed cell.
__global__ void __launch_bounds__(256) dsm_bucket_order_kernel(const unsigned int* __restrict__ G,
                                                               unsigned int n_buckets,
                                                               const PointRec* __restrict__ rec,
                                                               unsigned int* __restrict__ order,
                                                               unsigned char* __restrict__ flags) {
  constexpr int kMaxK = 32 * kSortRegs;  // bucket sizes handled through shared memory
  __shared__ __align__(16) unsigned int skeys[8][kMaxK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned int warps_total = gridDim.x * (blockDim.x >> 5);
  // a warp takes 32 consecutive buckets at a time: one flag byte per lane, then the flagged ones in turn
  for (unsigned int b0 = (blockIdx.x * (blockDim.x >> 5) + warp) * 32u; b0 < n_buckets; b0 += warps_total * 32u) {
    const unsigned int bl = b0 + lane;
    bool mine = bl < n_buckets;
    if (mine && flags) {
      mine = flags[bl] != 0;
      if (mine) flags[bl] = 0;
    }
    unsigned int todo = __ballot_sync(0xffffffffu, mine);
    while (todo) {
      const unsigned int b = b0 + static_cast<unsigned int>(__ffs(todo) - 1);
      todo &= todo - 1u;
      const unsigned int s = G[b], e = G[b + 1];
      const unsigned int k = e - s;
      if (k == 0) continue;
      if (k <= 32u) {
        rank_bucket<1>(rec, order, skeys[warp], s, k, lane);
      } else if (k <= 64u) {
        rank_bucket<2>(rec, order, skeys[warp], s, k, lane);
      } else if (k <= static_cast<unsigned int>(kMaxK)) {
        rank_bucket<kSortRegs>(rec, order, skeys[warp], s, k, lane);
      } else {
        // far denser than the bucket size was chosen for: rank against the keys in global memory
        for (unsigned int q = lane; q < k; q += 32) {
          const unsigned int mine_id = rec_id(__ldg(&rec[s + q].idx));
          unsigned int rank = 0;
          for (unsigned int o = 0; o < k; ++o) rank += rec_id(__ldg(&rec[s + o].idx)) < mine_id ? 1u : 0u;
          order[s + rank] = s + q;
        }
      }
      __syncwarp();  // skeys is reused by the next bucket
    }
  }
}

// The buckets the warp-per-cell kernel visits for the listed cells (window of the largest threshold, exactly the
// bucket range dsm_cell_kernel derives): one thread per listed cell.
__global__ void __launch_bounds__(256) dsm_mark_buckets_kernel(const __grid_constant__ DsmPlan plan,
                                                               const unsigned int* __restrict__ cell_list,
                                                               const unsigned int* __restrict__ counters,
                                                               unsigned char* __restrict__ flags) {
  // 64-bit cursor: a list can hold nearly 2^32 cells (amb_create), and a 32-bit c + stride would wrap past its end
  const size_t n_cells = counters[CTR_DSM_LIST];
  for (size_t c = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; c < n_cells;
       c += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const unsigned int cell = cell_list[c];
    const int i = static_cast<int>(cell % static_cast<unsigned int>(plan.rows));
    const int jl = static_cast<int>(cell / static_cast<unsigned int>(plan.rows));
    const BucketWindow w = bucket_window(plan, i + plan.Pa, plan.col_begin + jl - plan.gj0, plan.P);
    for (int kj = w.kbj0; kj <= w.kbj1; ++kj)
      for (int ki = w.kbi0; ki <= w.kbi1; ++ki) flags[static_cast<size_t>(kj) * plan.KR + ki] = 1;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// K4: tile gather, one block per TI x TJ tile: the records of the buckets overlapping the tile's window (the tile and W
// cells around it) are staged in shared memory by bin, then every thread evaluates a 1 x kStrip strip of cells.  Two
// kernels share the staging below: dsm_gather_kernel (dsm_gather_body.inc, all FP64, bins of one cell) and
// dsm_gather_kernel_f32 (dsm_gather_f32.inc, FP32 sums, bins of 1 x kBinJ cells; the default).
constexpr int kBinJ = kStrip;

struct GatherArgs {
  const unsigned int* G;   // bucket starts
  const PointRec* rec;
  float* elevation;
  unsigned int* cell_list;  // cells handed to the warp-per-cell kernel
  unsigned int* counters;   // amb::CounterSlot
  int* dbg_count;
  signed char* dbg_level;
  int capacity;  // points that fit the shared-memory stage
  int tiles_i;
};

// Shared-memory carve of a gather block (byte offsets into the dynamic shared memory), used by dsm_run to size the stage
// and by both kernels to place their arrays:
//   A[N + 2] | srow[n_bin_rows] | run_pre[max_runs + 1] | run_g0[max_runs] | pad to 16 B |  capacity x per_point
// A: per bin of the window, its count and then its start.  The staged points, FP64 (28 B): xy 16 | z 8 | original
// index 4.  FP32 (30 B): {x, z - z0, y, y} 16 | original index in bin order 4 | pass 1's compact lists of the kept
// records: HBM position 4 | original index 4 | bin 2.
struct GatherCarve {
  int NIw, NJw;    // window of the tile in cells
  int bin_j;       // cells per bin along j
  int N;           // bins of the window
  int n_bin_rows;  // bin rows a strip's window spans (window row 0 is bin-aligned)
  int srow, run_pre, run_g0;
  int table_bytes, per_point;
  int pts, z, sidx;     // z: FP64 only
  int ksrc, kid, klin;  // FP32 only
};
__host__ __device__ inline GatherCarve gather_carve(int W, int B, bool f32, int capacity) {
  GatherCarve c = {};
  c.NIw = TI + 2 * W;
  c.NJw = TJ + 2 * W;
  c.bin_j = f32 ? kBinJ : 1;
  c.N = c.NIw * ((c.NJw + c.bin_j - 1) / c.bin_j);
  c.n_bin_rows = (kStrip + 2 * W + c.bin_j - 1) / c.bin_j;
  const int max_runs = (c.NJw + B - 1) / B + 1;  // bucket rows overlapping the window
  c.srow = 4 * (c.N + 2);
  c.run_pre = c.srow + 4 * c.n_bin_rows;
  c.run_g0 = c.run_pre + 4 * (max_runs + 1);
  c.table_bytes = (c.run_g0 + 4 * max_runs + 15) & ~15;
  c.pts = c.table_bytes;
  if (f32) {
    c.per_point = 16 + 4 + 4 + 4 + 2;
    c.sidx = c.pts + 16 * capacity;
    c.ksrc = c.sidx + 4 * capacity;
    c.kid = c.ksrc + 4 * capacity;
    c.klin = c.kid + 4 * capacity;
  } else {
    c.per_point = 16 + 8 + 4;
    c.z = c.pts + 16 * capacity;
    c.sidx = c.z + 8 * capacity;
  }
  return c;
}

// The block's tile, its window in fine bins and the buckets overlapping the window.
struct GatherTile {
  int i0;                        // first row of the tile
  int gj;                        // global column of its first cell
  int jl0;                       // slab-local column of its first cell (negative if the tile starts left of the stripe)
  int wi0, wj0;                  // window origin in fine bins (>= 0: Pa >= W)
  int kbi0, kbi1, kbj0, n_runs;  // buckets: rows kbj0 .. kbj0 + n_runs - 1, each over bucket columns kbi0 .. kbi1
};
__device__ __forceinline__ GatherTile gather_tile(const DsmPlan& plan, const GatherArgs& args, const GatherCarve& c) {
  GatherTile t;
  t.i0 = static_cast<int>(blockIdx.x % args.tiles_i) * TI;
  t.gj = (plan.tile_j0 + static_cast<int>(blockIdx.x / args.tiles_i)) * TJ;
  t.jl0 = t.gj - plan.col_begin;
  t.wi0 = t.i0 + plan.Pa - plan.W;
  t.wj0 = t.gj - plan.gj0 - plan.W;
  t.kbi0 = t.wi0 >> plan.Bshift;
  t.kbi1 = min(t.wi0 + c.NIw - 1, plan.BR - 1) >> plan.Bshift;
  t.kbj0 = t.wj0 >> plan.Bshift;
  t.n_runs = (min(t.wj0 + c.NJw - 1, plan.BC - 1) >> plan.Bshift) - t.kbj0 + 1;
  return t;
}

// Tables of the tile (the caller's barrier publishes them):
//   run_pre / run_g0: one contiguous record run per bucket row of the window; run q holds the window's raw records
//     [run_pre[q], run_pre[q + 1]), starting at record run_g0[q].  Warp 0 fetches the bounds, one lane per bucket row,
//     and prefix-sums the lengths with a shuffle scan (no serial chain of dependent global loads).
//   srow[b]: half-width (in bins along i) of bin row b of a strip's window, the widest reach among its cell rows and the
//     strip's cells; -1: out of reach.
//   A: zeroed.
__device__ __forceinline__ void gather_tables(const DsmPlan& plan, const GatherArgs& args, const GatherCarve& c,
                                              const GatherTile& t) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned int* A = reinterpret_cast<unsigned int*>(smem_raw);
  int* srow = reinterpret_cast<int*>(smem_raw + c.srow);
  unsigned int* run_pre = reinterpret_cast<unsigned int*>(smem_raw + c.run_pre);
  unsigned int* run_g0 = reinterpret_cast<unsigned int*>(smem_raw + c.run_g0);
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    unsigned int carry = 0;
    for (int r0 = 0; r0 < t.n_runs; r0 += 32) {
      const int r = r0 + lane;
      unsigned int g0 = 0, len = 0;
      if (r < t.n_runs) {
        const size_t row = static_cast<size_t>(t.kbj0 + r) * plan.KR;
        g0 = __ldg(&args.G[row + t.kbi0]);
        len = __ldg(&args.G[row + t.kbi1 + 1]) - g0;
      }
      unsigned int inc = len;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned int v = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += v;
      }
      if (r < t.n_runs) {
        run_pre[r] = carry + inc - len;
        run_g0[r] = g0;
      }
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) run_pre[t.n_runs] = carry;
  }
  for (int b = threadIdx.x; b < c.n_bin_rows; b += kGatherThreads) {
    int hmax = -1;
    for (int rr = 0; rr < c.bin_j; ++rr) {
      const int r = b * c.bin_j + rr;  // cell row of the strip's window: (first cell's j) - W + r
      for (int m = 0; m < kStrip; ++m) {
        const int dj = r - plan.W - m;
        const int ad = dj < 0 ? -dj : dj;
        const int h = ad <= plan.W ? plan.hw[ad] : -1;
        hmax = max(hmax, h);
      }
    }
    srow[b] = hmax;
  }
  for (int e = threadIdx.x; e < c.N + 2; e += kGatherThreads) A[e] = 0;
}

// A raw record of the window: its position in HBM, its index word (PointRec::idx) and the window row of its bucket
// row's first fine bin row.
struct RawRecord {
  unsigned int src;
  int jrow;
  unsigned long long word;
};
// Locates raw record `raw` (< run_pre[n_runs]) and reads its index word.  Runs are about equally long, so the search
// starts at the proportional guess (raw * run_scale) >> 16, run_scale = (n_runs << 16) / n_in.  (Locating and binning
// are two calls so that a caller can keep several loads in flight before it bins.)
__device__ __forceinline__ RawRecord locate_record(const DsmPlan& plan, const GatherArgs& args, const GatherCarve& c,
                                                   const GatherTile& t, unsigned int run_scale, unsigned int raw) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const unsigned int* run_pre = reinterpret_cast<const unsigned int*>(smem_raw + c.run_pre);
  const unsigned int* run_g0 = reinterpret_cast<const unsigned int*>(smem_raw + c.run_g0);
  int run = min(static_cast<int>((raw * run_scale) >> 16), t.n_runs - 1);
  while (raw < run_pre[run]) --run;
  while (raw >= run_pre[run + 1]) ++run;
  RawRecord r;
  r.src = run_g0[run] + (raw - run_pre[run]);
  r.jrow = ((t.kbj0 + run) << plan.Bshift) - t.wj0;
  r.word = __ldg(&args.rec[r.src].idx);
  return r;
}
// Bin of the window a located record falls in, or -1 outside the window.  The binning stored the point's fine bin
// (fine_bin(), double precision) in the index word, so only integer arithmetic is left: bi = code >> 4, and bj's low
// bits are code & (B - 1) on top of the bucket row's first fine bin row.
__device__ __forceinline__ int record_bin(const DsmPlan& plan, const GatherCarve& c, const GatherTile& t,
                                          const RawRecord& r) {
  const unsigned int code = rec_code(r.word);
  const int ii = static_cast<int>(code >> 4) - t.wi0;
  const int jj = r.jrow + static_cast<int>(code & static_cast<unsigned int>(plan.B - 1));
  return ii >= 0 && ii < c.NIw && jj >= 0 && jj < c.NJw ? (jj / c.bin_j) * c.NIw + ii : -1;
}

// x, y, z of a record without its index word
__device__ __forceinline__ void load_xyz(const PointRec* src, double* x, double* y, double* z) {
#ifdef AMB_CUDA_EMU
  *x = src->x;
  *y = src->y;
  *z = src->z;
#else
  asm volatile("ld.global.nc.v2.f64 {%0, %1}, [%3];\n\tld.global.nc.f64 %2, [%3+16];"
               : "=d"(*x), "=d"(*y), "=d"(*z)
               : "l"(src));
#endif
}

// In-place inclusive scan of A[0 .. n) (thread t owns a contiguous chunk), then a barrier.
__device__ __forceinline__ void scan_bins(unsigned int* A, int n) {
  __shared__ unsigned int total;
  const int per = (n + kGatherThreads - 1) / kGatherThreads;
  const int lo = min(static_cast<int>(threadIdx.x) * per, n), hi = min(lo + per, n);
  unsigned int s = 0;
  for (int e = lo; e < hi; ++e) s += A[e];
  unsigned int run = block_exclusive_scan(s, &total);
  for (int e = lo; e < hi; ++e) {
    run += A[e];
    A[e] = run;
  }
  __syncthreads();
}

// Every cell of the tile goes to the warp-per-cell kernel (dense tile, non-finite heights ...).  The decision depends
// only on the point set the tile stages, which is the same for every striping of the map (tiles align to global
// columns, amb_dsm_halo_reach covers whole tile windows).
__device__ __forceinline__ void tile_to_cell_list(const DsmPlan& plan, const GatherArgs& args, const GatherTile& t) {
  if (threadIdx.x == 0) atomicAdd(&args.counters[CTR_DSM_DENSE], 1u);
  const int ti = threadIdx.x & 31, tq = threadIdx.x >> 5;
  for (int m = 0; m < kStrip; ++m) {
    const int i = t.i0 + ti, jl = t.jl0 + kStrip * tq + m;
    const bool valid = i < plan.rows && jl >= 0 && jl < plan.cols_slab;
    warp_append(valid, &args.counters[CTR_DSM_LIST], args.cell_list,
                static_cast<unsigned int>(static_cast<size_t>(jl) * plan.rows + i));
  }
}

#include "dsm_gather_body.inc"
#include "dsm_gather_f32.inc"

// ---------------------------------------------------------------------------------------------------------------
// K6: one warp per listed cell.  Evaluates the reference's complete per-cell sequence (primary query, then the
// expanding-radius retry dsm.cc:133-144) from the bucket records in HBM: cells left empty by the tile kernel and
// every cell of a tile too dense for the shared-memory stage.
struct CellArgs {
  const unsigned int* G;
  const unsigned int* order;  // canonical visiting order of the bucket records
  const PointRec* rec;
  float* elevation;
  const unsigned int* cell_list;
  unsigned int* counters;
  int* dbg_count;
  signed char* dbg_level;
};

__global__ void __launch_bounds__(256) dsm_cell_kernel(const __grid_constant__ DsmPlan plan, const CellArgs args) {
  const int lane = threadIdx.x & 31;
  const size_t n_cells = args.counters[CTR_DSM_LIST];
  const size_t warps_total = static_cast<size_t>(gridDim.x) * (blockDim.x >> 5);  // 64-bit cursor, as above
  for (size_t c = blockIdx.x * static_cast<size_t>(blockDim.x >> 5) + (threadIdx.x >> 5); c < n_cells; c += warps_total) {
    const unsigned int cell = args.cell_list[c];
    const int i = static_cast<int>(cell % static_cast<unsigned int>(plan.rows));
    const int jl = static_cast<int>(cell / static_cast<unsigned int>(plan.rows));
    const double qx = cell_x(plan, i);
    const double qy = cell_y(plan, plan.col_begin + jl);
    // buckets overlapping the window of the largest threshold (fine bins [b - P, b + P] on both axes)
    const BucketWindow w = bucket_window(plan, i + plan.Pa, plan.col_begin + jl - plan.gj0, plan.P);
    const double dmin = window_min_d2(plan, args.G, args.rec, w, qx, qy, lane);
    // first threshold whose (strict) ball is non-empty: k = 0 is the primary query itself
    int level = -1;
    for (int k = 0; k < plan.n_thr; ++k) {
      if (dmin < plan.thr[k]) {
        level = k;
        break;
      }
    }
    if (level < 0) {  // stays untouched (NaN or the previous elevation)
      if (args.dbg_count && lane == 0) {
        args.dbg_count[cell] = 0;
        args.dbg_level[cell] = -1;
      }
      continue;
    }
    const double thr = plan.thr[level];
    double num = 0.0, den = 0.0;
    int cnt = 0;
    bool coincident = false;
    // OrthoFromPcl: the zero-distance point with the LARGEST id, i.e. the last one the reference's loop would visit in
    // point order (ortho-from-pcl.cc:90-96 keeps the last perfect match; its kd-tree order is not reproducible here)
    long long match_idx = -1;
    double match_z = 0.0;
    for (int kj = w.kbj0; kj <= w.kbj1; ++kj) {
      const size_t row = static_cast<size_t>(kj) * plan.KR;
      const unsigned int a = args.G[row + w.kbi0];
      const unsigned int b = args.G[row + w.kbi1 + 1];
      for (unsigned int k = a + lane; k < b; k += 32) {
        const PointRec* pr = args.rec + __ldg(args.order + k);  // canonical order: lane partial sums are fixed
        const double2 v = __ldg(reinterpret_cast<const double2*>(pr));
        const double dx = qx - v.x;
        const double dy = qy - v.y;
        const double d2 = __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy));
        if (d2 < thr) {
          const double pz = __ldg(reinterpret_cast<const double*>(pr) + 2);
          ++cnt;
          if (d2 > 0.0) {
            const double w = fast_rcp(d2);
            num = fma(pz, w, num);
            den += w;
          } else {
            coincident = true;
            const long long id = static_cast<long long>(rec_id(__ldg(&pr->idx)));
            if (id > match_idx) {
              match_idx = id;
              match_z = pz;
            }
          }
        }
      }
    }
    for (int o = 16; o > 0; o >>= 1) {
      num += __shfl_xor_sync(0xffffffffu, num, o);
      den += __shfl_xor_sync(0xffffffffu, den, o);
      cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
      const long long oi = __shfl_xor_sync(0xffffffffu, match_idx, o);
      const double oz = __shfl_xor_sync(0xffffffffu, match_z, o);
      if (oi > match_idx) {
        match_idx = oi;
        match_z = oz;
      }
    }
    coincident = __any_sync(0xffffffffu, coincident);
    if (lane == 0) {
      if (coincident && plan.mode == 0) atomicExch(&args.counters[CTR_DSM_COINCIDENT], 1u);
      // OrthoFromPcl perfect match: numerator = that height, denominator = 1 (ortho-from-pcl.cc:90-96)
      const double value = (coincident && plan.mode == 1) ? match_z : __ddiv_rn(num, den);
      args.elevation[cell] = __double2float_rn(value);
      if (args.dbg_count) {
        args.dbg_count[cell] = cnt;
        args.dbg_level[cell] = static_cast<signed char>(level);
      }
    }
  }
}

// chunked evaluation: the list of the chunk just evaluated is done; keep its length for amb_get_timings
__global__ void roll_list_counter_kernel(unsigned int* counters) {
  counters[CTR_DSM_LIST_DONE] += counters[CTR_DSM_LIST];
  counters[CTR_DSM_LIST] = 0;
}

}  // namespace

double dsm_tile_reach_cells(double resolution, int32_t interpolation_radius) {
  const double slack = 1e-6;
  const int W = static_cast<int>(std::floor(std::sqrt(static_cast<double>(interpolation_radius)) / resolution + 0.5 + slack));
  return static_cast<double>(TJ + W + 1);
}

namespace {

// Half-width (in bins along i) of the window that can hold a point with d2 < thr, for a bin row |dj| away.
// A point binned to cell b lies within (0.5 + slack) cells of that cell's centre along each axis, so its
// distance along j to the query centre is at least (|dj| - 0.5 - slack) cells; what is left of the threshold
// bounds the reach along i.  -1: that bin row cannot contribute.
void half_widths(double thr, double res, int W, short* out) {
  const double slack = 1e-6;
  const double r = std::sqrt(thr) / res;  // reach in cells
  for (int dj = 0; dj <= kMaxHalfWidth; ++dj) {
    if (dj > W) {
      out[dj] = -1;
      continue;
    }
    const double dy = std::max(0.0, dj - 0.5 - slack);
    const double rem2 = r * r * (1.0 + 1e-12) - dy * dy;
    if (rem2 <= 0.0) {
      out[dj] = -1;
      continue;
    }
    int h = static_cast<int>(std::floor(std::sqrt(rem2) + 0.5 + slack));
    out[dj] = static_cast<short>(std::min(h, W));
  }
}

inline int round_up(int v, int m) { return ((v + m - 1) / m) * m; }

}  // namespace

// The border halo (halo_push.h) of a sharded cloud as separate arrays: coordinates, intensities (INTENSITIES, OrthoFromPcl)
// and ids.  Unordered append; order does not matter because every point carries its global id.
template <bool INTENSITIES>
__global__ void __launch_bounds__(256) halo_compact_kernel(const double* __restrict__ xyz,
                                                           const int* __restrict__ intensities,
                                                           const unsigned long long* __restrict__ ids, size_t n,
                                                           double y_lo, double y_hi, double reach, double shift_y,
                                                           double* __restrict__ out_xyz, int* __restrict__ out_intensities,
                                                           unsigned long long* __restrict__ out_ids,
                                                           unsigned int capacity, unsigned int* __restrict__ count) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n_round = ((n + stride - 1) / stride) * stride;  // whole warps stay converged for the ballot
  for (size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; t < n_round; t += stride) {
    bool take = false;
    double x = 0, y = 0, z = 0;
    int v = 0;
    if (t < n) {
      x = xyz[3 * t + 0];
      y = xyz[3 * t + 1];
      z = xyz[3 * t + 2];
      if (INTENSITIES) v = intensities[t];
      const BorderSides b = border_sides(y - shift_y, y_lo, y_hi, reach);
      take = b.up || b.down;
    }
    warp_reserve(take, count, [&](unsigned int slot) {
      if (slot >= capacity) return;
      out_xyz[3 * static_cast<size_t>(slot) + 0] = x;
      out_xyz[3 * static_cast<size_t>(slot) + 1] = y;
      out_xyz[3 * static_cast<size_t>(slot) + 2] = z;
      if (INTENSITIES) out_intensities[slot] = v;
      out_ids[slot] = ids ? ids[t] : static_cast<unsigned long long>(t);
    });
  }
}

int dsm_extract_halo(amb_ctx* ctx, const double* d_xyz, const unsigned long long* d_ids, size_t n, double y_lo,
                     double y_hi, double reach, double center_easting, double* d_out_xyz,
                     unsigned long long* d_out_ids, unsigned int capacity, unsigned int* d_count,
                     const int* d_intensities, int* d_out_intensities) {
  AMB_CUDA(ctx, cudaMemsetAsync(d_count, 0, sizeof(unsigned int), ctx->stream));
  if (d_intensities)  // OrthoFromPcl: no centre shift (ortho-from-pcl.cc bins the raw coordinates)
    halo_compact_kernel<true><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(d_xyz, d_intensities, d_ids, n, y_lo, y_hi,
                                                                          reach, 0.0, d_out_xyz, d_out_intensities,
                                                                          d_out_ids, capacity, d_count);
  else
    halo_compact_kernel<false><<<ctx->num_sms * 8, 256, 0, ctx->stream>>>(d_xyz, nullptr, d_ids, n, y_lo, y_hi, reach,
                                                                           center_easting, d_out_xyz, nullptr,
                                                                           d_out_ids, capacity, d_count);
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

int dsm_run(amb_ctx* ctx, const double* d_xyz, const unsigned long long* d_ids, size_t n,
            int32_t interpolation_radius, double center_easting, double center_northing, int mode,
            const int* d_intensities, const HaloSource* halo, const HaloPush* push, bool whole_map_bins) {
  const amb_geometry& g = ctx->geom;
  if (n == 0 && !halo) return AMB_ERR_EMPTY;
  // whole_map_bins (adaptive OrthoFromPcl on a stripe, pcl_adaptive_kernels.cu): bin the points into the bin grid of a
  // context owning the whole map — same bucket edge, same global bucket lattice — and stop after the binning.  The plan
  // left in last_dsm_plan keeps that grid but names this stripe's first column and width, so that its cells map into it.
  const int32_t col_begin = whole_map_bins ? 0 : ctx->col_begin;
  const int32_t col_end = whole_map_bins ? g.cols : ctx->col_end;
  const size_t n_own = n;
  // with halos: [own points | padding to a whole tile | halo slots] — an upper bound of the records this rank bins
  if (halo) n = ((n_own + 2047) / 2048) * 2048 + static_cast<size_t>(halo->nranks) * halo->capacity;
  if (interpolation_radius < 1 || n >= size_t(0xffffffffu)) return AMB_ERR_INVALID_ARGUMENT;
  const int out_layer = mode == 1 ? AMB_LAYER_ORTHO : AMB_LAYER_ELEVATION;  // ortho-from-pcl.cc:51 / dsm.cc:116
  int st = ensure_layer(ctx, out_layer);
  if (st != AMB_OK) return st;
  wait_layer_copy(ctx, out_layer);

  DsmPlan plan;
  std::memset(&plan, 0, sizeof(plan));
  plan.mode = mode;
  // Dsm: the retry thresholds of dsm.cc:133-144.  OrthoFromPcl without adaptive interpolation: the one query of
  // ortho-from-pcl.cc:57-60.
  const std::vector<double> thr = mode == 1 ? std::vector<double>(1, static_cast<double>(interpolation_radius))
                                            : dsm_thresholds(interpolation_radius);
  if (thr.size() > static_cast<size_t>(kMaxThresholds)) return AMB_ERR_UNSUPPORTED;
  double thr_max = 0.0;
  for (size_t k = 0; k < thr.size(); ++k) {
    plan.thr[k] = thr[k];
    thr_max = std::max(thr_max, thr[k]);
  }
  plan.n_thr = static_cast<int>(thr.size());
  plan.thr0 = static_cast<double>(interpolation_radius);
  plan.rows = g.rows;
  plan.cols_slab = col_end - col_begin;
  plan.col_begin = col_begin;
  plan.res = g.resolution;
  plan.inv_res = 1.0 / g.resolution;
  plan.base_x = g.pos_x + (0.5 * g.length_x - 0.5 * g.resolution);
  plan.base_y = g.pos_y + (0.5 * g.length_y - 0.5 * g.resolution);
  plan.shift_x = center_northing;  // dsm.cc:42 (sic)
  plan.shift_y = center_easting;   // dsm.cc:43
  const double slack = 1e-6;
  plan.W = static_cast<int>(std::floor(std::sqrt(plan.thr0) / g.resolution + 0.5 + slack));
  plan.P = static_cast<int>(std::floor(std::sqrt(thr_max) / g.resolution + 0.5 + slack));
  plan.P = std::max(plan.P, plan.W);
  if (plan.P > kMaxHalfWidth) return AMB_ERR_UNSUPPORTED;  // resolution far finer than the search radius
  if (g.rows >= (1 << 27)) return AMB_ERR_UNSUPPORTED;      // PointRec::idx keeps the fine bin row in 28 bits
  half_widths(plan.thr0, g.resolution, plan.W, plan.hw);

  // Bucket edge: a power of two (<= 16 cells) such that a bucket holds a few dozen points at the cloud's average
  // density over the map (the points actually binned may be fewer: that only makes buckets emptier).
  // With a sharded cloud `n` is only this rank's share: the caller then states the density of the whole cloud
  // (amb_dsm_set_density_hint), so that bucket size and stage capacity — which fix the summation orders — are the
  // same for every sharding of the same job.
  const double per_cell = ctx->dsm_density_hint > 0.0
                              ? ctx->dsm_density_hint
                              : static_cast<double>(n) / (static_cast<double>(g.rows) * static_cast<double>(g.cols));
  int B = 1, shift = 0;
  while (B < 16 && per_cell * (2.0 * B) * (2.0 * B) <= 48.0) {
    B *= 2;
    ++shift;
  }
  plan.B = B;
  plan.Bshift = shift;
  plan.Pa = round_up(plan.P, B);
  // Tiles align to GLOBAL columns (multiples of TJ), so that the content of a tile — hence the shared-memory /
  // warp-per-cell path decision and every summation order — does not depend on how the map is striped.
  plan.tile_j0 = col_begin / TJ;
  const int tile_j1 = (col_end - 1) / TJ;  // last tile column (inclusive)
  plan.gj0 = plan.tile_j0 * TJ - plan.Pa;
  plan.BR = round_up(round_up(g.rows, TI) + 2 * plan.Pa, B);
  plan.BC = round_up((tile_j1 + 1) * TJ + plan.Pa - plan.gj0, B);
  plan.KR = plan.BR / B;
  plan.KC = plan.BC / B;

  const size_t nbk = static_cast<size_t>(plan.KR) * plan.KC;
  const size_t g_elems = ((nbk + 2 + 3) / 4) * 4;  // uint4-aligned length
  const size_t n_vec = g_elems / 4;
  const int scan_blocks = static_cast<int>((n_vec + kScanChunk / 4 - 1) / (kScanChunk / 4));
  const size_t cells = ctx->slab_cells();

  AMB_CUDA(ctx, ctx->bin_starts.reserve(g_elems * sizeof(unsigned int)));
  AMB_CUDA(ctx, ctx->block_sums.reserve(static_cast<size_t>(scan_blocks) * sizeof(unsigned int)));
  AMB_CUDA(ctx, ctx->records.reserve(n * sizeof(PointRec)));
  AMB_CUDA(ctx, ctx->point_order.reserve(n * sizeof(unsigned int)));
  AMB_CUDA(ctx, ctx->bucket_flags.reserve(nbk));
  AMB_CUDA(ctx, ctx->empty_cells.reserve(cells * sizeof(unsigned int)));
  st = ensure_counters(ctx);
  if (st != AMB_OK) return st;
  if (ctx->dsm_debug) {
    AMB_CUDA(ctx, ctx->dbg_count.reserve(cells * sizeof(int)));
    AMB_CUDA(ctx, ctx->dbg_level.reserve(cells));
  }
  cudaStream_t s = ctx->stream;
  unsigned int* G = ctx->bin_starts.as<unsigned int>();
  unsigned int* counters = ctx->counters.as<unsigned int>();
  PointRec* rec = ctx->records.as<PointRec>();

  // the bins are rewritten from here on: until this call stores its plan they describe no plan
  ctx->last_dsm_plan.clear();
  ctx->last_bin_destinations = 0;
  AMB_CUDA(ctx, cudaMemsetAsync(G, 0, g_elems * sizeof(unsigned int), s));
  AMB_CUDA(ctx, cudaMemsetAsync(ctx->bucket_flags.ptr, 0, nbk, s));
  // only this stage's own slots: the sticky CHECK flags of earlier asynchronous calls stay until they are reported
  AMB_CUDA(ctx, cudaMemsetAsync(counters + CTR_DSM_LIST, 0, sizeof(unsigned int), s));
  AMB_CUDA(ctx, cudaMemsetAsync(counters + CTR_DSM_BINNED, 0, 4 * sizeof(unsigned int), s));  // [2..5]
  if (ctx->dsm_debug && !whole_map_bins) {
    AMB_CUDA(ctx, cudaMemsetAsync(ctx->dbg_count.ptr, 0xff, cells * sizeof(int), s));
    AMB_CUDA(ctx, cudaMemsetAsync(ctx->dbg_level.ptr, 0xff, cells, s));
  }
  if (!whole_map_bins) ctx->dsm_launches = 0;

  const int stream_grid = ctx->num_sms * 8;
  const HaloSource hs = halo ? *halo : HaloSource();
  // two-level binning (dsm_partition.inc): P1 bins, counts and groups every tile of points by coarse destination
  PartPlan pp;
  std::memset(&pp, 0, sizeof(pp));
  pp.n_own = n_own;
  pp.halo_base = halo ? ((n_own + kPartTile - 1) / kPartTile) * kPartTile : n_own;   // halo slots start a new tile
  pp.n_total = n;
  // a destination = a band of bucket columns whose final records span ~48 MB at a uniform density, about the H100's
  // 50 MB L2; at most kMaxCoarse bands.  Measured on an H100 SXM (80 GB, 400 W power limit) at 50 M points, whole binning
  // stage: 48 MB 4.69 ms, 32 MB 4.77 ms, 24 MB 4.87 ms, 16 MB 4.92 ms
  // (test knob AMB_DSM_PART_WINDOW: bytes per destination — small values exercise many destinations on small maps)
  static const size_t window_bytes = [] {
    const char* e = std::getenv("AMB_DSM_PART_WINDOW");
    const long long v = e ? std::atoll(e) : 0;
    return v > 0 ? static_cast<size_t>(v) : size_t(48) << 20;
  }();
  int S = static_cast<int>(std::min<size_t>((n * sizeof(PointRec) + window_bytes - 1) / window_bytes, kMaxCoarse));
  S = std::max(1, std::min(S, plan.KC));
  pp.kj_per = (plan.KC + S - 1) / S;
  pp.S = (plan.KC + pp.kj_per - 1) / pp.kj_per;
  pp.n_tiles = static_cast<unsigned int>((n + kPartTile - 1) / kPartTile);
  pp.n_groups = (pp.n_tiles + kFineTilesPerBlock - 1) / kFineTilesPerBlock;
  AMB_CUDA(ctx, ctx->records_tmp.reserve(static_cast<size_t>(pp.n_tiles) * kPartTile * sizeof(PointRec)));
  AMB_CUDA(ctx, ctx->tile_offsets.reserve(static_cast<size_t>(pp.S + 1) * pp.n_tiles * sizeof(unsigned short)));
  {
    PointRec* tmp = ctx->records_tmp.as<PointRec>();
    unsigned short* offs = ctx->tile_offsets.as<unsigned short>();
    const unsigned int own_tiles = static_cast<unsigned int>(pp.halo_base / kPartTile);
    const unsigned int max_grid = static_cast<unsigned int>(ctx->num_sms) * 4u;
    AMB_CUDA(ctx, cudaFuncSetAttribute(dsm_partition_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       kPartStageBytes));
    if (push) {
      // peer-push exchange (amb_comm.cu): the own points are binned first and their border records stored into the
      // adjacent ranks' segments on the way; the incoming halos — the tiles after halo_base — follow once both neighbours
      // have published theirs.  (At least one block even without own points: it publishes the empty lists.)
      pp.tile_begin = 0;
      pp.tile_end = own_tiles;
      AMB_CUDA(ctx, cudaFuncSetAttribute(dsm_partition_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         kPartStageBytes));
      dsm_partition_kernel<true><<<std::max(1u, std::min(own_tiles, max_grid)), kPartThreads, kPartStageBytes, s>>>(
          d_xyz, d_intensities, d_ids, plan, pp, G, tmp, offs, counters, hs, *push);
      st = halo_wait_launch(ctx, *push);
      if (st != AMB_OK) return st;
      // timings: the "halo" interval of a peer-push step ends here (own points binned + pushed, neighbours' halos arrived)
      AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_H2D_END], s));
      pp.tile_begin = own_tiles;
      pp.tile_end = pp.n_tiles;
      if (pp.tile_end > pp.tile_begin)
        dsm_partition_kernel<false><<<std::min(pp.tile_end - pp.tile_begin, max_grid), kPartThreads, kPartStageBytes, s>>>(
            d_xyz, d_intensities, d_ids, plan, pp, G, tmp, offs, counters, hs, HaloPush());
      ctx->dsm_launches += 2;
    } else {
      pp.tile_begin = 0;
      pp.tile_end = pp.n_tiles;
      dsm_partition_kernel<false><<<std::min(pp.n_tiles, max_grid), kPartThreads, kPartStageBytes, s>>>(
          d_xyz, d_intensities, d_ids, plan, pp, G, tmp, offs, counters, hs, HaloPush());
    }
  }
  scan_reduce_kernel<<<scan_blocks, 256, 0, s>>>(reinterpret_cast<const uint4*>(G), n_vec,
                                                 ctx->block_sums.as<unsigned int>());
  scan_spine_kernel<<<1, 1024, 0, s>>>(ctx->block_sums.as<unsigned int>(), scan_blocks);
  scan_apply_kernel<<<scan_blocks, 256, 0, s>>>(reinterpret_cast<uint4*>(G), n_vec,
                                                ctx->block_sums.as<unsigned int>());
  dsm_fine_scatter_kernel<<<static_cast<unsigned int>(pp.S) * pp.n_groups, kFineThreads, 0, s>>>(
      plan, pp, ctx->records_tmp.as<PointRec>(), ctx->tile_offsets.as<unsigned short>(), G, rec);
  ctx->last_bin_destinations = pp.S;
  // Canonical order inside the buckets: Dsm orders only the buckets its warp-per-cell kernel will read (marked from the
  // cell list after the gather); OrthoFromPcl's adaptive pass may read any bucket, so that mode orders all of them here.
  unsigned char* bucket_flags = ctx->bucket_flags.as<unsigned char>();
  if (mode == 1) {
    dsm_bucket_order_kernel<<<stream_grid, 256, 0, s>>>(G, static_cast<unsigned int>(nbk), rec,
                                                        ctx->point_order.as<unsigned int>(), nullptr);
    ctx->dsm_launches += 1;
  }
  ctx->dsm_launches += 5;
  if (whole_map_bins) {
    AMB_CUDA(ctx, cudaGetLastError());
    plan.col_begin = ctx->col_begin;
    plan.cols_slab = ctx->col_end - ctx->col_begin;
    ctx->last_dsm_plan.assign(reinterpret_cast<const unsigned char*>(&plan),
                              reinterpret_cast<const unsigned char*>(&plan) + sizeof(plan));
    return AMB_OK;
  }
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_BIN_END], s));

  // gather
  // FP32 gather (the default; amb_dsm_set_precision): Dsm only — OrthoFromPcl keeps the all-FP64 kernel
  const bool f32 = ctx->dsm_precision == AMB_DSM_F32 && mode == 0;
  const GatherCarve carve = gather_carve(plan.W, B, f32, 0);
  const size_t off_bytes = static_cast<size_t>(carve.table_bytes), per_point = static_cast<size_t>(carve.per_point);
  {
    // Bound on |d2_f32 - d2| (dsm_gather_f32.inc): local coordinates |c| <= M are rounded to float (relative u = 2^-24),
    // the difference adds one rounding, the two squares and the sum three more:
    //   |d(dx)| <= 2uM + u|dx|,   |d(d2)| <= 2(|dx| + |dy|)(2uM + u sqrt(d2)) + 3u d2,   |dx| + |dy| <= sqrt(2 d2)
    // evaluated at d2 = thr0 (+ the band itself) with a safety factor of 2.
    const double u = 5.9604644775390625e-8;
    const double M = (TI / 2 + plan.W + 2) * g.resolution;
    const double t = plan.thr0 * 1.01;
    const double bound = 2.0 * std::sqrt(2.0 * t) * (2.0 * u * M + u * std::sqrt(t)) + 3.0 * u * t;
    plan.thr_f = static_cast<float>(plan.thr0);
    plan.eps_f = static_cast<float>(2.0 * bound);
    plan.zrange_limit = 4096.0;
    // the same rounding as a distance vector: |d(dx)|, |d(dy)| <= 2uM + u |d_f|  =>  |v_f - v| <= 2 sqrt(2) u M + u |v_f|
    plan.hdelta = static_cast<float>(2.0 * std::sqrt(2.0) * u * M * (1.0 + 1e-6));
    plan.hden_max = static_cast<float>(std::pow((0.01 - u) / (plan.hdelta * (1.0 + 3.0 * u)), 2.0) * (1.0 - 1e-6));
  }
  // Stage size: 1.6x the expected number of points in a tile window under a uniform density (the tail of a
  // Poisson count is far inside that; denser tiles go to the warp-per-cell kernel), clamped to [24 KB, 100 KB]
  // so that several blocks stay resident per SM (227 KB usable).
  if (off_bytes + per_point * 64 > 200 * 1024) return AMB_ERR_UNSUPPORTED;
  const double expect = per_cell * static_cast<double>(carve.NIw) * static_cast<double>(carve.NJw);
  size_t smem = off_bytes + static_cast<size_t>((f32 ? 1.4 : 1.6) * expect + 64.0) * per_point;
  smem = std::min<size_t>(std::max<size_t>(smem, 24 * 1024), 100 * 1024);
  smem = std::max(smem, off_bytes + per_point * 64);
  smem = (smem + 1023) & ~static_cast<size_t>(1023);
  const int capacity = static_cast<int>((smem - off_bytes) / per_point) & ~1;
  void (*const gather)(DsmPlan, GatherArgs) = f32 ? dsm_gather_kernel_f32 : dsm_gather_kernel;
  AMB_CUDA(ctx, cudaFuncSetAttribute(gather, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem)));
  GatherArgs ga;
  ga.G = G;
  ga.rec = rec;
  ga.elevation = ctx->layers[out_layer];
  ga.cell_list = ctx->empty_cells.as<unsigned int>();
  ga.counters = counters;
  ga.dbg_count = ctx->dsm_debug ? ctx->dbg_count.as<int>() : nullptr;
  ga.dbg_level = ctx->dsm_debug ? ctx->dbg_level.as<signed char>() : nullptr;
  ga.capacity = capacity;
  ga.tiles_i = (plan.rows + TI - 1) / TI;
  CellArgs ca;
  ca.G = G;
  ca.order = ctx->point_order.as<unsigned int>();
  ca.rec = rec;
  ca.elevation = ga.elevation;
  ca.cell_list = ga.cell_list;
  ca.counters = counters;
  ca.dbg_count = ga.dbg_count;
  ca.dbg_level = ga.dbg_level;
  const int tiles_j = tile_j1 - plan.tile_j0 + 1;
  // Opt-in chunking (amb_dsm_set_stream_chunks, only with a registered host mirror): the tile columns are evaluated in K
  // groups — gather + warp-per-cell fill per group — and each group's finished columns start travelling to the host
  // at once, so the download of the layer overlaps the evaluation of the remaining groups.  The launches of a group are
  // the un-chunked ones restricted to its tile columns (plan.tile_j0 and the grid size), so every result is unchanged.
  // (Dsm only: OrthoFromPcl's adaptive pass rewrites the layer afterwards, so its columns are not final per chunk)
  // Without chunking the whole stripe is one group.
  const int chunks = (mode == 0 && ctx->dsm_stream_chunks > 1 && ctx->host_mirror[out_layer])
                         ? std::min(ctx->dsm_stream_chunks, tiles_j) : 1;
  for (int c = 0; c < chunks; ++c) {
    const int tj0 = static_cast<int>(static_cast<long long>(tiles_j) * c / chunks);
    const int tj1 = static_cast<int>(static_cast<long long>(tiles_j) * (c + 1) / chunks);
    if (tj1 <= tj0) continue;
    DsmPlan pc = plan;
    pc.tile_j0 = plan.tile_j0 + tj0;
    if (c > 0) roll_list_counter_kernel<<<1, 1, 0, s>>>(counters);  // the cell list restarts; its length is kept
    gather<<<ga.tiles_i * (tj1 - tj0), kGatherThreads, smem, s>>>(pc, ga);
    if (chunks == 1) AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_GATHER_END], s));
    if (mode == 0) {
      dsm_mark_buckets_kernel<<<ctx->num_sms * 2, 256, 0, s>>>(pc, ga.cell_list, counters, bucket_flags);
      dsm_bucket_order_kernel<<<stream_grid, 256, 0, s>>>(G, static_cast<unsigned int>(nbk), rec,
                                                          ctx->point_order.as<unsigned int>(), bucket_flags);
      ctx->dsm_launches += 2;
    }
    dsm_cell_kernel<<<ctx->num_sms * 8, 256, 0, s>>>(pc, ca);
    ctx->dsm_launches += 2;
    if (chunks > 1) {
      // slab-local columns of this group's tiles (tiles are aligned to GLOBAL columns)
      const int col0 = std::max((plan.tile_j0 + tj0) * TJ - ctx->col_begin, 0);
      const int col1 = std::min((plan.tile_j0 + tj1) * TJ - ctx->col_begin, ctx->col_end - ctx->col_begin);
      st = mirror_layer_columns(ctx, out_layer, col0, col1);
      if (st != AMB_OK) return st;
    }
  }
  // chunked: the stage split is not meaningful, both events mark the end
  if (chunks > 1) AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_GATHER_END], s));
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_FILL_END], s));
  AMB_CUDA(ctx, cudaGetLastError());
  if (chunks == 1) {
    st = mirror_layer(ctx, out_layer);  // the result starts streaming to its host mirror (if one is registered)
    if (st != AMB_OK) return st;
  }
  ctx->dsm_debug_valid = ctx->dsm_debug;
  ctx->last_dsm_plan.assign(reinterpret_cast<const unsigned char*>(&plan),
                            reinterpret_cast<const unsigned char*>(&plan) + sizeof(plan));
  return AMB_OK;
}

}  // namespace amb
