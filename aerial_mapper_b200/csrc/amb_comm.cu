// amb_comm.cu — the one exchange step of the path inside the library (SURVEY.md §8e): a context can join an NCCL
// communicator (one process per GPU, or several contexts of one process), and amb_dsm_process_sharded_device (and
// amb_ortho_from_pcl_process_sharded_device, whose records carry the intensities as z) runs
//     border-halo compaction  ->  ONE ncclAllGather of the halos  ->  binning over [own points | neighbours' halos]
// entirely on the context's stream: no host synchronisation, no framework plumbing, device-side counts.
//
// NCCL is loaded at run time (dlopen "libnccl.so.2"): the library keeps depending on the CUDA runtime only, a process
// that already carries an NCCL (e.g. PyTorch's bundled one) shares it, and single-GPU users never need it.
#include <dlfcn.h>
#include <unistd.h>

#include <algorithm>
#include <cstdlib>
#include <mutex>

#include "amb_context.h"
#include "dsm_plan.h"
#include "halo_push.h"

namespace amb {

// ---- the few NCCL entry points used, declared locally (ABI-stable since NCCL 2.0) ----
struct NcclUniqueId {
  char internal[128];
};
typedef void* nccl_comm_t;
typedef int (*nccl_get_unique_id_fn)(NcclUniqueId*);
typedef int (*nccl_comm_init_rank_fn)(nccl_comm_t*, int, NcclUniqueId, int);
typedef int (*nccl_comm_destroy_fn)(nccl_comm_t);
typedef int (*nccl_all_gather_fn)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t);
typedef int (*nccl_send_fn)(const void*, size_t, int, int, nccl_comm_t, cudaStream_t);
typedef int (*nccl_recv_fn)(void*, size_t, int, int, nccl_comm_t, cudaStream_t);
typedef int (*nccl_group_fn)(void);
typedef const char* (*nccl_error_string_fn)(int);
constexpr int kNcclInt8 = 0;  // ncclInt8 / ncclChar

struct NcclApi {
  void* handle = nullptr;
  nccl_get_unique_id_fn get_unique_id = nullptr;
  nccl_comm_init_rank_fn comm_init_rank = nullptr;
  nccl_comm_destroy_fn comm_destroy = nullptr;
  nccl_all_gather_fn all_gather = nullptr;
  nccl_send_fn send = nullptr;
  nccl_recv_fn recv = nullptr;
  nccl_group_fn group_start = nullptr, group_end = nullptr;
  nccl_error_string_fn error_string = nullptr;
  bool ok = false;
};

static NcclApi& nccl() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
#ifndef AMB_CUDA_EMU
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      api.handle = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (api.handle) break;
    }
    if (!api.handle) return;
    api.get_unique_id = reinterpret_cast<nccl_get_unique_id_fn>(dlsym(api.handle, "ncclGetUniqueId"));
    api.comm_init_rank = reinterpret_cast<nccl_comm_init_rank_fn>(dlsym(api.handle, "ncclCommInitRank"));
    api.comm_destroy = reinterpret_cast<nccl_comm_destroy_fn>(dlsym(api.handle, "ncclCommDestroy"));
    api.all_gather = reinterpret_cast<nccl_all_gather_fn>(dlsym(api.handle, "ncclAllGather"));
    api.send = reinterpret_cast<nccl_send_fn>(dlsym(api.handle, "ncclSend"));
    api.recv = reinterpret_cast<nccl_recv_fn>(dlsym(api.handle, "ncclRecv"));
    api.group_start = reinterpret_cast<nccl_group_fn>(dlsym(api.handle, "ncclGroupStart"));
    api.group_end = reinterpret_cast<nccl_group_fn>(dlsym(api.handle, "ncclGroupEnd"));
    api.error_string = reinterpret_cast<nccl_error_string_fn>(dlsym(api.handle, "ncclGetErrorString"));
    api.ok = api.get_unique_id && api.comm_init_rank && api.comm_destroy && api.all_gather && api.group_start &&
             api.group_end && api.send && api.recv;
#endif
  });
  return api;
}

static int nccl_fail(amb_ctx* ctx, int rc, const char* what) {
  if (ctx) {
    const char* msg = nccl().error_string ? nccl().error_string(rc) : "?";
    ctx->last_error = std::string(what) + ": NCCL error " + std::to_string(rc) + " (" + msg + ")";
  }
  return AMB_ERR_CUDA;
}

// Border halo of a sharded cloud as 32-byte records {x, y, z, id} behind a 32-byte header {count, ...}: exactly what the
// binning kernels of every rank read after the all-gather.  Unordered append (warp-aggregated atomic): order does not
// matter, every point carries its global id.
// seg_up / seg_down: two segments (header + records).  A point near the stripe's LOW-column border (large y) goes to
// seg_up — what the previous rank needs — one near the HIGH-column border to seg_down; with `split` = false everything
// goes to seg_up (the all-gather exchange delivers one list per rank to everybody).
__device__ __forceinline__ void halo_append(bool take, int lane, unsigned char* seg, unsigned int capacity, double x,
                                            double y, double z, unsigned long long id) {
  const unsigned int mask = __ballot_sync(0xffffffffu, take);
  if (!mask) return;
  const int leader = __ffs(mask) - 1;
  unsigned int base = 0;
  if (lane == leader) base = atomicAdd(reinterpret_cast<unsigned int*>(seg), static_cast<unsigned int>(__popc(mask)));
  base = __shfl_sync(0xffffffffu, base, leader);
  if (take) {
    const unsigned int slot = base + __popc(mask & ((1u << lane) - 1u));
    if (slot < capacity) {
      double* r = reinterpret_cast<double*>(seg + 32) + 4 * static_cast<size_t>(slot);
      r[0] = x;
      r[1] = y;
      r[2] = z;
      r[3] = __longlong_as_double(static_cast<long long>(id));
    }
  }
}

// INTENSITIES (OrthoFromPcl): the record's z is double(intensities[t]), what that pass bins (ortho-from-pcl.cc:33)
template <bool INTENSITIES>
__device__ __forceinline__ void halo_records(const double* __restrict__ xyz, const int* __restrict__ intensities,
                                             const unsigned long long* __restrict__ ids, size_t n, double y_lo,
                                             double y_hi, double reach, double shift_y, unsigned char* seg_up,
                                             unsigned char* seg_down, bool split, unsigned int capacity) {
  const int lane = threadIdx.x & 31;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n_round = ((n + stride - 1) / stride) * stride;  // whole warps stay converged for the ballots
  for (size_t t = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; t < n_round; t += stride) {
    bool up = false, down = false;
    double x = 0, y = 0, z = 0;
    unsigned long long id = 0;
    if (t < n) {
      y = xyz[3 * t + 1];
      const double ys = y - shift_y;
      up = ys > y_hi - reach;    // column 0 is the max-y side: the previous rank's stripe lies beyond y_hi
      down = ys < y_lo + reach;
      if (up || down) {
        x = xyz[3 * t + 0];
        z = INTENSITIES ? static_cast<double>(intensities[t]) : xyz[3 * t + 2];
        id = ids ? ids[t] : static_cast<unsigned long long>(t);
      }
    }
    if (split) {
      halo_append(up, lane, seg_up, capacity, x, y, z, id);
      halo_append(down, lane, seg_down, capacity, x, y, z, id);
    } else {
      halo_append(up || down, lane, seg_up, capacity, x, y, z, id);
    }
  }
}

__global__ void __launch_bounds__(256) dsm_halo_records_kernel(const double* __restrict__ xyz,
                                                               const unsigned long long* __restrict__ ids, size_t n,
                                                               double y_lo, double y_hi, double reach, double shift_y,
                                                               unsigned char* seg_up, unsigned char* seg_down, bool split,
                                                               unsigned int capacity) {
  halo_records<false>(xyz, nullptr, ids, n, y_lo, y_hi, reach, shift_y, seg_up, seg_down, split, capacity);
}

__global__ void __launch_bounds__(256) pcl_halo_records_kernel(const double* __restrict__ xyz,
                                                               const int* __restrict__ intensities,
                                                               const unsigned long long* __restrict__ ids, size_t n,
                                                               double y_lo, double y_hi, double reach,
                                                               unsigned char* seg_up, unsigned char* seg_down, bool split,
                                                               unsigned int capacity) {
  halo_records<true>(xyz, intensities, ids, n, y_lo, y_hi, reach, 0.0, seg_up, seg_down, split, capacity);
}


// ---- fused compaction + transfer over NVLink peer memory (exchange mode "peer push") -------------------------------
// With consecutive stripes each at least `reach` wide a rank's border points are needed by its two adjacent ranks only.
// Instead of a compaction pass over the rank's points followed by ncclSend/ncclRecv (a second read of the cloud, a second
// kernel, NCCL's launch and rendezvous latency, which do not shrink with the halo's size),
// the binning's own partition kernel (dsm_partition.inc, which reads every point anyway) stores every border record
// STRAIGHT INTO THE NEIGHBOUR'S receive segment (its cudaMalloc'ed buffer, mapped here with cudaIpcOpenMemHandle: the
// stores travel over NVLink / NVSwitch as they are produced), counts with local atomics, and its last block publishes
// {count, step stamp} in the neighbour's segment header with a system-scope release (halo_push.h).  The consumer runs
// halo_wait_kernel in front of the binning of the incoming halos: two lanes spin (acquire, system scope) until both
// headers carry this step's stamp.  Segments are double-buffered by step parity: a rank can only be two steps
// ahead of a neighbour after having received that neighbour's halo of the step in between, which the neighbour sends
// after it has finished reading the earlier one (stream order) — so a segment is never overwritten while it is read.
//
// Lane 0 / 1: wait until the header of the segment filled by rank - 1 / rank + 1 carries this step's stamp.
// Bounded (about twenty seconds of polling — far beyond any legitimate skew between ranks): a neighbour that never arrives
// raises the sticky halo flag instead of hanging the GPU.
__global__ void halo_wait_kernel(const unsigned char* seg_prev, const unsigned char* seg_next, unsigned int stamp,
                                 unsigned int* counters) {
  const unsigned char* seg = threadIdx.x == 0 ? seg_prev : seg_next;
  if (threadIdx.x > 1 || !seg) return;
  const long long t0 = clock64();
  for (;;) {
    const unsigned long long h = load_acquire_sys(seg);
    if (static_cast<unsigned int>(h >> 32) == stamp) return;
    if (clock64() - t0 > 40000000000ll) {
      atomicExch(&counters[CTR_HALO_OVERFLOW], 1u);
      return;
    }
    __nanosleep(200);
  }
}

}  // namespace amb

namespace amb {

int halo_wait_launch(amb_ctx* ctx, const HaloPush& push) {
  const int st = ensure_counters(ctx);
  if (st != AMB_OK) return st;
  halo_wait_kernel<<<1, 32, 0, ctx->stream>>>(push.wait_prev, push.wait_next, push.stamp, ctx->counters.as<unsigned int>());
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

// Blob every rank contributes to the handle exchange of the peer-push halo.
struct PeerBlob {
  cudaIpcMemHandle_t handle;
  long long pid;
  unsigned long long raw_ptr;  // same-process contexts: the pointer itself
  int device;
  int ok;
};

static void peer_halo_release(amb_ctx* ctx) {
  HaloPeer& hp = ctx->halo_peer;
  if (hp.prev && hp.prev_ipc) cudaIpcCloseMemHandle(hp.prev);
  if (hp.next && hp.next_ipc) cudaIpcCloseMemHandle(hp.next);
  hp.prev = hp.next = nullptr;
  hp.prev_ipc = hp.next_ipc = false;
  if (hp.recv) cudaFree(hp.recv);
  if (hp.counters) cudaFree(hp.counters);
  hp.recv = nullptr;
  hp.counters = nullptr;
  hp.side_capacity = 0;
  hp.enabled = false;
}

// (Re)allocate this rank's receive segments for `side_capacity` records per side and map the two neighbours'.
// COLLECTIVE (one small ncclAllGather + a host synchronisation): runs on the first sharded call and whenever the
// capacity grows — every rank passes the same halo_capacity, so every rank takes this branch in the same call.
// On any failure anywhere, every rank agrees to keep the NCCL exchange.
static int peer_halo_setup(amb_ctx* ctx, uint32_t side_capacity) {
  HaloPeer& hp = ctx->halo_peer;
  cudaStream_t s = ctx->stream;
  const int nranks = ctx->comm_size, rank = ctx->comm_rank;
  AMB_CUDA(ctx, cudaStreamSynchronize(s));  // this rank no longer reads its segments nor writes its neighbours'
  // A neighbour may still be pushing into this rank's OLD segments (it reaches this collective later): on a re-setup
  // (larger capacity) they are retired, not freed — amb_comm_destroy frees them.
  if (hp.recv) {
    hp.retired.push_back(hp.recv);
    hp.retired.push_back(reinterpret_cast<unsigned char*>(hp.counters));
    hp.recv = nullptr;
    hp.counters = nullptr;
  }
  peer_halo_release(ctx);
  hp.tried = true;
  const size_t side_bytes = 32 * (static_cast<size_t>(side_capacity) + 1);
  PeerBlob mine;
  std::memset(&mine, 0, sizeof(mine));
  mine.pid = static_cast<long long>(getpid());
  mine.device = ctx->device;
  mine.ok = 1;
  if (cudaMalloc(reinterpret_cast<void**>(&hp.recv), 4 * side_bytes) != cudaSuccess ||
      cudaMalloc(reinterpret_cast<void**>(&hp.counters), 2 * 4 * sizeof(unsigned int)) != cudaSuccess ||
      cudaMemset(hp.recv, 0, 4 * side_bytes) != cudaSuccess ||
      cudaMemset(hp.counters, 0, 2 * 4 * sizeof(unsigned int)) != cudaSuccess ||
      cudaIpcGetMemHandle(&mine.handle, hp.recv) != cudaSuccess) {
    cudaGetLastError();
    mine.ok = 0;
  }
  mine.raw_ptr = reinterpret_cast<unsigned long long>(hp.recv);
  DeviceBuffer tmp;
  AMB_CUDA(ctx, tmp.reserve(sizeof(PeerBlob) * (static_cast<size_t>(nranks) + 1)));
  unsigned char* d = tmp.as<unsigned char>();
  std::vector<PeerBlob> all(static_cast<size_t>(nranks));
  AMB_CUDA(ctx, cudaMemcpyAsync(d, &mine, sizeof(mine), cudaMemcpyHostToDevice, s));
  int rc = nccl().all_gather(d, d + sizeof(PeerBlob), sizeof(PeerBlob), kNcclInt8,
                             static_cast<nccl_comm_t>(ctx->nccl_comm), s);
  if (rc != 0) return nccl_fail(ctx, rc, "ncclAllGather(peer halo handles)");
  AMB_CUDA(ctx, cudaMemcpyAsync(all.data(), d + sizeof(PeerBlob), sizeof(PeerBlob) * nranks, cudaMemcpyDeviceToHost, s));
  AMB_CUDA(ctx, cudaStreamSynchronize(s));
  int ok = 1;
  for (int r = 0; r < nranks; ++r) ok &= all[r].ok;
  auto map_peer = [&](int r, unsigned char** out, bool* ipc) {
    const PeerBlob& b = all[r];
    if (b.pid == mine.pid) {  // another context of this process: plain peer access
      if (b.device != ctx->device) {
        const cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) return false;
        cudaGetLastError();
      }
      *out = reinterpret_cast<unsigned char*>(b.raw_ptr);
      *ipc = false;
      return true;
    }
    void* p = nullptr;
    if (cudaIpcOpenMemHandle(&p, b.handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
      cudaGetLastError();
      return false;
    }
    *out = static_cast<unsigned char*>(p);
    *ipc = true;
    return true;
  };
  if (ok && rank > 0 && !map_peer(rank - 1, &hp.prev, &hp.prev_ipc)) ok = 0;
  if (ok && rank < nranks - 1 && !map_peer(rank + 1, &hp.next, &hp.next_ipc)) ok = 0;
  // second round: everybody mapped its neighbours?
  int* flag = reinterpret_cast<int*>(d);
  std::vector<int> flags(static_cast<size_t>(nranks), 0);
  AMB_CUDA(ctx, cudaMemcpyAsync(flag, &ok, sizeof(int), cudaMemcpyHostToDevice, s));
  rc = nccl().all_gather(flag, flag + 1, sizeof(int), kNcclInt8, static_cast<nccl_comm_t>(ctx->nccl_comm), s);
  if (rc != 0) return nccl_fail(ctx, rc, "ncclAllGather(peer halo status)");
  AMB_CUDA(ctx, cudaMemcpyAsync(flags.data(), flag + 1, sizeof(int) * nranks, cudaMemcpyDeviceToHost, s));
  AMB_CUDA(ctx, cudaStreamSynchronize(s));
  tmp.release();
  for (int r = 0; r < nranks; ++r) ok &= flags[r];
  if (!ok) {
    peer_halo_release(ctx);
    hp.tried = true;
    return AMB_OK;  // the NCCL exchange stays in charge
  }
  hp.side_capacity = side_capacity;
  hp.enabled = true;
  hp.step = 0;
  return AMB_OK;
}

}  // namespace amb

using namespace amb;

extern "C" {

int amb_comm_unique_id(void* id128) {
  if (!id128) return AMB_ERR_INVALID_ARGUMENT;
  if (!nccl().ok) return AMB_ERR_UNSUPPORTED;
  NcclUniqueId id;
  const int rc = nccl().get_unique_id(&id);
  if (rc != 0) return AMB_ERR_CUDA;
  std::memcpy(id128, &id, sizeof(id));
  return AMB_OK;
}

int amb_comm_init(amb_ctx* ctx, int rank, int nranks, const void* id128) {
  if (!ctx || !id128 || nranks < 1 || rank < 0 || rank >= nranks) return AMB_ERR_INVALID_ARGUMENT;
  if (ctx->nccl_comm) return AMB_ERR_INVALID_ARGUMENT;  // already a member
  if (!nccl().ok) {
    ctx->last_error = "libnccl.so.2 could not be loaded (dlopen)";
    return AMB_ERR_UNSUPPORTED;
  }
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  NcclUniqueId id;
  std::memcpy(&id, id128, sizeof(id));
  nccl_comm_t comm = nullptr;
  const int rc = nccl().comm_init_rank(&comm, nranks, id, rank);
  if (rc != 0) return nccl_fail(ctx, rc, "ncclCommInitRank");
  ctx->nccl_comm = comm;
  ctx->comm_rank = rank;
  ctx->comm_size = nranks;
  // every member learns every stripe (decides, identically on all ranks, whether the halo step may talk to the two
  // neighbours only)
  {
    DeviceBuffer tmp;
    AMB_CUDA(ctx, tmp.reserve(2 * sizeof(int32_t) * (static_cast<size_t>(nranks) + 1)));
    int32_t mine[2] = {ctx->col_begin, ctx->col_end};
    int32_t* d = tmp.as<int32_t>();
    AMB_CUDA(ctx, cudaMemcpyAsync(d, mine, sizeof(mine), cudaMemcpyHostToDevice, ctx->stream));
    const int rc2 = nccl().all_gather(d, d + 2, sizeof(mine), kNcclInt8, comm, ctx->stream);
    if (rc2 != 0) {
      tmp.release();
      return nccl_fail(ctx, rc2, "ncclAllGather(stripes)");
    }
    ctx->comm_stripes.assign(2 * static_cast<size_t>(nranks), 0);
    AMB_CUDA(ctx, cudaMemcpyAsync(ctx->comm_stripes.data(), d + 2, 2 * sizeof(int32_t) * nranks, cudaMemcpyDeviceToHost,
                                  ctx->stream));
    AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    tmp.release();
  }
  return AMB_OK;
}

int amb_comm_set_exchange(amb_ctx* ctx, int mode) {
  if (!ctx || mode < 0 || mode > 3) return AMB_ERR_INVALID_ARGUMENT;
  ctx->halo_exchange_mode = mode;
  return AMB_OK;
}

int amb_comm_destroy(amb_ctx* ctx) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  if (ctx->nccl_comm && nccl().ok) {
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    peer_halo_release(ctx);
    for (unsigned char* p : ctx->halo_peer.retired) cudaFree(p);
    ctx->halo_peer.retired.clear();
    nccl().comm_destroy(static_cast<nccl_comm_t>(ctx->nccl_comm));
  }
  ctx->nccl_comm = nullptr;
  ctx->comm_rank = 0;
  ctx->comm_size = 1;
  return AMB_OK;
}

int amb_comm_last_exchange(const amb_ctx* ctx) { return ctx ? ctx->halo_last_exchange : 0; }
int amb_comm_size(const amb_ctx* ctx) { return ctx ? ctx->comm_size : 0; }
int amb_comm_rank(const amb_ctx* ctx) { return ctx ? ctx->comm_rank : -1; }

}  // extern "C"

namespace amb {

// The sharded step shared by Dsm (mode 0) and OrthoFromPcl (mode 1, d_intensities: every record's z is the point's
// intensity, no centre shift): exchange of the border halos, then the binning over [own points | neighbours' halos].
// The caller has checked the arguments and that the context belongs to a communicator of several ranks.
int sharded_step(amb_ctx* ctx, const double* d_xyz, const int* d_intensities, const uint64_t* d_ids,
                 size_t n_local, int32_t interpolation_radius, double center_easting, double center_northing,
                 uint32_t halo_capacity, int mode) {
  if (halo_capacity == 0) return AMB_ERR_INVALID_ARGUMENT;
  const int nranks = ctx->comm_size, rank = ctx->comm_rank;
  const size_t seg_bytes = 32 * (static_cast<size_t>(halo_capacity) + 1);  // header + records
  cudaStream_t s = ctx->stream;
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_BEGIN], s));
  double y_lo = 0, y_hi = 0;
  int st = amb_stripe_y_interval(&ctx->geom, ctx->col_begin, ctx->col_end, &y_lo, &y_hi);
  if (st != AMB_OK) return st;
  const double reach = amb_dsm_halo_reach(&ctx->geom, interpolation_radius);
  // compaction of this rank's border points into exchange segments (the NCCL exchanges; peer push compacts in the binning)
  auto compact = [&](unsigned char* seg_up, unsigned char* seg_down, bool split, uint32_t capacity) {
    if (n_local == 0) return cudaSuccess;
    const unsigned long long* ids = reinterpret_cast<const unsigned long long*>(d_ids);
    if (d_intensities)
      pcl_halo_records_kernel<<<ctx->num_sms * 8, 256, 0, s>>>(d_xyz, d_intensities, ids, n_local, y_lo, y_hi, reach,
                                                               seg_up, seg_down, split, capacity);
    else
      dsm_halo_records_kernel<<<ctx->num_sms * 8, 256, 0, s>>>(d_xyz, ids, n_local, y_lo, y_hi, reach, center_easting,
                                                               seg_up, seg_down, split, capacity);
    return cudaGetLastError();
  };

  // Who needs this rank's border points?  If the stripes are consecutive (rank r + 1 starts where rank r ends) and every
  // stripe is at least `reach` wide, only the two adjacent ranks do: two ncclSend / ncclRecv pairs in one group move each
  // half of the halo to the one rank that stages it.  Otherwise (narrow or irregular stripes) ONE ncclAllGather gives
  // every rank every halo.  The decision uses the stripes gathered at amb_comm_init: identical on all ranks.
  bool neighbours = ctx->halo_exchange_mode != 1;
  if (ctx->halo_exchange_mode == 0 || ctx->halo_exchange_mode == 3) {
    const double reach_cols = reach / ctx->geom.resolution;
    for (int r = 0; r < nranks && neighbours; ++r) {
      const int32_t b = ctx->comm_stripes[2 * r], e = ctx->comm_stripes[2 * r + 1];
      if (static_cast<double>(e - b) < reach_cols + 1.0) neighbours = false;
      if (r > 0 && ctx->comm_stripes[2 * r - 1] != b) neighbours = false;
    }
  }
  HaloSource halo;
  HaloPush push;
  bool use_push = false;
  halo.capacity = halo_capacity;
  halo.seg_bytes = seg_bytes;
  if (neighbours) {
    // each list holds ONE side of the halo: half the capacity
    const uint32_t side_capacity = halo_capacity / 2 + 1;
    const size_t side_bytes = 32 * (static_cast<size_t>(side_capacity) + 1);
    halo.capacity = side_capacity;
    halo.seg_bytes = side_bytes;
    HaloPeer& hp = ctx->halo_peer;
    if (!hp.tried) {
      const char* e = std::getenv("AMB_HALO_PEER");  // development switch: AMB_HALO_PEER=0 keeps ncclSend/ncclRecv
      hp.disabled = e && e[0] == '0';
    }
    // (collective, see peer_halo_setup: first sharded call, or the capacity grew — the same on every rank)
    if (ctx->halo_exchange_mode != 3 && !hp.disabled && (!hp.tried || (hp.enabled && side_capacity > hp.side_capacity))) {
      hp.tried_capacity = side_capacity;
      st = peer_halo_setup(ctx, side_capacity);
      if (st != AMB_OK) return st;
    }
    if (hp.enabled && ctx->halo_exchange_mode != 3) {
      // peer push: the partition kernel of the binning (dsm_run) stores the border records into the neighbours' segments of
      // this step's parity while it bins the rank's own points and publishes the counts; halo_wait_kernel then holds the
      // binning of the incoming halos back until both neighbours have published theirs
      const size_t peer_side_bytes = 32 * (static_cast<size_t>(hp.side_capacity) + 1);
      const unsigned int parity = static_cast<unsigned int>(hp.step & 1u);
      const unsigned int stamp = static_cast<unsigned int>(hp.step + 1);
      ++hp.step;
      // segment layout of every rank: [parity][0 = filled by rank - 1 | 1 = filled by rank + 1]
      push.seg_up = hp.prev ? hp.prev + (2 * parity + 1) * peer_side_bytes : nullptr;    // I am rank - 1's "rank + 1"
      push.seg_down = hp.next ? hp.next + (2 * parity + 0) * peer_side_bytes : nullptr;  // I am rank + 1's "rank - 1"
      push.counters = hp.counters + 4 * parity;
      push.capacity = side_capacity;
      push.stamp = stamp;
      push.y_lo = y_lo;
      push.y_hi = y_hi;
      push.reach = reach;
      push.shift_y = center_easting;
      unsigned char* mine = hp.recv + 2 * parity * peer_side_bytes;
      push.wait_prev = rank > 0 ? mine : nullptr;
      push.wait_next = rank < nranks - 1 ? mine + peer_side_bytes : nullptr;
      use_push = true;
      ctx->halo_last_exchange = 4;
      halo.gathered = mine;
      halo.seg_bytes = peer_side_bytes;
      halo.nranks = 2;
      halo.my_rank = -1;  // both segments are foreign (a missing neighbour's header stays {0, 0}: an empty list)
    } else {
    // send: [up | down], recv: [from rank - 1 | from rank + 1]
    AMB_CUDA(ctx, ctx->halo_send.reserve(2 * side_bytes));
    AMB_CUDA(ctx, ctx->halo_recv.reserve(2 * side_bytes));
    unsigned char* send = ctx->halo_send.as<unsigned char>();
    unsigned char* recv = ctx->halo_recv.as<unsigned char>();
    AMB_CUDA(ctx, cudaMemsetAsync(send, 0, 32, s));
    AMB_CUDA(ctx, cudaMemsetAsync(send + side_bytes, 0, 32, s));
    AMB_CUDA(ctx, cudaMemsetAsync(recv, 0, 32, s));              // a missing neighbour contributes an empty list
    AMB_CUDA(ctx, cudaMemsetAsync(recv + side_bytes, 0, 32, s));
    AMB_CUDA(ctx, compact(send, send + side_bytes, true, side_capacity));
    nccl_comm_t comm = static_cast<nccl_comm_t>(ctx->nccl_comm);
    int rc = nccl().group_start();
    if (rc == 0 && rank > 0) rc = nccl().send(send, side_bytes, kNcclInt8, rank - 1, comm, s);
    if (rc == 0 && rank > 0) rc = nccl().recv(recv, side_bytes, kNcclInt8, rank - 1, comm, s);
    if (rc == 0 && rank < nranks - 1) rc = nccl().send(send + side_bytes, side_bytes, kNcclInt8, rank + 1, comm, s);
    if (rc == 0 && rank < nranks - 1) rc = nccl().recv(recv + side_bytes, side_bytes, kNcclInt8, rank + 1, comm, s);
    const int rc_end = nccl().group_end();
    if (rc != 0 || rc_end != 0) return nccl_fail(ctx, rc != 0 ? rc : rc_end, "ncclSend/ncclRecv (halo)");
    ctx->halo_last_exchange = 2;
    halo.gathered = recv;
    halo.nranks = 2;
    halo.my_rank = -1;  // both segments are foreign
    }
  } else {
    AMB_CUDA(ctx, ctx->halo_send.reserve(seg_bytes));
    AMB_CUDA(ctx, ctx->halo_recv.reserve(seg_bytes * nranks));
    unsigned char* send = ctx->halo_send.as<unsigned char>();
    AMB_CUDA(ctx, cudaMemsetAsync(send, 0, 32, s));
    AMB_CUDA(ctx, compact(send, send, false, halo_capacity));
    // the one collective of the step
    const int rc = nccl().all_gather(send, ctx->halo_recv.ptr, seg_bytes, kNcclInt8,
                                     static_cast<nccl_comm_t>(ctx->nccl_comm), s);
    if (rc != 0) return nccl_fail(ctx, rc, "ncclAllGather");
    ctx->halo_last_exchange = 1;
    halo.gathered = ctx->halo_recv.as<unsigned char>();
    halo.nranks = nranks;
    halo.my_rank = rank;
  }
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_H2D_END], s));  // "h2d" slot of the timings = the halo step
  ctx->dsm_had_h2d = true;
  st = dsm_run(ctx, d_xyz, reinterpret_cast<const unsigned long long*>(d_ids), n_local, interpolation_radius,
               center_easting, center_northing, mode, d_intensities, &halo, use_push ? &push : nullptr);
  ctx->dsm_timed = (st == AMB_OK);
  return st;
}

}  // namespace amb
