// halo_push.h — the border halo of a sharded cloud: which points it holds, the segment that carries it to the neighbours,
// and the device helpers of its three producers (amb_dsm_extract_halo's SoA output in dsm_kernels.cu, the NCCL
// compaction in amb_comm.cu, the peer push of the binning's partition kernel in dsm_partition.inc) and of its reader
// (the same partition kernel, which bins the neighbours' halos after the rank's own points).
//
// A stripe's border halo: its points within `reach` of the two borders of the y-interval (y_lo, y_hi] it owns, tested
// on ys = y - shift_y (Dsm: center_easting; OrthoFromPcl: 0).  Column 0 is the max-y side, so the "up" side is what
// rank - 1 needs and the "down" side what rank + 1 needs.
//
// Segment: a 32-byte header {uint32 count | uint32 stamp << 32, unused} followed by `capacity` 32-byte records
// {x, y, z, id} of raw coordinates (OrthoFromPcl: z = double(intensity)).  The count is the true number of border
// points; only the first `capacity` of them are stored, and a reader that finds count > capacity raises the sticky
// halo-overflow flag.  The id word: readers use its low 32 bits; producers may leave the high bits unset.
#ifndef AMB_HALO_PUSH_H_
#define AMB_HALO_PUSH_H_

#include <cuda_runtime.h>

#include <cstddef>

struct amb_ctx;

namespace amb {

constexpr size_t kHaloHeaderBytes = 32;  // = the size of one record

inline size_t halo_segment_bytes(unsigned int capacity) {
  return kHaloHeaderBytes * (static_cast<size_t>(capacity) + 1);
}
__device__ __forceinline__ unsigned int* halo_count(unsigned char* seg) { return reinterpret_cast<unsigned int*>(seg); }
__device__ __forceinline__ unsigned int halo_count(const unsigned char* seg) {
  return *reinterpret_cast<const unsigned int*>(seg);
}
__device__ __forceinline__ double* halo_slot(unsigned char* seg, size_t k) {
  return reinterpret_cast<double*>(seg + kHaloHeaderBytes) + 4 * k;
}
__device__ __forceinline__ const double* halo_slot(const unsigned char* seg, size_t k) {
  return reinterpret_cast<const double*>(seg + kHaloHeaderBytes) + 4 * k;
}

// The halos a rank bins after its own points: nranks segments of seg_bytes, each read up to min(count, capacity);
// the segment of my_rank is skipped (those points are already local; -1: every segment is foreign).
struct HaloSource {
  const unsigned char* gathered = nullptr;
  int nranks = 0, my_rank = 0;
  unsigned int capacity = 0;
  size_t seg_bytes = 0;
};

// Slot `s` of the halos -> its record, or nullptr (own segment, beyond the segment's count).
__device__ __forceinline__ const double* halo_record(const HaloSource& h, size_t s) {
  const unsigned int r = static_cast<unsigned int>(s / h.capacity);
  const unsigned int k = static_cast<unsigned int>(s - static_cast<size_t>(r) * h.capacity);
  if (static_cast<int>(r) == h.my_rank) return nullptr;
  const unsigned char* seg = h.gathered + static_cast<size_t>(r) * h.seg_bytes;
  if (k >= halo_count(seg)) return nullptr;
  return halo_slot(seg, k);
}

// The one border test: is a point with ys = y - shift_y in the halo of rank - 1 (up) and of rank + 1 (down)?
struct BorderSides {
  bool up, down;
};
__device__ __forceinline__ BorderSides border_sides(double ys, double y_lo, double y_hi, double reach) {
  return {ys > y_hi - reach, ys < y_lo + reach};
}

// One record = two 128-bit stores (sm_90's widest) = exactly one DRAM sector.
__device__ __forceinline__ void store_record(double* dst, double x, double y, double z, unsigned long long id) {
#ifdef AMB_CUDA_EMU  // tests/emu (CPU emulation of the kernel source)
  dst[0] = x;
  dst[1] = y;
  dst[2] = z;
  dst[3] = __longlong_as_double(static_cast<long long>(id));
#else
  asm volatile("st.global.v2.f64 [%0], {%1, %2};\n\tst.global.v2.f64 [%0+16], {%3, %4};" ::"l"(dst), "d"(x), "d"(y), "d"(z),
               "d"(__longlong_as_double(static_cast<long long>(id)))
               : "memory");
#endif
}

// Warp-aggregated slot reservation: every lane of the warp calls it; the lanes with `take` get consecutive slots in
// lane order, reserved by one atomic on `*counter`, and call `use(slot)`.
template <typename Use>
__device__ __forceinline__ void warp_reserve(bool take, unsigned int* counter, Use use) {
  const unsigned int mask = __ballot_sync(0xffffffffu, take);
  if (mask) {
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(mask) - 1;
    unsigned int base = 0;
    if (lane == leader) base = atomicAdd(counter, static_cast<unsigned int>(__popc(mask)));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (take) use(base + __popc(mask & ((1u << lane) - 1u)));
  }
}

// A rank's points and its stripe's border test, as the NCCL compaction reads them.
struct HaloCloud {
  const double* xyz = nullptr;
  const int* intensities = nullptr;  // OrthoFromPcl: the records' z
  const unsigned long long* ids = nullptr;  // nullptr: the array positions
  size_t n = 0;
  double y_lo = 0, y_hi = 0, reach = 0, shift_y = 0;
};

// amb_comm.cu: zero the headers of the segments and compact the cloud's border points into them, each side into its
// own segment with `split` (ncclSend / ncclRecv), both into seg_up without (ncclAllGather: one list per rank).
int halo_compact(struct ::amb_ctx* ctx, const HaloCloud& c, unsigned char* seg_up, unsigned char* seg_down, bool split,
                 unsigned int capacity);

// ---- peer push: the partition kernel stores the border records straight into the adjacent ranks' segments over
// NVLink peer memory while it bins the rank's own points, and its last block publishes {count, step stamp}
struct HaloPush {
  unsigned char* seg_up = nullptr;     // PEER memory: the segment of rank - 1 that this rank fills (nullptr: no such rank)
  unsigned char* seg_down = nullptr;   // PEER memory: the segment of rank + 1 that this rank fills
  unsigned int* counters = nullptr;    // LOCAL: [0] up count, [1] down count, [2] blocks done
  unsigned int capacity = 0;           // records per segment
  unsigned int stamp = 0;              // step + 1
  double y_lo = 0, y_hi = 0, reach = 0, shift_y = 0;   // the border test
  // consumer side: this rank's own segments of the same parity (nullptr: no such neighbour)
  const unsigned char* wait_prev = nullptr;
  const unsigned char* wait_next = nullptr;
};

__device__ __forceinline__ void store_release_sys(unsigned char* p, unsigned long long v) {
#ifdef AMB_CUDA_EMU
  *reinterpret_cast<volatile unsigned long long*>(p) = v;
#else
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#endif
}
__device__ __forceinline__ unsigned long long load_acquire_sys(const unsigned char* p) {
#ifdef AMB_CUDA_EMU
  return *reinterpret_cast<const volatile unsigned long long*>(p);
#else
  unsigned long long h;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(h) : "l"(p) : "memory");
  return h;
#endif
}

// End of the producing kernel, called by every thread of every block: each thread's peer stores are fenced (system
// scope) before its block takes a ticket; the block that takes the last ticket has therefore observed all of them and
// releases the two headers {count | stamp << 32}.
__device__ __forceinline__ void halo_publish(const HaloPush& a) {
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int ticket = atomicAdd(a.counters + 2, 1u);
    if (ticket == gridDim.x - 1) {
      __threadfence();
      const unsigned int c_up = atomicExch(a.counters + 0, 0u);  // (reset for the next step of this parity)
      const unsigned int c_down = atomicExch(a.counters + 1, 0u);
      atomicExch(a.counters + 2, 0u);
      __threadfence_system();
      const unsigned long long stamp = static_cast<unsigned long long>(a.stamp) << 32;
      if (a.seg_up) store_release_sys(a.seg_up, static_cast<unsigned long long>(c_up) | stamp);
      if (a.seg_down) store_release_sys(a.seg_down, static_cast<unsigned long long>(c_down) | stamp);
    }
  }
}

// amb_comm.cu: enqueue the kernel in which two lanes spin (acquire, system scope, bounded) until both of this rank's
// segments carry the step's stamp
int halo_wait_launch(struct ::amb_ctx* ctx, const HaloPush& push);

}  // namespace amb
#endif  // AMB_HALO_PUSH_H_
