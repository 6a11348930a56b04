// emu_test_hooks.cc — TEST INFRASTRUCTURE ONLY (tests/emu): entry points of the EMULATED library that reach product
// internals no C-ABI call exposes on a single process.  Compiled into libamb_emu.so only; the product library does not
// contain this file.
//
// amb_emu_halo_segments: the three producers of border-halo segments (csrc/halo_push.h) need other ranks on real hardware.
// Here the "neighbours' segments" are two local buffers, filled by
//   producer 0: the peer push — the DSM / OrthoFromPcl binning of a stripe through amb::dsm_run with a HaloPush whose
//               segments point at them (and an empty incoming halo; dsm_partition_kernel<PUSH>, halo_publish);
//   producer 1: the compaction of the send/recv exchange (amb::halo_compact, split: one segment per side);
//   producer 2: the compaction of the all-gather exchange (amb::halo_compact, both sides into seg_up).
// The caller gets the segments back to compare with the border sets it computes itself.  intensities != NULL:
// OrthoFromPcl (records carry the intensities as z, no centre shift: pass center_easting = 0).
// amb_emu_self_push: producer 0 for the DSM.
#include <cstring>

#include "amb_context.h"
#include "halo_push.h"

extern "C" int amb_emu_halo_segments(amb_ctx* ctx, int producer, const double* xyz, const int* intensities,
                                     const unsigned long long* ids, size_t n, int32_t interpolation_radius,
                                     double center_easting, double center_northing, unsigned int capacity,
                                     int have_prev, int have_next, unsigned int stamp, unsigned char* seg_up_out,
                                     unsigned char* seg_down_out) {
  if (!ctx || !xyz || !ids || !seg_up_out || !seg_down_out || producer < 0 || producer > 2)
    return AMB_ERR_INVALID_ARGUMENT;
  const size_t seg_bytes = amb::halo_segment_bytes(capacity);
  std::memset(seg_up_out, 0, seg_bytes);
  std::memset(seg_down_out, 0, seg_bytes);
  amb::HaloCloud c;
  c.xyz = xyz;
  c.intensities = intensities;
  c.ids = ids;
  c.n = n;
  int st = amb_stripe_y_interval(&ctx->geom, ctx->col_begin, ctx->col_end, &c.y_lo, &c.y_hi);
  if (st != AMB_OK) return st;
  c.reach = amb_dsm_halo_reach(&ctx->geom, interpolation_radius);
  c.shift_y = center_easting;
  if (producer != 0) return amb::halo_compact(ctx, c, seg_up_out, seg_down_out, producer == 1, capacity);

  // the incoming halo: two empty segments (count 0)
  unsigned char* incoming = nullptr;
  unsigned int* counters = nullptr;
  if (cudaMalloc(&incoming, 2 * seg_bytes) != cudaSuccess || cudaMalloc(&counters, 4 * sizeof(unsigned int)) != cudaSuccess)
    return AMB_ERR_CUDA;
  std::memset(incoming, 0, 2 * seg_bytes);
  std::memset(counters, 0, 4 * sizeof(unsigned int));
  amb::HaloSource halo;
  halo.gathered = incoming;
  halo.nranks = 2;
  halo.my_rank = -1;
  halo.capacity = capacity;
  halo.seg_bytes = seg_bytes;
  amb::HaloPush push;
  push.seg_up = have_prev ? seg_up_out : nullptr;
  push.seg_down = have_next ? seg_down_out : nullptr;
  push.counters = counters;
  push.capacity = capacity;
  push.stamp = stamp;
  push.y_lo = c.y_lo;
  push.y_hi = c.y_hi;
  push.reach = c.reach;
  push.shift_y = c.shift_y;
  push.wait_prev = nullptr;  // nobody to wait for: the incoming segments are final (empty)
  push.wait_next = nullptr;
  st = amb::dsm_run(ctx, xyz, ids, n, interpolation_radius, center_easting, center_northing, intensities ? 1 : 0,
                    intensities, &halo, &push);
  const unsigned int left[3] = {counters[0], counters[1], counters[2]};
  cudaFree(incoming);
  cudaFree(counters);
  if (st != AMB_OK) return st;
  return (left[0] | left[1] | left[2]) ? AMB_ERR_CHECK_FAILED : AMB_OK;  // the last block resets the three counters
}

extern "C" int amb_emu_self_push(amb_ctx* ctx, const double* xyz, const unsigned long long* ids, size_t n,
                                 int32_t interpolation_radius, double center_easting, double center_northing,
                                 unsigned int capacity, int have_prev, int have_next, unsigned int stamp,
                                 unsigned char* seg_up_out, unsigned char* seg_down_out) {
  return amb_emu_halo_segments(ctx, 0, xyz, nullptr, ids, n, interpolation_radius, center_easting, center_northing,
                               capacity, have_prev, have_next, stamp, seg_up_out, seg_down_out);
}
