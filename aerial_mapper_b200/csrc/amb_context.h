// amb_context.h — internal state behind the C ABI (include/aerial_mapper_b200.h).  sm_90a (H100) only.
#pragma once

#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "../../include/aerial_mapper_b200.h"

namespace amb {

// A grow-only device buffer: process() is called repeatedly on the same context (incremental mapping,
// main-ortho-backward-grid-incremental.cc:143-163), so scratch is allocated once and kept.
struct DeviceBuffer {
  void* ptr = nullptr;
  size_t bytes = 0;
  cudaError_t reserve(size_t want) {
    if (want <= bytes) return cudaSuccess;
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    bytes = 0;
    // round up so that slowly growing inputs do not reallocate every call
    size_t alloc = (want + (size_t(1) << 20) - 1) & ~((size_t(1) << 20) - 1);
    cudaError_t e = cudaMalloc(&ptr, alloc);
    if (e == cudaSuccess) bytes = alloc;
    return e;
  }
  void release() {
    if (ptr) cudaFree(ptr);
    ptr = nullptr;
    bytes = 0;
  }
  template <typename T>
  T* as() const {
    return static_cast<T*>(ptr);
  }
};

// Page-locked host staging for the small per-call tables (frame constants, cull data, bounding boxes ...).
// Copies from PAGEABLE memory serialise with copies in flight on other streams; from pinned memory they do not,
// which is what lets result downloads overlap the next stage.
struct HostStage {
  unsigned char* ptr = nullptr;
  size_t bytes = 0, used = 0;
  cudaError_t reserve(size_t want) {
    if (want <= bytes) return cudaSuccess;
    if (ptr) cudaFreeHost(ptr);
    ptr = nullptr;
    bytes = 0;
    const size_t alloc = (want + 65535) & ~static_cast<size_t>(65535);
    cudaError_t e = cudaHostAlloc(reinterpret_cast<void**>(&ptr), alloc, cudaHostAllocMapped);
    if (e == cudaSuccess) bytes = alloc;
    return e;
  }
  template <typename T>
  T* take(size_t count) {  // 64-byte aligned slices; reserve() must have been called with the total
    used = (used + 63) & ~static_cast<size_t>(63);
    T* p = reinterpret_cast<T*>(ptr + used);
    used += count * sizeof(T);
    return p;
  }
  void release() {
    if (ptr) cudaFreeHost(ptr);
    ptr = nullptr;
    bytes = used = 0;
  }
};

enum EventId {
  EV_DSM_BEGIN = 0,
  EV_DSM_H2D_END,
  EV_DSM_BIN_END,
  EV_DSM_GATHER_END,
  EV_DSM_FILL_END,
  EV_ORTHO_BEGIN,
  EV_ORTHO_H2D_END,
  EV_ORTHO_SELECT_END,
  EV_ORTHO_COPY_END,
  EV_ORTHO_END,
  EV_COUNT
};

// Slots of the small device flag/counter block (amb_ctx::counters, 16 x uint32).  Every stage resets only its own slots.
// The two deferred reference-CHECK flags are STICKY: kernels set them, the next amb_sync() or host entry point reports
// and clears them — an asynchronous `_device` sequence (ortho -> dsm -> amb_sync) cannot lose an earlier call's failure.
enum CounterSlot {
  CTR_DSM_LIST = 0,        // length of the warp-per-cell list (reset per DSM launch group)
  CTR_DSM_COINCIDENT = 1,  // sticky: CHECK(distances[i] > 0.0), dsm.cc:165
  CTR_DSM_BINNED = 2,      // points the binning kept
  CTR_DSM_DENSE = 3,       // tiles handed whole to the warp-per-cell kernel
  CTR_DSM_LIST_DONE = 5,   // chunked evaluation: list lengths of the chunks already evaluated
  CTR_HALO_OVERFLOW = 6,   // sticky: a rank's border halo did not fit the capacity passed to amb_dsm_process_sharded_device
  CTR_DSM_AMBIGUOUS = 4,   // f32 gather: cells re-evaluated exactly (a pair inside the guard band, an unbounded height)
  CTR_ORTHO_CHECK = 8,     // sticky: CHECK(alpha > 0.0), ortho-backward-grid.cc:178
  CTR_PCL_CELLS = 10,      // adaptive OrthoFromPcl: cells listed for the 10^k radius growth
  CTR_PCL_UNRESOLVED = 11, // adaptive OrthoFromPcl: cells no level could fill
  CTR_COUNT = 16
};

// Narrow transport of a small-integer result layer to its host mirror (mirror_compact.cu)
struct CompactMirror {
  bool enabled = true;                // (ortho / observation_index mirrors) amb_set_host_mirror_compact(.., 0) turns it off
  std::atomic<bool> failed{false};    // an expander thread could not wait for its chunk: reported by amb_sync, which then
                                      // re-downloads the layer as float32
  DeviceBuffer codes;                 // one byte per slab cell
  uint8_t* host_codes = nullptr;      // pinned landing zone of the codes
  size_t host_bytes = 0;
  unsigned int* host_flag = nullptr;  // pinned + mapped: set by the pack kernel when a value has no code
  std::vector<cudaEvent_t> chunk_events;
  std::atomic<int> jobs_in_flight{0}; // chunks of the current round still being widened by the expander pool
};

// Peer-push halo exchange (amb_comm.cu, halo_push.h): this rank's receive segments [parity 0/1][from rank - 1 | from
// rank + 1] and the mapped pointers to the two neighbours' segments.
struct HaloPeer {
  bool enabled = false, tried = false, disabled = false;
  unsigned char* recv = nullptr;       // own, cudaMalloc: 4 segments of halo_segment_bytes(side_capacity)
  unsigned int* counters = nullptr;    // own: [parity][up count, down count, blocks done, -]
  unsigned char* prev = nullptr;       // rank - 1's `recv`, mapped (cudaIpcOpenMemHandle or same-process peer access)
  unsigned char* next = nullptr;
  bool prev_ipc = false, next_ipc = false;
  uint32_t side_capacity = 0, tried_capacity = 0;
  uint64_t step = 0;
  std::vector<unsigned char*> retired;   // segments replaced by a larger re-setup: freed when the communicator is left
};

}  // namespace amb

struct amb_ctx {
  amb_geometry geom;
  int device = 0;
  int num_sms = 1;  // multiprocessors of the device: the grid-stride launches size their grids by it (amb_create)
  int32_t col_begin = 0, col_end = 0;  // owned column stripe
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;  // H2D staging overlapped with compute
  cudaEvent_t events[amb::EV_COUNT] = {};
  cudaEvent_t copy_done[2] = {};
  // pinned staging of per-call tables, double-buffered: call k fills stages[k & 1] while the asynchronous copies and the
  // kernel of call k - 1 may still read stages[(k - 1) & 1] — with one buffer the host could not prepare the next
  // process() before the previous kernel had finished (measured: ortho-only steps were host-bound)
  amb::HostStage stages[2];
  cudaEvent_t stage_events[2] = {nullptr, nullptr};   // last use of each buffer by an asynchronous copy
  unsigned int stage_turn = 0;
  unsigned int* host_flags = nullptr;   // pinned: device flags read back at the end of a host entry point
  float* host_mirror[AMB_NUM_LAYERS] = {};  // pinned host slabs that receive a layer as soon as it is final
  amb::CompactMirror compact[AMB_NUM_LAYERS];  // opt-in one-byte transport (amb_set_host_mirror_compact)
  cudaEvent_t layer_copy_event[AMB_NUM_LAYERS] = {};  // completion of an asynchronous download of that layer
  bool layer_copy_pending[AMB_NUM_LAYERS] = {};
  bool dsm_timed = false, ortho_timed = false, dsm_had_h2d = false, ortho_had_h2d = false;
  int32_t dsm_launches = 0, ortho_launches = 0;
  std::string last_error;

  float* layers[AMB_NUM_LAYERS] = {};

  // DSM scratch
  amb::DeviceBuffer points;       // device copy of the caller's xyz (host entry point)
  amb::DeviceBuffer point_ids;    // device copy of the caller's global point ids (sharded host entry point)
  amb::DeviceBuffer intensities;  // device copy of the caller's intensities (OrthoFromPcl host entry point)
  amb::DeviceBuffer records;      // bucket-sorted 32-byte point records
  amb::DeviceBuffer records_tmp;  // two-level binning: the points as 32-byte records, tile by tile, grouped by coarse destination
  amb::DeviceBuffer tile_offsets; // ... and the uint16 run starts, [(S + 1)][n_tiles]
  amb::DeviceBuffer point_order;  // uint32 per record: canonical (original-index) visiting order inside a bucket
  amb::DeviceBuffer bucket_flags; // one byte per bucket: the warp-per-cell kernel will read it (dsm_mark_buckets_kernel)
  amb::DeviceBuffer bin_starts;   // uint32 G[nb + 2]
  amb::DeviceBuffer block_sums;   // scan spine
  amb::DeviceBuffer empty_cells;  // uint32 list of cells that need the expanding-radius pass
  amb::DeviceBuffer counters;     // small flag/counter block, see amb::CounterSlot
  amb::DeviceBuffer dbg_count;    // int32 per slab cell
  amb::DeviceBuffer dbg_level;    // int8 per slab cell
  amb::DeviceBuffer raster_band;  // amb_export_raster: the converted band before its copy to the host;
                                  // amb_import_raster: the raster window after its copy to the device
  amb::DeviceBuffer raster_taps;  // amb_import_raster*: the per-axis tables of the last import
  amb::DeviceBuffer jpeg_mcu;     // JPEG encoder (jpeg_encode.cu): DC per block, bit offset per MCU, byte offset per interval
  amb::DeviceBuffer jpeg_spine;   // ... tile sums of its scans
  amb::DeviceBuffer jpeg_words;   // ... the entropy-coded stream before byte stuffing, and 0xFF counts per chunk
  amb::DeviceBuffer jpeg_out;     // ... the stuffed stream with its RST markers, copied to the host
  double dsm_density_hint = 0.0;  // points per cell of the whole cloud (0: derive from the points passed)
  bool dsm_debug = false;
  int dsm_stream_chunks = 4;  // (> 1, only with a host mirror of the output layer) gather + fill in column chunks, each chunk's
                              // result mirrored to the host at once, so the download overlaps the remaining chunks
  // multi-GPU (amb_comm.cu): NCCL communicator this context is a member of, and the halo buffers of the exchange step
  void* nccl_comm = nullptr;
  int comm_rank = 0, comm_size = 1;
  std::vector<int32_t> comm_stripes;   // [2 * nranks]: col_begin, col_end of every member (gathered by amb_comm_init)
  int halo_exchange_mode = 0;          // 0 auto, 1 all-gather, 2 neighbours (amb_comm_set_exchange)
  amb::DeviceBuffer halo_send, halo_recv;
  amb::HaloPeer halo_peer;
  int halo_last_exchange = 0;          // what the last sharded call used: 1 all-gather, 2 ncclSend/ncclRecv, 4 peer push
  int dsm_precision = AMB_DSM_F32;  // amb_dsm_set_precision: arithmetic of the tile gather's weights and sums
  bool dsm_debug_valid = false;
  int64_t last_points_binned = 0, last_cells_empty = 0;
  std::vector<unsigned char> last_dsm_plan;  // the DsmPlan of the last dsm_run (read by the adaptive OrthoFromPcl pass;
                                             // on a stripe: of its whole-map binning, dsm_run(.., whole_map_bins))
  int32_t last_bin_destinations = 0;         // coarse destinations S of the last binning (0: none yet; amb_dsm_download_bins)

  // Ortho scratch
  amb::DeviceBuffer frames;       // device copies of the caller's frames (host entry point)
  amb::DeviceBuffer frame_table;  // per-frame device image pointers
  amb::DeviceBuffer frame_cull;   // per-frame camera centre + R_C_G rows (tile cull test)
  amb::DeviceBuffer frame_rects;  // host-frame path: per-frame uploaded sub-rectangle
  amb::DeviceBuffer ortho_pix;    // host-frame path: winner pixel per cell
  amb::DeviceBuffer ortho_bbox;   // host-frame path: per-frame bounding box of the winners' pixels
  int64_t ortho_h2d_bytes = 0;
  bool ortho_two_phase = false;
  bool ortho_brute_force = false;
  bool ortho_dominance = true;   // per-tile dominance cull of the frame list (OrthoArgs::dominance); amb_ortho_set_dominance_cull(0) = plain list

  size_t slab_cells() const { return static_cast<size_t>(geom.rows) * static_cast<size_t>(col_end - col_begin); }
};

namespace amb {

struct HaloSource;  // halo_push.h
struct HaloPush;

inline int fail(amb_ctx* ctx, cudaError_t e, const char* what) {
  if (ctx) {
    ctx->last_error = std::string(what) + ": " + cudaGetErrorString(e);
  }
  return AMB_ERR_CUDA;
}

#define AMB_CUDA(ctx, call)                                   \
  do {                                                        \
    cudaError_t e__ = (call);                                 \
    if (e__ != cudaSuccess) return amb::fail(ctx, e__, #call); \
  } while (0)

int ensure_counters(amb_ctx* ctx);  // allocates (zeroed) the flag/counter block on first use
int ensure_layer(amb_ctx* ctx, int layer);
int wait_layer_copy(amb_ctx* ctx, int layer);  // writers of a layer wait for its pending asynchronous download
int enqueue_layer_download(amb_ctx* ctx, int layer, float* host_slab);  // on the copy stream, after current work
int mirror_layer(amb_ctx* ctx, int layer);
int mirror_layer_columns(amb_ctx* ctx, int layer, int col0, int col1);  // slab-local column range
// mirror_compact.cu
int mirror_layer_compact(amb_ctx* ctx, int layer);
int join_compact_mirrors(amb_ctx* ctx);         // AMB_ERR_CUDA if an expander failed (the layer was re-downloaded as float32)
void wait_compact_layer(amb_ctx* ctx, int layer);  // the expander pool has finished this layer's round
void release_compact_mirrors(amb_ctx* ctx);     // enqueue_layer_download to the registered host mirror, if any

// host_staging.cu: copies whose host side may be PAGEABLE memory (staged through pinned slots by a worker pool)
bool host_memory_is_pageable(const void* p);
int staged_h2d(amb_ctx* ctx, void* dst_dev, const void* src_host, size_t bytes, cudaStream_t s);
int staged_d2h(amb_ctx* ctx, void* dst_host, const void* src_dev, size_t bytes, cudaStream_t s);  // synchronous
struct StagedRect {
  unsigned char* dst;        // device
  size_t dst_pitch;
  const unsigned char* src;  // host
  size_t src_pitch, w, h;    // bytes per row, rows
};
int staged_h2d_rects(amb_ctx* ctx, const StagedRect* rects, size_t n, cudaStream_t s);

// Implemented in dsm_kernels.cu / ortho_kernels.cu
int dsm_run(amb_ctx* ctx, const double* d_xyz, const unsigned long long* d_ids, size_t n,
            int32_t interpolation_radius, double center_easting, double center_northing, int mode = 0,
            const int* d_intensities = nullptr, const HaloSource* halo = nullptr, const HaloPush* push = nullptr,
            bool whole_map_bins = false);
// d_intensities != nullptr (OrthoFromPcl): the halo's intensities go to d_out_intensities, no centre shift
int dsm_extract_halo(amb_ctx* ctx, const double* d_xyz, const unsigned long long* d_ids, size_t n, double y_lo,
                     double y_hi, double reach, double center_easting, double* d_out_xyz,
                     unsigned long long* d_out_ids, unsigned int capacity, unsigned int* d_count,
                     const int* d_intensities = nullptr, int* d_out_intensities = nullptr);
// Implemented in pcl_adaptive_kernels.cu: ortho::Settings::use_adaptive_interpolation around dsm_run(mode = 1).  On a
// stripe, finish bins the same points (the whole cloud) again on the whole map's bin grid.
int pcl_adaptive_prepare(amb_ctx* ctx, float** saved);
int pcl_adaptive_finish(amb_ctx* ctx, int pass_status, const double* d_xyz, const unsigned long long* d_ids,
                        const int* d_intensities, size_t n, int32_t interpolation_radius, float* saved);
int ortho_run(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B, const uint8_t* const* d_images,
              const uint8_t* const* h_images, size_t n, int32_t channels, size_t row_step, int32_t colored_ortho);
// amb_comm.cu: one step of a sharded cloud on a context of a communicator of several ranks (halo exchange, then
// dsm_run over the rank's points and the neighbours' halos); records the DSM events and sets dsm_timed itself
int sharded_step(amb_ctx* ctx, const double* d_xyz, const int* d_intensities, const uint64_t* d_ids, size_t n_local,
                 int32_t interpolation_radius, double center_easting, double center_northing, uint32_t halo_capacity,
                 int mode);
std::vector<double> dsm_thresholds(int32_t interpolation_radius);
double dsm_tile_reach_cells(double resolution, int32_t interpolation_radius);  // tile width + window apron + 1, in cells

}  // namespace amb
