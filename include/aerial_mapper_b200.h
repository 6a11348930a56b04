/*
 * aerial_mapper_b200.h — C ABI of the H100-native grid-mapping hot path.
 *
 * This is the drop-in boundary for the ONE data-parallel path of ethz-asl/aerial_mapper:
 *   - dsm::Dsm::process                       (reference aerial_mapper_dsm/src/dsm.cc:186-201, cell loop :113-184)
 *   - ortho::OrthoBackwardGrid::process       (reference aerial_mapper_ortho/src/ortho-backward-grid.cc:223-239,
 *                                              cell loop :128-221)
 * The reference has no FFI layer of its own: its boundary is those two C++ classes operating on a
 * grid_map::GridMap (float32, column-major layers).  The C++ shim under aerial_mapper_b200/shim/ re-creates the
 * two classes with the reference signatures and marshals to the functions below; the Python mirror
 * (aerial_mapper_b200/api.py) binds the same functions through ctypes.  Plain pointers and sizes only.
 *
 * Conventions
 *   - Layers are float32, column-major, `rows x cols` with rows = size(0) (x / easting, Eigen row index) and
 *     cols = size(1) (y / northing); element (i,j) lives at `i + j*rows`
 *     (grid_map::Matrix = Eigen::MatrixXf, reference aerial-mapper-grid-map.cc:25-48).
 *   - A context owns ONE device and ONE contiguous column stripe [col_begin, col_end) of the map (a slab of
 *     rows*(col_end-col_begin) floats per layer).  A single-GPU context owns [0, cols).
 *   - Every function returns AMB_OK (0) or a negative amb_status.  The reference aborts through glog CHECK on
 *     contract violations; the shim turns a non-zero status back into that behaviour.
 *   - Entry points taking HOST pointers are synchronous (like the reference's blocking process()).
 *     `_device` entry points take device pointers valid on the context's device, enqueue on the context's
 *     stream and return without synchronising; call amb_sync() before reading results.
 */
#ifndef AERIAL_MAPPER_B200_H_
#define AERIAL_MAPPER_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AMB_ABI_VERSION 2

typedef enum amb_status {
  AMB_OK = 0,
  AMB_ERR_EMPTY = -1,            /* empty point cloud / no frames (dsm.cc:189-192 warns+returns; ortho CHECKs) */
  AMB_ERR_SIZE_MISMATCH = -2,    /* poses vs images count, stripe bounds, layer sizes */
  AMB_ERR_COINCIDENT_POINT = -3, /* a point lies exactly on a cell centre: reference CHECK(distances[i] > 0) dsm.cc:165 */
  AMB_ERR_CUDA = -4,
  AMB_ERR_INVALID_ARGUMENT = -5,
  AMB_ERR_CHECK_FAILED = -6,     /* reference CHECK(alpha > 0.0), ortho-backward-grid.cc:178 */
  AMB_ERR_NO_DEVICE = -7,
  AMB_ERR_UNSUPPORTED = -8,
  AMB_ERR_CORRUPT_DATA = -9      /* a JPEG scan that is not valid for its header (amb_jpeg_decode_device), or a TIFF
                                    chunk that does not inflate to its data (amb_tiff_decode_device) */
} amb_status;

/* Geometry of the grid_map (grid_map::GridMap::setGeometry as called at aerial-mapper-grid-map.cc:30-33). */
typedef struct amb_geometry {
  int32_t rows;        /* size(0) = round(length_x_requested / resolution) */
  int32_t cols;        /* size(1) */
  double resolution;   /* metres per cell */
  double length_x;     /* rows * resolution */
  double length_y;     /* cols * resolution */
  double pos_x;        /* map centre, x = easting  */
  double pos_y;        /* map centre, y = northing */
} amb_geometry;

/* Layer ids in the order AerialGridMap creates them (aerial-mapper-grid-map.cc:25-28). */
typedef enum amb_layer_id {
  AMB_LAYER_ORTHO = 0,
  AMB_LAYER_ELEVATION = 1,
  AMB_LAYER_ELEVATION_ANGLE = 2,
  AMB_LAYER_NUM_OBSERVATIONS = 3,
  AMB_LAYER_ELEVATION_ANGLE_FIRST_VIEW = 4,
  AMB_LAYER_DELTA = 5,
  AMB_LAYER_OBSERVATION_INDEX = 6,
  AMB_LAYER_OBSERVATION_INDEX_FIRST = 7,
  AMB_LAYER_COLORED_ORTHO = 8,
  AMB_NUM_LAYERS = 9
} amb_layer_id;

/* Camera 0 of the aslam::NCamera rig (ortho-backward-grid.cc:131,232): pinhole + distortion + T_C_B. */
typedef enum amb_distortion {
  AMB_DIST_NONE = 0,
  AMB_DIST_RADTAN = 1,       /* k1 k2 p1 p2 */
  AMB_DIST_EQUIDISTANT = 2,  /* k1 k2 k3 k4 */
  /* aslam FisheyeDistortion ("FOV" model), dist[0] = w.  PROVENANCE: unlike rad-tan / equidistant (cross-checked against
   * OpenCV), this branch is restated from RECOLLECTION of upstream aslam_cv2 distortion-fisheye.cc — the source is not
   * under the reference tree and no offline cross-check exists.  Formula as implemented: r_d/r_u = atan(2 tan(w/2) r_u) /
   * (r_u w); w*w < 1e-5 -> 1; r_u*r_u < 1e-5 -> 2 tan(w/2) / w.  The two 1e-5 thresholds and the limit value are the
   * parts to verify against the upstream file before relying on bit-level parity for this model. */
  AMB_DIST_FOV = 3
} amb_distortion;

typedef struct amb_camera {
  int32_t width, height;     /* imageWidth(), imageHeight() */
  double fu, fv, cu, cv;     /* pinhole intrinsics */
  int32_t dist_type;         /* amb_distortion */
  int32_t reserved_;
  double dist[4];
  double q_C_B[4];           /* rotation of T_C_B as unit quaternion (w, x, y, z) */
  double t_C_B[3];           /* translation of T_C_B */
} amb_camera;

/* Device-side stage timings of the last process call, CUDA events on the context's stream (milliseconds). */
typedef struct amb_timings {
  float dsm_h2d_ms;      /* host->device copy of the points (host entry point only) */
  float dsm_bin_ms;      /* bin count + scan */
  float dsm_gather_ms;   /* scatter into the bins and the tile IDW gather (the dominant DSM kernel), which run at the
                            same time (+ OrthoFromPcl's in-bin canonical ordering) */
  float dsm_fill_ms;     /* expanding-radius hole fill kernel */
  float dsm_total_ms;
  float ortho_h2d_ms;    /* host->device copy of the needed frame sub-rectangles (host entry point only) */
  float ortho_kernel_ms; /* project/select kernel(s) (+ texel gather kernel on the host entry point) */
  float ortho_total_ms;
  int32_t dsm_kernel_launches;
  int32_t ortho_kernel_launches;
  int64_t dsm_points_binned;  /* points that fell inside the stripe + halo */
  int64_t dsm_cells_empty;    /* cells evaluated by the warp-per-cell kernel (empty primary ball / dense tiles) */
  int64_t ortho_h2d_bytes;    /* host entry point: bytes of frame sub-rectangles actually copied to the device */
} amb_timings;

typedef struct amb_ctx amb_ctx;

/* ---- library ---- */
int amb_abi_version(void);
const char* amb_status_string(int status);
/* Last CUDA/driver error text recorded on this context (never NULL). */
const char* amb_last_error(const amb_ctx* ctx);
/* Number of CUDA devices visible; negative amb_status on failure. */
int amb_device_count(void);

/* ---- geometry ---- */
/* grid_map::GridMap::setGeometry(Length(delta_easting, delta_northing), resolution, Position(center_easting,
 * center_northing)) as AerialGridMap::initialize calls it (aerial-mapper-grid-map.cc:30-33):
 * size = round(length / resolution), length = size * resolution. */
int amb_geometry_init(double delta_easting, double delta_northing, double resolution, double center_easting,
                      double center_northing, amb_geometry* out);
/* grid_map::GridMap::getPosition(Index(i, j)) (call sites dsm.cc:124-125, ortho-backward-grid.cc:149-150). */
int amb_geometry_position(const amb_geometry* geom, int32_t i, int32_t j, double* x, double* y);

/* ---- context ---- */
/* Create a context on `device` owning columns [col_begin, col_end) of the map.  Pass 0, geom->cols for the
 * whole map.  Device layer slabs are allocated lazily (first upload / init / process that touches them).
 * Limits: a context holds fewer than 2^32 - 1 cells, rows * (col_end - col_begin) (else AMB_ERR_UNSUPPORTED), and the
 * DSM and OrthoFromPcl take maps of fewer than 2^27 rows (else their process calls return AMB_ERR_UNSUPPORTED). */
int amb_create(const amb_geometry* geom, int device, int32_t col_begin, int32_t col_end, amb_ctx** out);
void amb_destroy(amb_ctx* ctx);
int amb_sync(amb_ctx* ctx);
/* The cudaStream_t the context enqueues on (as an opaque pointer), so callers holding device buffers can order
 * their own work against it. */
void* amb_stream(amb_ctx* ctx);

/* Set every layer slab to the value AerialGridMap::initialize gives it (aerial-mapper-grid-map.cc:40-48):
 * ortho=255, elevation=NaN, elevation_angle=0, num_observations=0, the rest NaN. */
int amb_init_layers(amb_ctx* ctx);
/* Copy one layer slab host->device / device->host.  `host_slab` points at element (0, col_begin), i.e. the
 * caller offsets a full-map pointer by rows*col_begin; rows*(col_end-col_begin) floats are moved. */
int amb_upload_layer(amb_ctx* ctx, int layer, const float* host_slab);
int amb_download_layer(amb_ctx* ctx, int layer, float* host_slab);
/* Set a layer slab from DEVICE memory valid on the context's device (rows*(col_end-col_begin) floats, e.g. an elevation
 * layer produced by another stage that never leaves HBM).  Asynchronous on the context's stream. */
int amb_upload_layer_device(amb_ctx* ctx, int layer, const float* device_slab);
/* Same, asynchronous: the copy is ordered after the work enqueued so far and runs on a second stream, so it
 * overlaps later kernels and host->device copies (use page-locked host memory); amb_sync() completes it. */
int amb_download_layer_async(amb_ctx* ctx, int layer, float* host_slab);
/* Register (or clear with NULL) a page-locked host slab as the MIRROR of a layer: every process() call then starts
 * copying that layer to it as soon as the layer is final (elevation right after the DSM kernels; elevation_angle
 * and observation_index right after the winners are selected, while the frame rectangles are still being
 * uploaded; the ortho layer after the texel gather), on a second stream.  amb_sync() completes the copies.  This is
 * the host-authoritative model of the reference (process() mutates the caller's map) without serialising PCIe. */
int amb_set_host_mirror(amb_ctx* ctx, int layer, float* host_slab);
/* Narrow transport for the mirrors of AMB_LAYER_ORTHO and AMB_LAYER_OBSERVATION_INDEX (others: AMB_ERR_INVALID_ARGUMENT),
 * on by default, enable = 0 turns it off: the layer crosses PCIe as one byte per cell and a pool of host threads inside
 * the library widens it to the float32 values of the mirror (amb_sync waits for them).  Whenever a value has no one-byte code — anything but the
 * integers 0..255 (`ortho`) / 0..254 and the canonical NaN (`observation_index`) — the layer travels as float32 as before:
 * the mirror always receives the layer's exact bits. */
int amb_set_host_mirror_compact(amb_ctx* ctx, int layer, int enable);
/* Device pointer of a layer slab (allocating it if needed), for device-side consumers (NCCL all-gather of
 * finished stripes, downstream kernels). */
int amb_layer_device_ptr(amb_ctx* ctx, int layer, float** device_slab);

/* ---- DSM: dsm::Dsm::process (dsm.cc:186-201) ---- */
/* xyz: n points, array-of-structs double[3], 24-byte stride — the memory layout of
 * AlignedType<std::vector, Eigen::Vector3d>::type (dsm.h:41-43).  interpolation_radius, center_easting and
 * center_northing are the dsm::Settings fields (dsm.h:25-32); the radius is an int compared against SQUARED
 * distances in m^2 (nanoflann RadiusResultSet, nanoflann.hpp:156-158).  n == 0 returns AMB_ERR_EMPTY and leaves
 * the elevation layer untouched (dsm.cc:189-192).  Result: the context's `elevation` slab. */
int amb_dsm_process(amb_ctx* ctx, const double* xyz, size_t n, int32_t interpolation_radius,
                    double center_easting, double center_northing);
int amb_dsm_process_device(amb_ctx* ctx, const double* d_xyz, size_t n, int32_t interpolation_radius,
                           double center_easting, double center_northing);
/* ---- DSM on a cloud that arrives sharded by column stripe (multi-GPU, SURVEY.md §8e) ----
 * Every point carries a caller-defined 64-bit id (< 2^32, unique over the whole cloud): it replaces "position in
 * the array" as the canonical summation-order key, so a stripe computed from {its own points + its neighbours'
 * border halos} is bit-identical to the same stripe of the undivided map. */
int amb_dsm_process_device_ids(amb_ctx* ctx, const double* d_xyz, const uint64_t* d_ids, size_t n,
                               int32_t interpolation_radius, double center_easting, double center_northing);
/* Average number of points per grid cell of the WHOLE cloud (n_global / (rows*cols)).  The bucket size and the
 * shared-memory stage are sized from the density; with a sharded cloud each rank sees only its share, so every
 * rank passes the same global figure to keep all summation orders — every output bit — independent of the
 * sharding.  0 (default): derive it from the points passed to each call. */
int amb_dsm_set_density_hint(amb_ctx* ctx, double points_per_cell);
/* Arithmetic of the tile gather's IDW weights and sums.  Neighbour SETS (d2 < threshold), retry levels and the NaN mask
 * are the reference's exact double-precision decisions in both modes.
 *   AMB_DSM_F32 (default): weights 1/d2 and both sums in float32 from tile-local coordinates and heights; any cell with a
 *       (cell, point) pair too close to the decision boundary for float32 to decide is re-evaluated in double, and so is
 *       any cell whose float32 height a rounding-error bound cannot place within 1e-4 relative of the reference's (a
 *       point close to the cell centre among contrasting heights, a tile height offset far from the cell's heights;
 *       DESIGN.md §4.1).  Every height is therefore within 1e-4 relative of the reference's; on terrain-like clouds
 *       almost all are within 1 float32 ulp.
 *   AMB_DSM_F64: everything in double in the reference's operation order (<= 1 float32 ulp by construction; ~2x slower). */
typedef enum amb_dsm_precision { AMB_DSM_F64 = 0, AMB_DSM_F32 = 1 } amb_dsm_precision;
int amb_dsm_set_precision(amb_ctx* ctx, int precision);
/* Default 4 (1 = off): with a host mirror registered for the output layer (amb_set_host_mirror), evaluate the map's
 * tile columns in `chunks` groups and start each group's download as soon as it is final, so that the layer's trip to the
 * host overlaps the evaluation of the remaining groups.  Same launches restricted to tile-column ranges: same output bits. */
int amb_dsm_set_stream_chunks(amb_ctx* ctx, int chunks);
/* The y-interval (y_lo, y_hi] covered by the cells of columns [col_begin, col_end) (points are assigned to the
 * rank whose interval holds y - center_easting), and how far a point can act across a stripe border. */
int amb_stripe_y_interval(const amb_geometry* geom, int32_t col_begin, int32_t col_end, double* y_lo, double* y_hi);
double amb_dsm_halo_reach(const amb_geometry* geom, int32_t interpolation_radius);
/* Compact the points within `reach` of the borders of (y_lo, y_hi] into d_out_* (device buffers of `capacity`
 * points): the border halo this rank contributes to the single all-gather.  *d_count = number found (may exceed
 * capacity: then the halo was truncated and the caller must retry with larger buffers).  Asynchronous. */
int amb_dsm_extract_halo(amb_ctx* ctx, const double* d_xyz, const uint64_t* d_ids, size_t n, double y_lo, double y_hi,
                         double reach, double center_easting, double* d_out_xyz, uint64_t* d_out_ids,
                         uint32_t capacity, uint32_t* d_count);

/* ---- the exchange step inside the library (multi-GPU, SURVEY.md §8e) ----
 * One context per GPU (one process per GPU, or several contexts in one process) joins an NCCL communicator; NCCL is
 * loaded at run time (dlopen of libnccl.so.2 — a process that already carries one, e.g. PyTorch's, shares it).
 *   rank 0:      amb_comm_unique_id(id)            128 bytes; distribute them to every rank by any means
 *   every rank:  amb_comm_init(ctx, rank, nranks, id)   (collective: blocks until all ranks have called it)
 * amb_destroy leaves the communicator. */
int amb_comm_unique_id(void* id128);
int amb_comm_init(amb_ctx* ctx, int rank, int nranks, const void* id128);
int amb_comm_destroy(amb_ctx* ctx);
/* How amb_dsm_process_sharded* exchanges the border halos: 0 (default) = automatic — with consecutive stripes, each at
 * least amb_dsm_halo_reach wide, only the two adjacent ranks need a rank's border points: the compaction kernel then
 * stores them straight into the neighbours' receive segments over NVLink peer memory (cudaIpc-mapped; counts and a step
 * stamp published with a system-scope release, the binning waits on them: no collective call in the step), or, where peer
 * mapping is unavailable, two ncclSend/ncclRecv pairs move the compacted lists; narrow or irregular stripes use one
 * ncclAllGather.  1 = always the all-gather; 2 = always neighbours (the caller guarantees the condition); 3 = neighbours
 * through ncclSend/ncclRecv only (no peer push).  Same value on every rank.  The first sharded call (and a later one
 * with a larger halo_capacity) exchanges the memory handles: a collective with one host synchronisation. */
int amb_comm_set_exchange(amb_ctx* ctx, int mode);
/* What the last amb_dsm_process_sharded* call used: 1 all-gather, 2 ncclSend/ncclRecv, 4 peer push (0: none yet). */
int amb_comm_last_exchange(const amb_ctx* ctx);
int amb_comm_size(const amb_ctx* ctx);
int amb_comm_rank(const amb_ctx* ctx);
/* Dsm::process on a cloud that arrives sharded by stripe, the exchange included: this rank's points (device memory, global
 * ids as in amb_dsm_process_device_ids; the rank owns the points whose y - center_easting lies in amb_stripe_y_interval of
 * its stripe, the outer ranks also what lies beyond the map) -> compaction of the points within amb_dsm_halo_reach of
 * the stripe borders -> ONE ncclAllGather of the halos (at most halo_capacity points per rank; a larger halo raises
 * AMB_ERR_SIZE_MISMATCH at the next amb_sync) -> binning over [own points | neighbours' halos] -> the stripe's elevation.
 * Everything is enqueued on the context's stream: no host synchronisation inside the step.  Collective: every rank of
 * the communicator must call it.  Without a communicator (or with one rank) it is amb_dsm_process_device_ids.
 * Bit-identical to the undivided map when every rank passes the same amb_dsm_set_density_hint. */
int amb_dsm_process_sharded_device(amb_ctx* ctx, const double* d_xyz, const uint64_t* d_ids, size_t n_local,
                                   int32_t interpolation_radius, double center_easting, double center_northing,
                                   uint32_t halo_capacity);
/* Same with this rank's points and ids in HOST memory (copied to the device inside; returns when the stripe's elevation
 * is final on the device — result layers travel through amb_set_host_mirror / amb_download_layer as usual). */
int amb_dsm_process_sharded(amb_ctx* ctx, const double* xyz, const uint64_t* ids, size_t n_local,
                            int32_t interpolation_radius, double center_easting, double center_northing,
                            uint32_t halo_capacity);

/* Ask the next amb_dsm_process* calls to also record, per cell of the slab, the number of neighbours that
 * entered the IDW sum (result_set.size(), dsm.cc:146) and the index k of the threshold lambda_k*radius that
 * produced them (0 = first query succeeded, 1.. = expanding-radius retries dsm.cc:133-144, -1 = cell untouched). */
int amb_dsm_enable_debug(amb_ctx* ctx, int enable);
int amb_dsm_download_debug(amb_ctx* ctx, int32_t* neighbour_count, int8_t* threshold_index);
/* The bins of the last binning on this context (Dsm, OrthoFromPcl, or the whole-map re-binning of an adaptive
 * OrthoFromPcl stripe), for tests of the binning stage.  Synchronises the context's stream; AMB_ERR_INVALID_ARGUMENT
 * before the first binning.  Every buffer may be NULL: a first call with NULL buffers but `layout` returns the sizes.
 *   layout         AMB_DSM_BINS_LAYOUT int32: B, Pa, BR, BC, KR, KC, gj0, tile_j0 (the plan's bin grid), n_binned, and
 *                  S, the number of coarse destinations the partition used
 *   bucket_starts  KR*KC + 1 uint32: record range [G[b], G[b + 1]) of bucket b = (bi >> log2 B) + (bj >> log2 B) * KR
 *   records        4 * n_binned doubles, bit for bit: x - center_northing, y - center_easting, z (OrthoFromPcl:
 *                  double(intensity)), and a word whose low 32 bits are the point's id (array position or caller id)
 *                  and high 32 bits (bi << 4) | (bj & 15)
 *   order          n_binned uint32: per bucket, its record positions by ascending id.  OrthoFromPcl orders every bucket;
 *                  Dsm only the buckets its warp-per-cell pass reads (the other entries are unspecified). */
#define AMB_DSM_BINS_LAYOUT 10
int amb_dsm_download_bins(amb_ctx* ctx, int32_t* layout, uint32_t* bucket_starts, double* records, uint32_t* order);
/* The thresholds lambda_k * radius the reference's retry loop visits (dsm.cc:133-144), computed with its exact
 * recurrence.  Returns the count (<= capacity) or a negative status. */
int amb_dsm_thresholds(int32_t interpolation_radius, double* thresholds, int32_t capacity);

/* ---- "next" row N1: ortho::OrthoFromPcl::process (aerial_mapper_ortho/src/ortho-from-pcl.cc:20-113) ----
 * IDW of point INTENSITIES into the `ortho` layer: the DSM kernels with z = double(intensities[i]), one radius query
 * (ortho::Settings::interpolation_radius of ortho-from-pcl.h:28-35, default 2, squared metres), no centre shift, and
 * a zero-distance point taken as a "perfect match" (:90-96) instead of a CHECK failure.  Cells without a neighbour
 * keep their value.  use_adaptive_interpolation != 0 (:63-72, off in the demo's flag file): a cell whose primary
 * ball is empty takes the IDW over the first non-empty ball of the thresholds 10*r, 100*r, 1000*r, ... (`int`
 * arithmetic in the reference, defined while 10^k * r <= INT_MAX), so every cell gets a value.  That mode needs the
 * WHOLE cloud in the call (on a stripe context too: the stripe then bins it a second time on the whole map's bin grid,
 * and amb_get_timings reports the points of that binning) and every point inside the map's bin grid (map + the apron
 * of the search radius); otherwise AMB_ERR_UNSUPPORTED and the layer keeps its content.
 * A stripe context gives, bit for bit, the same columns of the undivided map in both modes. */
int amb_ortho_from_pcl_process(amb_ctx* ctx, const double* xyz, const int32_t* intensities, size_t n,
                               int32_t interpolation_radius, int32_t use_adaptive_interpolation);
int amb_ortho_from_pcl_process_device(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities, size_t n,
                                      int32_t interpolation_radius, int32_t use_adaptive_interpolation);
/* ---- OrthoFromPcl on a cloud that arrives sharded by column stripe (multi-GPU; ortho-from-pcl.cc:20-113) ----
 * The counterparts of the DSM's sharded entry points above, with every point's intensity beside it.  Bit-identical to
 * the undivided map when every rank passes the same amb_dsm_set_density_hint.
 * _device_ids: d_ids (global ids < 2^32, unique over the whole cloud) replace the array position as the canonical
 * summation-order key, like amb_dsm_process_device_ids. */
int amb_ortho_from_pcl_process_device_ids(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities,
                                          const uint64_t* d_ids, size_t n, int32_t interpolation_radius,
                                          int32_t use_adaptive_interpolation);
/* amb_dsm_extract_halo with the intensities: the border halo's points, intensities and ids (d_ids may be NULL: array
 * positions) go to d_out_*; no centre shift.  Use the reach of amb_dsm_halo_reach (its thresholds include OrthoFromPcl's
 * single radius; extra halo points change no bit).  *d_count may exceed capacity (truncated halo).  Asynchronous. */
int amb_ortho_from_pcl_extract_halo(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities,
                                    const uint64_t* d_ids, size_t n, double y_lo, double y_hi, double reach,
                                    double* d_out_xyz, int32_t* d_out_intensities, uint64_t* d_out_ids,
                                    uint32_t capacity, uint32_t* d_count);
/* amb_dsm_process_sharded_device for OrthoFromPcl: the same exchange step (amb_comm_set_exchange, reported by
 * amb_comm_last_exchange; the records carry z = double(intensity)), then the stripe's `ortho`.  No adaptive mode: no rank
 * holds the whole cloud.  Collective; without a communicator (or with one rank) it is
 * amb_ortho_from_pcl_process_device_ids. */
int amb_ortho_from_pcl_process_sharded_device(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities,
                                              const uint64_t* d_ids, size_t n_local, int32_t interpolation_radius,
                                              uint32_t halo_capacity);
/* Same with this rank's points, intensities and ids in HOST memory; returns when the stripe's `ortho` is final on the
 * device. */
int amb_ortho_from_pcl_process_sharded(amb_ctx* ctx, const double* xyz, const int32_t* intensities, const uint64_t* ids,
                                       size_t n_local, int32_t interpolation_radius, uint32_t halo_capacity);

/* ---- "next" row N3: stereo::Densifier::computePointCloud (aerial_mapper_dense_pcl/src/densifier.cpp:25-108) ----
 * Disparity map -> world points, the step right before Dsm::process in the incremental pipeline
 * (stereo.cpp:149-193).  For every pixel in raster order with disparity > max_invalid_disparity
 * (Densifier::kMaxInvalidDisparity = 1): w = d / baseline; p = ((u-cx)/w, (fx/fy*v - cy*fx/fy)/w, fx/w);
 * P = R_G_C p + t_G_C1; kept unless (float)P.z is infinite.  Kept points (double[3]) and their gray values are
 * written in raster order (point_cloud_eigen / point_cloud_intensities).  K = {fx, fy, cx, cy}; R_G_C row-major.
 * *out_count = number of valid points (may exceed capacity: only the first `capacity` were written).
 * Strides are in elements (floats / bytes) per row and at least `width`; a smaller stride, a NULL pointer or a
 * width or height <= 0 returns AMB_ERR_INVALID_ARGUMENT, a zero baseline AMB_ERR_CHECK_FAILED. */
int amb_stereo_reproject(int device, const float* disparity, size_t disparity_stride, const uint8_t* image_left,
                         size_t image_stride, int32_t width, int32_t height, const double* K, double baseline,
                         const double* R_G_C, const double* t_G_C1, float max_invalid_disparity, double* out_xyz,
                         int32_t* out_intensity, size_t capacity, size_t* out_count);
/* Same with device buffers on `stream` (a cudaStream_t as void*, may be NULL); d_block_scratch needs
 * ceil(width*height/256) uint32; d_count receives the number of valid points.  Asynchronous. */
int amb_stereo_reproject_device(int device, void* stream, const float* d_disparity, size_t disparity_stride,
                                const uint8_t* d_image_left, size_t image_stride, int32_t width, int32_t height,
                                const double* K, double baseline, const double* R_G_C, const double* t_G_C1,
                                float max_invalid_disparity, double* d_out_xyz, int32_t* d_out_intensity,
                                size_t capacity, uint32_t* d_block_scratch, unsigned long long* d_count);

/* ---- "next" row N3, second half: stereo::Rectifier::rectifyStereoPair (aerial_mapper_dense_pcl/src/rectifier.cpp:36-107) ----
 * The step before block matching in the same pipeline.  Matrices are row-major 3x3 doubles; K is the full camera
 * matrix (stereo::StereoRigParameters::K, common.h:41).
 * setup (host arithmetic, no GPU; rectifier.cpp:43-79): Fusiello's compact rectification — baseline = |t_G_C2 - t_G_C1|,
 * R_G_C_rect (rows = new x/y/z axes; RectifiedStereoPair::R_G_C, what amb_stereo_reproject takes), and the two
 * rectifying homographies inverted and cast to float32 (T1_inv, T2_inv, 9 floats each, row-major).
 * A zero baseline or a singular matrix returns AMB_ERR_CHECK_FAILED. */
int amb_stereo_rectify_setup(const double* K, const double* R_G_C1, const double* R_G_C2, const double* t_G_C1,
                             const double* t_G_C2, double* baseline, double* R_G_C_rect, float* T1_inv,
                             float* T2_inv);
/* maps (rectifier.cpp:80-104): for every rectified pixel, [x y w]^T = T_i_inv [u v 1]^T in float32 and
 * map_rectify_i = (x / w, y / w) — the four CV_32FC1 maps cv::remap consumes; H x W, row stride map_stride floats.
 * w == 0 anywhere returns AMB_ERR_CHECK_FAILED (CHECK_NE(xyw(2), 0.0), :92,:99).  cv::remap and the contour mask
 * (OpenCV) stay with the caller, like block matching. */
int amb_stereo_rectify_maps(int device, const float* T1_inv, const float* T2_inv, int32_t width, int32_t height,
                            size_t map_stride, float* map1_x, float* map1_y, float* map2_x, float* map2_y);
/* Same with device maps on `stream` (a cudaStream_t as void*, may be NULL); T*_inv are HOST pointers (72 bytes of
 * kernel constants); d_zero_w_flag (nullable, int32 zeroed by the caller) is set to 1 if any w == 0.  Asynchronous. */
int amb_stereo_rectify_maps_device(int device, void* stream, const float* T1_inv, const float* T2_inv, int32_t width,
                                   int32_t height, size_t map_stride, float* d_map1_x, float* d_map1_y,
                                   float* d_map2_x, float* d_map2_y, int32_t* d_zero_w_flag);

/* ---- Orthomosaic: ortho::OrthoBackwardGrid::process (ortho-backward-grid.cc:223-239) ---- */
/* T_G_B: n poses, 7 doubles each in the order of the reference's pose files: x y z qw qx qy qz
 * (aerial-mapper-io.cc:110).  images: n host pointers to H x W x channels uint8 rasters with `row_step` bytes
 * per row (cv::Mat data/step); channels = 1 (CV_8UC1) or 3 (CV_8UC3, B,G,R byte order).  colored_ortho is
 * ortho::Settings::colored_ortho (ortho-backward-grid.h:39): non-zero writes the packed 0x00RRGGBB bit pattern
 * to `colored_ortho` and requires channels == 3, zero writes the gray value to `ortho` and requires
 * channels == 1.  Reads `elevation`; read-modify-writes `elevation_angle`; writes `observation_index`.
 * With HOST frames the winners are selected first (no pixel is touched), and only the bounding rectangle of the
 * pixels each frame actually contributes is copied to the device before the texels are gathered. */
int amb_ortho_process(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B, const uint8_t* const* images,
                      size_t n, int32_t channels, size_t row_step, int32_t colored_ortho);
/* Same with frames already resident on the context's device: d_images[i] are DEVICE pointers (the pointer
 * array itself is in host memory). */
int amb_ortho_process_device(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B,
                             const uint8_t* const* d_images, size_t n, int32_t channels, size_t row_step,
                             int32_t colored_ortho);
/* 0 = cull frames per tile with the conservative view-cone test (default), 1 = brute force over all frames
 * (the cull's own correctness reference). */
int amb_ortho_set_brute_force(amb_ctx* ctx, int brute_force);
/* Default 1 (0 = plain conservative list): per-tile DOMINANCE cull of the frame list.  A frame whose largest
 * possible observation angle over the tile is smaller — by a margin far above float32 rounding — than the smallest
 * possible one of a frame that sees every landmark of the tile can never end up as the winner of the reference's
 * running-maximum recurrence (ortho-backward-grid.cc:173-183) nor change who does, so it is not evaluated: same output
 * bits, ~1.2 instead of ~8.5 frames per cell at the benchmark geometry (tools/ortho_dominance_study.py). */
int amb_ortho_set_dominance_cull(amb_ctx* ctx, int enable);

/* ---- several GPUs of one process (SURVEY.md §8b: amb_create(geom, n_gpus)) ----
 * amb_multi owns one context per device 0..n_gpus-1, each with a contiguous column stripe (width ceil(cols / n_gpus)).
 * Entry points mirror the single-context ones with FULL host layers / the whole host cloud / all host frames, as the
 * reference's classes receive them (dsm.cc:186-201, ortho-backward-grid.cc:223-239); the stripes run concurrently.
 * DSM: every device gets the whole cloud over its own PCIe link and bins what reaches its stripe — nothing arrives sharded,
 * so this path has no exchange step (a cloud that arrives sharded uses amb_dsm_process_sharded* per context).  Every
 * stripe is bit-identical to the same columns of a single-GPU run. */
typedef struct amb_multi amb_multi;
int amb_multi_create(const amb_geometry* geom, int n_gpus, amb_multi** out);
void amb_multi_destroy(amb_multi* m);
int amb_multi_size(const amb_multi* m);                 /* stripes actually created (<= n_gpus) */
amb_ctx* amb_multi_context(amb_multi* m, int rank);     /* the stripe's context, for the per-context settings */
const char* amb_multi_last_error(const amb_multi* m);
int amb_multi_init_layers(amb_multi* m);
int amb_multi_upload_layer(amb_multi* m, int layer, const float* host_full);   /* rows x cols floats, column-major */
int amb_multi_download_layer(amb_multi* m, int layer, float* host_full);
int amb_multi_set_host_mirror(amb_multi* m, int layer, float* host_full);      /* page-locked; NULL clears */
int amb_multi_sync(amb_multi* m);
int amb_multi_dsm_process(amb_multi* m, const double* xyz, size_t n, int32_t interpolation_radius,
                          double center_easting, double center_northing);
int amb_multi_ortho_process(amb_multi* m, const amb_camera* camera, const double* T_G_B, const uint8_t* const* images,
                            size_t n, int32_t channels, size_t row_step, int32_t colored_ortho);
/* ortho::OrthoFromPcl::process (ortho-from-pcl.cc:20-113): like amb_multi_dsm_process, every device gets the whole cloud
 * with its intensities and the density n / (rows * cols); adaptive interpolation included. */
int amb_multi_ortho_from_pcl_process(amb_multi* m, const double* xyz, const int32_t* intensities, size_t n,
                                     int32_t interpolation_radius, int32_t use_adaptive_interpolation);

/* ---- export of a layer as a north-up georeferenced raster ("next" row N4) ----
 * Convention.  A map of rows x cols cells (rows = size(0) along x / easting, cols = size(1) along y / northing, cell
 * (0,0) at the max-x / max-y corner) is exported as an image W = rows pixels wide and H = cols pixels high, row-major,
 * north-up and east-right:
 *     pixel (r, c) = layer(i = rows - 1 - c, j = r)        r in [0, cols), c in [0, rows)
 * Image row r is layer column r read backwards: a per-column reversal plus a value conversion, no transpose.  A context
 * owning columns [col_begin, col_end) owns exactly image rows [col_begin, col_end), so stripes write disjoint, contiguous
 * bands of one image.  Geotransform in GDAL order (amb_raster_geotransform):
 *     gt = { pos_x - length_x/2, res, 0, pos_y + length_y/2, 0, -res }
 * The centre of pixel (r, c), (gt[0] + (c + 0.5) res, gt[3] - (r + 0.5) res), is amb_geometry_position(rows-1-c, r) up to
 * rounding.  Pixel formats (bytes per pixel):
 *   AMB_RASTER_F32    4  the layer's float32 bits, exactly (NaN payloads included: a DEM with NaN as no-data)
 *   AMB_RASTER_GRAY8  1  OpenCV saturate_cast<uchar>(float): round half to even, clamp to [0, 255]; NaN, +inf and every
 *                        value at or above 2^31 give 0 (cvRound's out-of-range result is INT_MIN, which saturates to 0)
 *   AMB_RASTER_BGR8   3  colored_ortho's packed 0x00RRGGBB bits as the bytes B, G, R (CV_8UC3 order), top byte ignored,
 *                        NaN -> 0, 0, 0; read as bits only, packed colours are float denormals
 *   AMB_RASTER_MASK8  1  0 where the layer is NaN (any payload), 255 elsewhere
 * `host_band` / `device_band` point at image row col_begin (the caller offsets a full-image pointer by
 * col_begin * rows * bytes-per-pixel, the slab convention of amb_upload_layer); exactly (col_end - col_begin) * rows *
 * bytes-per-pixel bytes are written, rows packed, at any byte alignment.  A NULL pointer, a bad layer or a bad format
 * returns AMB_ERR_INVALID_ARGUMENT and writes nothing. */
typedef enum amb_raster_format {
  AMB_RASTER_F32 = 0,
  AMB_RASTER_GRAY8 = 1,
  AMB_RASTER_BGR8 = 2,
  AMB_RASTER_MASK8 = 3
} amb_raster_format;
/* Host arithmetic, no GPU. */
int amb_raster_geotransform(const amb_geometry* geom, double gt[6]);
/* Synchronous: converted in HBM, then copied like amb_download_layer (pinned or pageable destination). */
int amb_export_raster(amb_ctx* ctx, int layer, int format, void* host_band);
/* Asynchronous on the context's stream, into device memory valid on the context's device. */
int amb_export_raster_device(amb_ctx* ctx, int layer, int format, void* device_band);
/* Every stripe of amb_multi writes its band of the caller's full image (rows x cols pixels), all devices at once. */
int amb_multi_export_raster(amb_multi* m, int layer, int format, void* host_image);

/* ---- import of a north-up raster into a layer, resampled to the map grid ----
 * Source.  A float32 band of width x height pixels, row-major, rows `row_stride` bytes apart (a multiple of 4, at least
 * 4 * width), with a GDAL-order geotransform gt[6] that is north-up (gt[2] == gt[4] == 0, gt[1] > 0, gt[5] < 0, all
 * finite): pixel (r, c) covers [gt0 + c gt1, gt0 + (c+1) gt1) x (gt3 + (r+1) gt5, gt3 + r gt5] (PixelIsArea, as
 * amb_raster_geotransform).  NaN is always no-data; with has_nodata, pixels that compare equal to `nodata` are no-data
 * too (IEEE equality: nodata 0 also matches -0).  The raster is in the map's planar frame (x = easting, y = northing,
 * the same projected CRS); nothing is reprojected.
 * Per-axis tables, host IEEE double: for every cell (i, j) of the context's stripe, (x_i, y_j) = amb_geometry_position(i, j)
 * (x depends on i only, y on j only), and
 *     u_i = (x_i - gt0) / gt1            v_j = (y_j - gt3) / gt5
 *     covered  iff  0 <= u_i < width  and  0 <= v_j < height          (else: the cell is untouched)
 *     NEAREST :  c = floor(u_i)                 r = floor(v_j)
 *     BILINEAR:  s = min(max(u_i - 0.5, 0), width - 1);  c0 = floor(s);  fx = s - c0
 *                if fx < 2^-20: fx = 0   elif fx > 1 - 2^-20: c0 += 1, fx = 0      (rows alike: t, r0, fy)
 * Per cell: NEAREST writes p = band[r][c] (its bits) unless p is no-data.  BILINEAR reads only the taps of non-zero
 * weight: row(r) = fx == 0 ? p(r, c0) : (1-fx) p(r, c0) + fx p(r, c0+1), h = fy == 0 ? row(r0) : (1-fy) row(r0) +
 * fy row(r0+1), in double, every operation rounded, no FMA contraction; the layer gets (float)h unless a tap it read is
 * no-data.  So a raster aligned with the map (same resolution, origin on a cell edge) is copied bit for bit by both
 * methods: importing an exported F32 layer gives the layer back, -0 included.  Cells outside the raster or fed by no-data
 * keep their value: importing tiles one after another mosaics them.
 * A NULL pointer, a bad layer or resample, width or height <= 0, a bad row_stride, a geotransform that is not north-up or
 * not finite, or a device band that is not 4-byte aligned returns AMB_ERR_INVALID_ARGUMENT and writes nothing.  A raster
 * that does not overlap the stripe returns AMB_OK and copies and writes nothing. */
typedef enum amb_resample { AMB_RESAMPLE_NEAREST = 0, AMB_RESAMPLE_BILINEAR = 1 } amb_resample;
/* Host band (pinned or pageable): only the window of rows and columns the stripe reads crosses PCIe; returns when the
 * band may be reused. */
int amb_import_raster(amb_ctx* ctx, int layer, const float* host_band, int32_t width, int32_t height, size_t row_stride,
                      const double gt[6], int has_nodata, float nodata, int resample);
/* Device band valid on the context's device, read in place; asynchronous on the context's stream. */
int amb_import_raster_device(amb_ctx* ctx, int layer, const float* device_band, int32_t width, int32_t height,
                             size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample);
/* Every stripe of amb_multi imports its own window of the same host band, all devices at once. */
int amb_multi_import_raster(amb_multi* m, int layer, const float* host_band, int32_t width, int32_t height,
                            size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample);
/* Host arithmetic, no GPU: the per-axis tables above for columns [col_begin, col_end) of `geom`.  src_col[rows] / fx[rows]
 * per cell row i and src_row[n] / fy[n] per column j = col_begin + k (n = col_end - col_begin); an index of -1 marks an
 * uncovered row or column (NEAREST: the fractions are 0).  What a caller needs to read only the window a stripe uses. */
int amb_raster_import_tables(const amb_geometry* geom, int32_t col_begin, int32_t col_end, int32_t width, int32_t height,
                             const double gt[6], int resample, int32_t* src_col, double* fx, int32_t* src_row,
                             double* fy);

/* ---- import of a Deflate-compressed (or uncompressed) TIFF band, inflated on the device ----
 * Convention.  One image (IFD) of a classic little-endian TIFF, described by amb_tiff_layout (the caller parses the
 * TIFF; the library never does): strips or tiles, PlanarConfiguration 1, Compression 1, 8 or 32946, Predictor 1, 2
 * (integer samples) or 3 (floating point), uint8, int16, uint16, int32, float32 or float64 samples, `spp` samples per
 * pixel of which band `band` is read.  The result is, bit for bit, the band as float32 the way numpy converts it
 * (a.astype(np.float32)): float32 samples are moved as bits (NaN payloads and -0 survive), int32 and float64 round to
 * nearest even, a float64 NaN stays a NaN (its payload is not promised).
 *   Chunks: chunk k of a tiled image is the tile at rows (k / across) * chunk_height, columns (k % across) *
 *     chunk_width (across = ceil(width / chunk_width)), every tile chunk_width x chunk_height pixels, the parts outside
 *     the image ignored; chunk k of a striped image (chunk_width == width) holds rows [k * chunk_height, + chunk_height)
 *     cut at the image's height.  A chunk's expected bytes are its rows x chunk_width x spp x the sample's bytes.
 *   Compressed chunk: one zlib stream (RFC 1950: CM 8, CINFO <= 7, a valid FCHECK, no preset dictionary) of RFC 1951
 *     stored, fixed and dynamic blocks, accepted as zlib.decompress accepts it: the stream must reach its final block
 *     and a correct Adler-32; bytes after the stream are ignored; it must inflate to at least the expected bytes, and
 *     bytes past them are ignored.  An uncompressed chunk must hold at least the expected bytes.
 *   Predictor, per predictor row (a tile row for tiles, an image row for strips): 2 adds each sample to the one spp
 *     samples before it, modulo the sample type; 3 (libtiff's floating-point predictor, the inverse of
 *     amb_deflate_strips_device's) adds each byte to the byte spp before it mod 256, over the row's big-endian byte
 *     planes, most significant plane first, then reassembles the samples.
 *   Corruption: a chunk that zlib.decompress would reject (a bad header, block type 3, an over-subscribed or incomplete
 *     code, a distance before the start of the output, a truncated stream, a wrong Adler-32, too few bytes) returns
 *     AMB_ERR_CORRUPT_DATA and nothing is written.  Only the chunks that intersect the rows and columns asked for are
 *     copied to the device and inflated: the others are never read, so their corruption is never seen.
 * Argument errors (AMB_ERR_INVALID_ARGUMENT, before anything is copied): a NULL pointer; width, height, chunk sides or
 * spp < 1; a band outside [0, spp); an unknown sample type, compression or predictor, or predictor 2 with float or 3
 * with integer samples; strips with chunk_width != width; n_chunks other than the chunk grid's count; a chunk whose
 * offset + byte count passes `bytes`; a chunk of more than 2^32 expected bytes.
 * Scratch, kept by the context: the window's float32 band, and chunks in groups whose compressed, inflated and 32 KB
 * window bytes stay under 1 GiB (a chunk that alone needs more forms a group of its own).
 * One warp inflates one zlib stream: an image stored as one strip inflates on one warp, slower than a host thread. */
typedef enum amb_sample_type {
  AMB_SAMPLE_U8 = 0, AMB_SAMPLE_I16 = 1, AMB_SAMPLE_U16 = 2, AMB_SAMPLE_I32 = 3, AMB_SAMPLE_F32 = 4, AMB_SAMPLE_F64 = 5
} amb_sample_type;
typedef struct amb_tiff_layout {
  int32_t width, height;             /* pixels */
  int32_t chunk_width, chunk_height; /* TileWidth x TileLength, or width x RowsPerStrip */
  int32_t tiled;                     /* 1: tiles, 0: strips */
  int32_t spp, band;                 /* samples per pixel, the one read */
  int32_t sample;                    /* amb_sample_type */
  int32_t compression;               /* 1, 8 or 32946 */
  int32_t predictor;                 /* 1, 2 or 3 */
  uint32_t n_chunks;
  uint32_t reserved_;
  const uint64_t* offsets;           /* [n_chunks]: StripOffsets / TileOffsets, into the file */
  const uint64_t* byte_counts;       /* [n_chunks]: StripByteCounts / TileByteCounts */
} amb_tiff_layout;
/* Decodes image rows [r0, r1) and columns [c0, c1) (0 <= r0 < r1 <= height, 0 <= c0 < c1 <= width) of the band into the
 * device float32 band d_band valid on the context's device (row r - r0 at d_band + (r - r0) * row_stride bytes, a
 * multiple of 4 of at least 4 (c1 - c0)), ordered after earlier work on the context's stream.  file: the whole file,
 * `bytes` long, in host memory (pinned or pageable).  Synchronous: corruption is found on the device. */
int amb_tiff_decode_device(amb_ctx* ctx, const void* file, size_t bytes, const amb_tiff_layout* layout, int32_t r0,
                           int32_t r1, int32_t c0, int32_t c1, float* d_band, size_t row_stride);
/* amb_import_raster of the decoded band (width x height, geotransform gt) with the same arguments and the same result:
 * only the window of rows and columns the stripe's import tables reference is decoded, so only the chunks it meets are
 * copied and inflated.  No overlap with the stripe: AMB_OK, nothing copied.  Returns when `file` may be reused. */
int amb_import_tiff(amb_ctx* ctx, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                    const double gt[6], int has_nodata, float nodata, int resample);
/* Every stripe of amb_multi decodes and imports its own window, all devices at once; a stripe whose window holds a
 * corrupt chunk leaves its layer untouched.  Returns the first stripe's non-OK status. */
int amb_multi_import_tiff(amb_multi* m, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                          const double gt[6], int has_nodata, float nodata, int resample);

/* ---- import of a longitude/latitude raster into a UTM map, every cell inverse-projected on the device ----
 * Frames.  The map's frame is a WGS84 UTM zone named by its EPSG code map_epsg: 32601-32660 (north, false northing 0)
 * or 32701-32760 (south, false northing 10^7).  A cell's position is amb_geometry_position's (easting, northing in that
 * zone, false easting and false northing included), exactly as amb_raster_geotransform states it.  The raster's frame is
 * geographic WGS84 (EPSG:4326): x = longitude, y = latitude, in degrees, with a north-up geotransform
 * (lon0, dlon, 0, lat0, 0, -dlat) and PixelIsArea pixels (read_geotiff already shifts a PixelIsPoint file's).  Any other
 * map_epsg, ETRS89, NAD83 and national grids included, returns AMB_ERR_INVALID_ARGUMENT.
 * Projection.  The inverse transverse Mercator as Krüger's series of order 6 in n (Karney 2011, "Transverse Mercator
 * with an accuracy of a few nanometers"; what PROJ and GeographicLib use) with a = 6378137, f = 1/298.257223563,
 * k0 = 0.9996, FE = 500000, lambda0 = 6 zone - 183 degrees; the conformal latitude goes to the geodetic one by two Newton
 * steps on tan(phi).  Every cell's (lon, lat) is within 1e-11 degrees (about 1 um) of a high-precision evaluation of the
 * same series, which is itself within a few nm of the exact projection within 3900 km of the central meridian.
 * Resampling.  Per cell, u = (lon - gt0) / gt1 and v = (lat - gt3) / gt5, each one IEEE double subtraction and one
 * division, no contraction; from (u, v) on, amb_resample's rule with u_i, v_j replaced by the cell's u, v: the same
 * coverage, taps, 2^-20 snap, rounded double blend, no-data and untouched cells.
 * Window.  For a host band or a TIFF, the host computes the raster window the stripe reads from the boundary cells of its
 * rectangle (longitude and isometric latitude are harmonic in easting and northing, so their extremes lie on the
 * boundary), one pixel wider on each side, clamped to the raster; only that window is copied (host band) or decoded
 * (TIFF).  A tap outside it (unreachable with the margin) fails the call with AMB_ERR_UNSUPPORTED instead of reading past
 * it.  A device band is read in place with no window: a raster that misses the stripe costs one launch, writes nothing
 * and returns AMB_OK.
 * Out of scope: datum shifts; geoid to ellipsoid heights (heights are imported as stored: SRTM and Copernicus heights
 * are geoid heights); wrapping across the antimeridian (longitudes past +-180 are not folded); polar (UPS) maps.  With a
 * host band or a TIFF, a map with a boundary cell whose position is not finite returns AMB_ERR_INVALID_ARGUMENT.
 * Arguments and results as amb_import_raster / amb_import_raster_device / amb_import_tiff / amb_multi_import_*, plus
 * map_epsg. */
int amb_import_raster_lonlat(amb_ctx* ctx, int layer, const float* host_band, int32_t width, int32_t height,
                             size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample,
                             int32_t map_epsg);
int amb_import_raster_lonlat_device(amb_ctx* ctx, int layer, const float* device_band, int32_t width, int32_t height,
                                    size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample,
                                    int32_t map_epsg);
int amb_multi_import_raster_lonlat(amb_multi* m, int layer, const float* host_band, int32_t width, int32_t height,
                                   size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample,
                                   int32_t map_epsg);
int amb_import_tiff_lonlat(amb_ctx* ctx, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                           const double gt[6], int has_nodata, float nodata, int resample, int32_t map_epsg);
int amb_multi_import_tiff_lonlat(amb_multi* m, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                                 const double gt[6], int has_nodata, float nodata, int resample, int32_t map_epsg);
/* Host arithmetic, no GPU: the window {c_lo, c_hi, r_lo, r_hi} (inclusive) of a width x height raster that the stripe
 * [col_begin, col_end) of `geom` reads, or {-1, -1, -1, -1} if the raster misses it.  What the imports above copy. */
int amb_lonlat_import_window(const amb_geometry* geom, int32_t col_begin, int32_t col_end, int32_t map_epsg,
                             int32_t width, int32_t height, const double gt[6], int32_t window[4]);
/* Test hook: (lon, lat) in degrees of every cell of the context's stripe, d_lonlat[2 ((j - col_begin) rows + i)] and
 * [.. + 1] (column-major like a layer), 8-byte-aligned device memory, computed by the device function the imports call;
 * asynchronous on the context's stream. */
int amb_lonlat_positions_device(amb_ctx* ctx, int32_t map_epsg, double* d_lonlat);

/* ---- baseline JPEG of an 8-bit raster ----
 * Convention.  The file is byte for byte what libjpeg(-turbo) writes (OpenCV cv2.imencode(".jpg", img, params)) for the
 * same image with its defaults: SOI; APP0 JFIF 1.01, density 1:1 without units; one DQT per table; SOF0 (baseline,
 * 8 bits); the standard Huffman tables of ITU-T T.81 Annex K as DHT DC0, AC0 (and DC1, AC1 for colour); DRI when the
 * restart interval is non-zero; one interleaved SOS; the entropy-coded data with RST0..7 markers; EOI.  Arithmetic:
 * islow integer DCT, quantisation tables of jpeg_set_quality(quality, force_baseline) for luma and chroma alike, and for
 * colour the 16-bit fixed-point RGB -> YCbCr conversion with, at 4:2:0, 2x2 averaging (bias 1, 2, 1, 2 ... along a row).
 * Inputs: channels 1 (GRAY8, one component) or 3 (BGR8 as B, G, R bytes, the export's order; YCbCr with three
 * components), width and height 1..65535, rows `row_stride` >= width * channels bytes apart, any byte alignment;
 * quality 1..100; sampling AMB_JPEG_420 or AMB_JPEG_444 (ignored for gray); restart_interval 0..65535 MCUs (0: no
 * restart markers).  Progressive, optimised Huffman tables and other samplings are not offered.
 * Errors: a NULL pointer, width or height <= 0, or a short row_stride returns AMB_ERR_INVALID_ARGUMENT; a parameter
 * outside the supported set (a side over 65535, channels, quality, sampling, restart interval) AMB_ERR_UNSUPPORTED.
 * Neither writes anything. */
typedef enum amb_jpeg_sampling { AMB_JPEG_420 = 0, AMB_JPEG_444 = 1, AMB_JPEG_422 = 2 /* decoder only */ } amb_jpeg_sampling;
/* Host arithmetic, no GPU: an upper bound on the file size (markers and byte stuffing included); 0 if unsupported. */
size_t amb_jpeg_max_size(int32_t width, int32_t height, int channels, int quality, int sampling,
                         int32_t restart_interval);
/* Encodes a device raster valid on the context's device, ordered after earlier work on the context's stream.
 * Synchronous: on return the *size bytes of the file are in host_out (pinned or pageable).  If capacity < the file's
 * size it returns AMB_ERR_SIZE_MISMATCH with the size needed in *size and writes nothing to host_out. */
int amb_jpeg_encode_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                           int channels, int quality, int sampling, int32_t restart_interval, void* host_out,
                           size_t capacity, size_t* size);
/* amb_export_raster_device of `layer` as AMB_RASTER_GRAY8 or AMB_RASTER_BGR8 into the context's scratch, then
 * amb_jpeg_encode_device of it: the context's band (image rows [col_begin, col_end)) as an image of its own. */
int amb_export_jpeg(amb_ctx* ctx, int layer, int format, int quality, int sampling, int32_t restart_interval,
                    void* host_out, size_t capacity, size_t* size);

/* ---- JPEG frames decoded on the device ----
 * Convention.  The output is byte for byte cv2.imread(path, IMREAD_COLOR) (channels 3: B, G, R bytes) or
 * cv2.imread(path, IMREAD_GRAYSCALE) (channels 1) of the same file, OpenCV 4.13 with libjpeg-turbo 3.1.2 at its default
 * decompression settings: islow integer IDCT (jidctint.c, with its `& RANGE_MASK` range limit), the DC predictor an
 * int stored as a 16-bit coefficient, fancy upsampling (jdsample.c h2v1 / h2v2 triangle filters; edges replicate the
 * last real chroma row or column; box replication when the chroma plane is at most 2 samples wide) and jdcolor.c's
 * table-based YCbCr -> BGR.  Gray output of a colour file is its Y plane; colour output of a gray file repeats the gray
 * value.
 * Supported: sequential baseline (SOF0) and extended sequential Huffman (SOF1) with 8-bit samples and one scan holding
 * every component; 1 component (gray) or 3 (YCbCr, JFIF) at 4:4:4, 4:2:2 (h2v1) or 4:2:0 (h2v2): luma factors 1x1,
 * 2x1 or 2x2, chroma 1x1; any DQT (8- or 16-bit) and DHT; any restart interval.  APPn and COM segments are skipped;
 * anything after the last MCU is ignored.  Refused with AMB_ERR_UNSUPPORTED, before anything is written: progressive,
 * arithmetic coding, 12/16-bit samples, lossless, hierarchical, multi-scan sequential, 2 or 4 components, an Adobe
 * segment (colour transforms, CMYK / YCCK), three components named R, G, B without JFIF, other sampling factors, DNL,
 * an EXIF orientation other than 1 (cv2.imread would rotate the image), Huffman tables the stream leaves out.  A stream
 * that is not JPEG or whose header is malformed returns AMB_ERR_INVALID_ARGUMENT.
 * Difference from cv2: a scan that is not valid for its header (a code no table holds, a run past coefficient 63, an
 * RSTn out of sequence or missing, an RSTn past those the restart interval calls for before the last MCU, data ending
 * before the last MCU) returns AMB_ERR_CORRUPT_DATA, where libjpeg-turbo warns and substitutes zeros. */
/* Host only, no GPU: parses and checks the header; sampling is an amb_jpeg_sampling (AMB_JPEG_444 for gray).  Any
 * output pointer may be NULL. */
int amb_jpeg_info(const void* file, size_t bytes, int32_t* width, int32_t* height, int* components, int* sampling,
                  int32_t* restart_interval);
/* Decodes n files in host memory (pinned or pageable) into device rasters d_out[i] (height rows of width * channels
 * bytes, row_step[i] bytes apart) on the context's stream, after earlier work on it.  Synchronous: corruption is found
 * on the device.  status[i] is that frame's result (AMB_OK, AMB_ERR_UNSUPPORTED, AMB_ERR_INVALID_ARGUMENT for a bad
 * header, a NULL destination or a short row_step, AMB_ERR_CORRUPT_DATA); a frame that fails is left unwritten and the
 * others are decoded.  Returns the first frame's non-OK status, or AMB_OK; AMB_ERR_INVALID_ARGUMENT for a NULL array or
 * channels other than 1 or 3.  The frames go through the kernels in groups whose device scratch stays under 1 GiB (a
 * frame that alone needs more forms a group of its own): the file and its unstuffed scan, 192 bytes per 8x8 block
 * (coefficients and planes) and 80 bytes per KB of scan. */
int amb_jpeg_decode_device(amb_ctx* ctx, const void* const* files, const size_t* file_bytes, size_t n, int channels,
                           void* const* d_out, const size_t* row_step, int* status);

/* amb_ortho_process with JPEG files (host memory, pinned or pageable) in place of decoded frames, the frames decoded on
 * the device as amb_jpeg_decode_device would (colored_ortho: BGR, else gray).  Every header is parsed first: a frame
 * whose size differs from the camera's returns AMB_ERR_SIZE_MISMATCH, one outside the supported set AMB_ERR_UNSUPPORTED
 * (a malformed one AMB_ERR_INVALID_ARGUMENT), and no layer is touched.  Then the winners are selected as
 * amb_ortho_process does, and only the frames that contribute are copied to the device and decoded, only the rows of
 * their bounding box of winner pixels (plus the MCU rows around them the upsampling needs).  A contributing frame whose
 * scan is corrupt returns AMB_ERR_CORRUPT_DATA: elevation_angle and observation_index then hold the selection and the
 * ortho layer is not written.  A frame that contributes nothing is never decoded, so its scan is not checked. */
int amb_ortho_process_jpeg(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B, const void* const* files,
                           const size_t* file_bytes, size_t n, int32_t colored_ortho);

/* ---- Deflate-compressed GeoTIFF strips ----
 * Convention.  The strips of a classic TIFF with Compression = 8 (Adobe Deflate), PlanarConfiguration 1 and
 * RowsPerStrip = rows_per_strip (a value over height means one strip), for a raster in one of the export's formats
 * (amb_raster_format; BGR8 arrives as B, G, R and is stored as R, G, B):
 *   Predictor 3 for AMB_RASTER_F32 (libtiff's floating-point predictor): each row's samples become big-endian byte
 *     planes, most significant plane first, then every byte but the row's first is replaced by its difference (mod 256)
 *     with the byte before it;
 *   Predictor 2 for AMB_RASTER_GRAY8, AMB_RASTER_BGR8, AMB_RASTER_MASK8: within each row, byte k minus byte k - spp,
 *     mod 256 (spp = 3 for BGR8, else 1).
 * Every strip (its rows' predicted bytes, n of them) is one zlib stream (RFC 1950 header 78 01, RFC 1951 blocks of at
 * most 65535 bytes each, the Adler-32 of the n bytes); matches never reach outside the strip, Huffman codes are at most
 * 15 bits and code-length codes at most 7.  A block whose coded size would exceed its stored size is stored, so a
 * strip is never longer than n + 5 ceil(n / 65535) + 6 bytes.  The bytes are a function of the raster, the format and
 * rows_per_strip only (not of the device, the launch schedule or earlier calls); they decode exactly, with zlib or any
 * TIFF reader, but are not promised to equal what zlib would write.
 * Errors: a NULL pointer, a bad format, width, height or rows_per_strip <= 0, a row_stride below the row's bytes, or an
 * F32 image or stride that is not a multiple of 4 bytes returns AMB_ERR_INVALID_ARGUMENT; a strip whose bound exceeds
 * 4 GiB AMB_ERR_UNSUPPORTED.  Neither writes anything. */
/* Host arithmetic, no GPU: the sum of the strips' bounds above; 0 if the arguments are invalid or unsupported. */
size_t amb_deflate_max_size(int32_t width, int32_t height, int format, int32_t rows_per_strip);
/* Compresses a device raster valid on the context's device (8-bit formats at any byte alignment), ordered after
 * earlier work on the context's stream.  Synchronous: on return the strips are in host_out back to back (*size bytes,
 * pinned or pageable) and strip_bytes[ceil(height / rows_per_strip)] holds each strip's length.  If capacity < *size it
 * returns AMB_ERR_SIZE_MISMATCH with the size needed in *size and writes nothing else.  Device scratch, kept by the
 * context: about 4.4x the raster's bytes at 8 KiB strips, plus ~1.3 KB per 13107 bytes of a strip and ~1.8 KB per
 * strip, so very short strips cost more than the raster. */
int amb_deflate_strips_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                              int format, int32_t rows_per_strip, void* host_out, size_t capacity, size_t* size,
                              uint32_t* strip_bytes);
/* amb_export_raster_device of `layer` in `format` into the context's scratch, then amb_deflate_strips_device of it: the
 * context's band (image rows [col_begin, col_end)) as an image of its own. */
int amb_export_deflate_strips(amb_ctx* ctx, int layer, int format, int32_t rows_per_strip, void* host_out,
                              size_t capacity, size_t* size, uint32_t* strip_bytes);

/* ---- Cloud-Optimized GeoTIFF tiles ----
 * Convention.  The tiles of a tiled, Deflate-compressed TIFF with internal overviews, for a raster in one of the export's
 * formats (amb_raster_format), width x height pixels, and a tile side T: a multiple of 16 with 16 <= T <= 4096.
 *   Levels: level 0 is the raster; level k + 1 is ceil(w_k / 2) x ceil(h_k / 2) (= ceil(W / 2^k), GDAL's size rule),
 *     added while level k is wider or taller than T.  A raster that fits one tile has no overviews.
 *   Reduction: level k + 1 from level k (not from level 0).  Pixel (y, x) reads the children (2y + a, 2x + b), a, b in
 *     {0, 1}, that lie inside level k (1 or 2 of them on the last row or column of an odd size):
 *       AMB_RASTER_F32: the children that are not NaN, summed in IEEE double in the order (0,0), (0,1), (1,0), (1,1)
 *         (the first one is the sum's start, so -0 survives), every operation rounded, no FMA; the sum divided by their
 *         count n and stored as (float).  A NaN result (n == 0, or +inf and -inf among the children) is stored as the
 *         quiet NaN 0x7FC00000, so NaN payloads never reach an overview.
 *       AMB_RASTER_GRAY8, AMB_RASTER_BGR8: per byte the rounded mean (sum + n / 2) / n in integers.
 *       AMB_RASTER_MASK8: the maximum, so the mask pyramid of a layer is "not NaN" of its F32 pyramid.
 *     This is the project's own box filter; it is not promised to equal any GDAL resampling.
 *   Tiles: each level is cut into ceil(w / T) x ceil(h / T) tiles, row-major; every tile is T x T pixels, those outside
 *     the level zero.  A tile is one zlib stream exactly as a strip of amb_deflate_strips_device (Predictor 3 for F32,
 *     2 for the 8-bit formats, BGR8 stored as RGB), a tile row of T pixels being the predictor's row, so a tile is never
 *     longer than n + 5 ceil(n / 65535) + 6 bytes for its n = T * T * bytes-per-pixel predicted bytes.
 *   Order: the smallest level's tiles first, then each larger level's, row-major within a level: the order of the
 *     tiles' data in the file.
 * Errors: those of amb_deflate_strips_device, and a bad T returns AMB_ERR_INVALID_ARGUMENT; a pyramid of more than
 * 2^31 - 1 tile rows in all AMB_ERR_UNSUPPORTED.  Neither writes anything. */
/* Host arithmetic, no GPU: the levels of a width x height raster at tile side `tile`; n_levels <= 32 entries of level_w
 * and level_h are written.  AMB_ERR_INVALID_ARGUMENT for a NULL pointer, width or height <= 0 or a bad tile side. */
int amb_cog_layout(int32_t width, int32_t height, int32_t tile, int32_t* n_levels, int32_t* level_w, int32_t* level_h);
/* Host arithmetic, no GPU: the sum of the tiles' bounds; 0 if the arguments are invalid or unsupported. */
size_t amb_cog_max_size(int32_t width, int32_t height, int format, int32_t tile);
/* Builds the pyramid, tiles it and compresses every tile on the device, for a raster valid on the context's device
 * (8-bit formats at any byte alignment), ordered after earlier work on the context's stream.  Synchronous: on return the
 * tiles are in host_out back to back in file order (*size bytes, pinned or pageable) and tile_bytes[] holds each tile's
 * length in the same order.  If capacity < *size it returns AMB_ERR_SIZE_MISMATCH with the size needed in *size and
 * writes nothing else.  Device scratch, kept by the context: the overview levels (about 1/3 of the raster), the stacked
 * tiles (the levels with their edge tiles padded) and the Deflate encoder's scratch for the stacked tiles. */
int amb_cog_tiles_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                         int format, int32_t tile, void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes);
/* amb_export_raster_device of `layer` in `format` into the context's scratch, then amb_cog_tiles_device of it: the
 * context's band (image rows [col_begin, col_end)) as an image of its own. */
int amb_export_cog_tiles(amb_ctx* ctx, int layer, int format, int32_t tile, void* host_out, size_t capacity,
                         size_t* size, uint32_t* tile_bytes);

/* ---- JPEG-compressed Cloud-Optimized GeoTIFF tiles, and 1-bit mask tiles ----
 * Convention.  The image tiles of a tiled TIFF with Compression 7 (JPEG) and JPEGTables, the layout GDAL writes with
 * COMPRESS=JPEG (PHOTOMETRIC=YCBCR for colour), for an AMB_RASTER_GRAY8 or AMB_RASTER_BGR8 raster.  Levels, reduction,
 * T x T tiles with the part outside the level zero, and the order (the smallest level first) are those of
 * amb_cog_tiles_device.
 *   Image tile: an abbreviated JPEG stream SOI, SOF0 (T x T), SOS, entropy-coded data, EOI, with no APP0, DQT, DHT or
 *     DRI.  Its entropy-coded data is exactly what cv2.imencode(".jpg", tile, [quality, sampling]) writes for the T x T
 *     tile image (convention of amb_jpeg_encode_device: quality 1..100, sampling AMB_JPEG_420 or AMB_JPEG_444 for BGR8,
 *     ignored for gray), so a tile is that file with its tables moved out.
 *   Tables: one stream per file, SOI, the DQT segments, the DHT segments, EOI, with the bytes cv2.imencode writes: the
 *     TIFF JPEGTables tag (347).  It depends on channels and quality only.
 *   Mask tile (amb_cog_mask_tiles_device): GDAL's internal mask, for an AMB_RASTER_MASK8 raster (e.g. the export of
 *     observation_index).  The pyramid is the MASK8 one (the maximum); every T x T tile is stored at 1 bit per pixel,
 *     most significant bit first, 1 where the MASK8 byte is not 0 (valid), rows of T / 8 bytes, padding 0; each tile is
 *     one zlib stream as in amb_cog_tiles_device but with no predictor (TIFF Predictor 1: libtiff has none for 1-bit
 *     samples), so never longer than n + 5 ceil(n / 65535) + 6 bytes for n = T * T / 8.
 * Inside, the stacked tiles are encoded as one JPEG image T wide and n_tiles * T high with a restart interval of
 * (T / 8)^2 MCUs (gray, 4:4:4) or (T / 16)^2 (4:2:0): one interval per tile.  A restart resets the DC predictors and pads
 * with 1 bits as the end of a separate stream does, so each interval's stuffed bytes are that tile's data.
 * Errors: those of amb_cog_tiles_device; a format other than GRAY8 / BGR8 (JPEG) returns AMB_ERR_INVALID_ARGUMENT, a
 * quality outside 1..100 or a bad sampling AMB_ERR_UNSUPPORTED.  Neither writes anything. */
/* Host arithmetic, no GPU: a bound on the tiles' total size (headers, byte stuffing and EOI included); 0 if the
 * arguments are invalid or unsupported. */
size_t amb_cog_jpeg_max_size(int32_t width, int32_t height, int format, int32_t tile, int quality, int sampling);
/* Host only, no GPU: the JPEGTables stream of channels 1 or 3 at `quality` into out (*size bytes, at most 600); a bad
 * channels or quality returns AMB_ERR_UNSUPPORTED, capacity < *size AMB_ERR_SIZE_MISMATCH with the size in *size. */
int amb_cog_jpeg_tables(int channels, int quality, void* out, size_t capacity, size_t* size);
/* As amb_cog_tiles_device, JPEG tiles: on return the tiles are in host_out back to back in file order (*size bytes,
 * pinned or pageable) and tile_bytes[] holds each tile's length.  If capacity < *size it returns AMB_ERR_SIZE_MISMATCH
 * with the size needed in *size and writes nothing else.  Device scratch, kept by the context: the overview levels, the
 * stacked tiles and the JPEG encoder's scratch for them (about 0.08 byte per stacked pixel at 4:2:0, 0.22 at 4:4:4,
 * plus the compressed tiles twice). */
int amb_cog_jpeg_tiles_device(amb_ctx* ctx, const void* d_image, int32_t width, int32_t height, size_t row_stride,
                              int format, int32_t tile, int quality, int sampling, void* host_out, size_t capacity,
                              size_t* size, uint32_t* tile_bytes);
/* amb_export_raster_device of `layer` as GRAY8 or BGR8, then amb_cog_jpeg_tiles_device of the context's band. */
int amb_export_cog_jpeg_tiles(amb_ctx* ctx, int layer, int format, int32_t tile, int quality, int sampling,
                              void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes);
/* Host arithmetic, no GPU: the sum of the mask tiles' bounds; 0 if the arguments are invalid or unsupported. */
size_t amb_cog_mask_max_size(int32_t width, int32_t height, int32_t tile);
/* The mask tiles of a MASK8 device raster (any byte alignment), with the contract of amb_cog_tiles_device. */
int amb_cog_mask_tiles_device(amb_ctx* ctx, const void* d_mask, int32_t width, int32_t height, size_t row_stride,
                              int32_t tile, void* host_out, size_t capacity, size_t* size, uint32_t* tile_bytes);
/* amb_export_raster_device of `layer` as AMB_RASTER_MASK8, then amb_cog_mask_tiles_device of the context's band. */
int amb_export_cog_mask_tiles(amb_ctx* ctx, int layer, int32_t tile, void* host_out, size_t capacity, size_t* size,
                              uint32_t* tile_bytes);

/* ---- measurement ---- */
int amb_get_timings(amb_ctx* ctx, amb_timings* out);

/* Host memory and transfer speed.  Every host entry point (amb_dsm_process, amb_ortho_process, amb_ortho_from_pcl_process,
 * amb_dsm_process_sharded, amb_upload_layer, amb_download_layer) accepts ordinary PAGEABLE memory — what the reference's
 * callers own (std::vector<Eigen::Vector3d>, cv::Mat, Eigen::MatrixXf storage) — as well as page-locked memory.
 * Pinned / registered buffers are copied directly (one asynchronous DMA at PCIe rate).  Pageable transfers of 4 MB and
 * more are staged by the library itself: a process-wide pool of worker threads (AMB_STAGING_THREADS, default 16) moves
 * the data through three pinned 32 MB slots per device, each slot's DMA overlapping the next slot's memcpy; the winners'
 * frame rectangles of amb_ortho_process are packed slot-wise.  Measured 2-4x faster than the driver's own staging of
 * pageable memory (AMB_STAGING_OFF=1 selects that, for comparison).  Host mirrors (amb_set_host_mirror) should be pinned (a pageable mirror works, but its copies are the driver's and do not overlap).
 * amb_host_alloc / amb_host_free: pinned host memory for callers that want full-rate copies inside process(). */
int amb_host_alloc(void** ptr, size_t bytes);
int amb_host_free(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* AERIAL_MAPPER_B200_H_ */
