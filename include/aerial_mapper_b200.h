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
  AMB_ERR_UNSUPPORTED = -8
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
  float dsm_bin_ms;      /* bin count + scan + scatter + in-bin canonical ordering */
  float dsm_gather_ms;   /* tile IDW gather kernel (the dominant DSM kernel) */
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
 * whole map.  Device layer slabs are allocated lazily (first upload / init / process that touches them). */
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
