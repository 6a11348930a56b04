// amb_api.cu — the extern "C" boundary (include/aerial_mapper_b200.h): context, layers, host entry points.
#include <cmath>
#include <cstdlib>
#include <limits>
#include <new>

#include "amb_context.h"
#include "jpeg_header.h"
#include "dsm_plan.h"

namespace amb {

__global__ void fill_kernel(float* p, size_t n, float v) {
  for (size_t k = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; k < n;
       k += static_cast<size_t>(gridDim.x) * blockDim.x)
    p[k] = v;
}

int wait_layer_copy(amb_ctx* ctx, int layer) {
  if (layer >= 0 && layer < AMB_NUM_LAYERS && ctx->layer_copy_pending[layer]) {
    AMB_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->layer_copy_event[layer], 0));
    ctx->layer_copy_pending[layer] = false;
  }
  return AMB_OK;
}

int enqueue_layer_download(amb_ctx* ctx, int layer, float* host_slab) {
  // ordered after everything enqueued so far on the compute stream, executed on the copy stream so that it
  // overlaps later kernels and host->device copies (PCIe is full duplex)
  AMB_CUDA(ctx, cudaEventRecord(ctx->copy_done[0], ctx->stream));
  AMB_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->copy_done[0], 0));
  AMB_CUDA(ctx, cudaMemcpyAsync(host_slab, ctx->layers[layer], ctx->slab_cells() * sizeof(float),
                                cudaMemcpyDeviceToHost, ctx->copy_stream));
  // later WRITERS of this layer on the compute stream wait for the copy (wait_layer_copy); readers do not
  if (!ctx->layer_copy_event[layer])
    AMB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->layer_copy_event[layer], cudaEventDisableTiming));
  AMB_CUDA(ctx, cudaEventRecord(ctx->layer_copy_event[layer], ctx->copy_stream));
  ctx->layer_copy_pending[layer] = true;
  return AMB_OK;
}

// Columns [col0, col1) of the slab (slab-local) to the layer's host mirror: the part of a layer that is already final
// while the rest is still being computed (chunked DSM, amb_dsm_set_stream_chunks).  Contiguous: layers are column-major.
int mirror_layer_columns(amb_ctx* ctx, int layer, int col0, int col1) {
  if (layer < 0 || layer >= AMB_NUM_LAYERS || !ctx->host_mirror[layer] || !ctx->layers[layer] || col1 <= col0)
    return AMB_OK;
  // column chunks always travel as float32; the expander pool may still be widening an earlier compact round into the mirror
  if (ctx->compact[layer].enabled) wait_compact_layer(ctx, layer);
  const size_t off = static_cast<size_t>(ctx->geom.rows) * static_cast<size_t>(col0);
  const size_t cnt = static_cast<size_t>(ctx->geom.rows) * static_cast<size_t>(col1 - col0);
  AMB_CUDA(ctx, cudaEventRecord(ctx->copy_done[0], ctx->stream));
  AMB_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->copy_done[0], 0));
  AMB_CUDA(ctx, cudaMemcpyAsync(ctx->host_mirror[layer] + off, ctx->layers[layer] + off, cnt * sizeof(float),
                                cudaMemcpyDeviceToHost, ctx->copy_stream));
  if (!ctx->layer_copy_event[layer])
    AMB_CUDA(ctx, cudaEventCreateWithFlags(&ctx->layer_copy_event[layer], cudaEventDisableTiming));
  AMB_CUDA(ctx, cudaEventRecord(ctx->layer_copy_event[layer], ctx->copy_stream));
  ctx->layer_copy_pending[layer] = true;
  return AMB_OK;
}

int mirror_layer(amb_ctx* ctx, int layer) {
  if (layer < 0 || layer >= AMB_NUM_LAYERS || !ctx->host_mirror[layer] || !ctx->layers[layer]) return AMB_OK;
  if (ctx->compact[layer].enabled && (layer == AMB_LAYER_ORTHO || layer == AMB_LAYER_OBSERVATION_INDEX))
    return mirror_layer_compact(ctx, layer);  // one byte per cell when every value has a code (amb_set_host_mirror_compact)
  return enqueue_layer_download(ctx, layer, ctx->host_mirror[layer]);
}

int ensure_counters(amb_ctx* ctx) {
  if (ctx->counters.ptr) return AMB_OK;
  AMB_CUDA(ctx, ctx->counters.reserve(CTR_COUNT * sizeof(unsigned int)));
  AMB_CUDA(ctx, cudaMemsetAsync(ctx->counters.ptr, 0, CTR_COUNT * sizeof(unsigned int), ctx->stream));
  return AMB_OK;
}

// AerialGridMap's initial value of a layer (aerial-mapper-grid-map.cc:40-48)
static float initial_value(int layer) {
  if (layer == AMB_LAYER_ORTHO) return 255.0f;
  if (layer == AMB_LAYER_ELEVATION_ANGLE || layer == AMB_LAYER_NUM_OBSERVATIONS) return 0.0f;
  return std::numeric_limits<float>::quiet_NaN();
}

static int fill_layer(amb_ctx* ctx, int layer) {
  wait_layer_copy(ctx, layer);
  fill_kernel<<<ctx->num_sms * 4, 256, 0, ctx->stream>>>(ctx->layers[layer], ctx->slab_cells(), initial_value(layer));
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

static int alloc_layer(amb_ctx* ctx, int layer) {
  if (ctx->layers[layer]) return AMB_OK;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  float* p = nullptr;
  AMB_CUDA(ctx, cudaMalloc(&p, ctx->slab_cells() * sizeof(float)));
  ctx->layers[layer] = p;
  ctx->layer_fresh[layer] = true;
  return AMB_OK;
}

int ensure_layer(amb_ctx* ctx, int layer) {
  if (layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  const int st = alloc_layer(ctx, layer);
  if (st != AMB_OK || !ctx->layer_fresh[layer]) return st;
  ctx->layer_fresh[layer] = false;
  return fill_layer(ctx, layer);
}

bool layer_is_fresh(const amb_ctx* ctx, int layer) {
  return !ctx->eager_layer_init && (!ctx->layers[layer] || ctx->layer_fresh[layer]);
}

int ensure_layer_overwrite(amb_ctx* ctx, int layer, bool* fresh) {
  if (layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  *fresh = false;
  if (ctx->eager_layer_init) return ensure_layer(ctx, layer);
  const int st = alloc_layer(ctx, layer);
  if (st != AMB_OK) return st;
  *fresh = ctx->layer_fresh[layer];
  ctx->layer_fresh[layer] = false;
  return AMB_OK;
}

// The flag travels through host-MAPPED memory (a store from a one-thread kernel), not through the device->host
// copy engine, where it would queue behind result layers still streaming to their host mirrors.
__global__ void flag_to_host_kernel(const unsigned int* __restrict__ src, unsigned int* __restrict__ dst) {
  *dst = *src;
  __threadfence_system();
}

static int finish_flags(amb_ctx* ctx, unsigned int offset_words, int err_code) {
  if (!ctx->host_flags)
    AMB_CUDA(ctx, cudaHostAlloc(reinterpret_cast<void**>(&ctx->host_flags), 64, cudaHostAllocMapped));
  unsigned int* mapped = nullptr;
  AMB_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&mapped), ctx->host_flags, 0));
  ctx->host_flags[0] = 0;
  flag_to_host_kernel<<<1, 1, 0, ctx->stream>>>(ctx->counters.as<unsigned int>() + offset_words, mapped);
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (!ctx->host_flags[0]) return AMB_OK;
  // reported: the sticky flag is cleared (ordered before any later kernel on the stream)
  AMB_CUDA(ctx, cudaMemsetAsync(ctx->counters.as<unsigned int>() + offset_words, 0, sizeof(unsigned int), ctx->stream));
  return err_code;
}

// One Dsm::process / OrthoFromPcl::process, wherever its inputs live: every amb_dsm_process* and
// amb_ortho_from_pcl_process* entry point is one call of run_cloud.
struct CloudCall {
  int mode = 0;           // 0 Dsm (elevation), 1 OrthoFromPcl (ortho): dsm_run's mode
  bool host = false;      // inputs in host memory: uploaded here, the call is synchronous
  bool sharded = false;   // a rank's share of a sharded cloud (the *_sharded* entry points)
  bool need_ids = false;  // NULL ids are rejected (sharded clouds, amb_ortho_from_pcl_process_device_ids)
  const double* xyz = nullptr;
  const int32_t* intensities = nullptr;  // mode 1 only
  const uint64_t* ids = nullptr;         // NULL: array positions are the canonical order
  size_t n = 0;
  int32_t radius = 0;
  double center_easting = 0.0, center_northing = 0.0;  // mode 0 only
  int32_t adaptive = 0;        // mode 1, not sharded: ortho-from-pcl.cc:63-72 (pcl_adaptive_kernels.cu)
  uint32_t halo_capacity = 0;  // sharded only
};

static int run_cloud(amb_ctx* ctx, const CloudCall& c) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  if (c.need_ids && !c.ids) return AMB_ERR_INVALID_ARGUMENT;
  const bool inputs = c.xyz && (c.mode == 0 || c.intensities);
  // A rank of a communicator may own no points of a sharded cloud, so its other arguments are checked before n and its
  // empty share still takes part in the exchange.  Without a communicator the share is the whole cloud.
  const bool exchange = c.sharded && ctx->comm_size > 1 && ctx->nccl_comm;
  if (c.sharded && (!inputs || c.radius < 1)) return AMB_ERR_INVALID_ARGUMENT;
  if (c.n == 0 && !exchange) return AMB_ERR_EMPTY;  // dsm.cc:189-192, CHECK(!pointcloud.empty()) ortho-from-pcl.cc:23
  if (!inputs) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));

  const double* xyz = c.xyz;
  const int* intensities = c.mode == 1 ? c.intensities : nullptr;
  const unsigned long long* ids = reinterpret_cast<const unsigned long long*>(c.ids);
  // The upload of a whole cloud is the "h2d" phase of the call's timings.  A sharded share is uploaded before the
  // timed region, whose "h2d" phase is the halo exchange (sharded_step); its buffers are never empty, so that a rank
  // without points still passes valid device pointers to the exchange.
  const bool timed_upload = c.host && !c.sharded;
  if (c.host) {
    const size_t cap = c.sharded ? std::max<size_t>(c.n, 1) : c.n;
    AMB_CUDA(ctx, ctx->points.reserve(cap * 3 * sizeof(double)));
    if (c.mode == 1) AMB_CUDA(ctx, ctx->intensities.reserve(cap * sizeof(int32_t)));
    if (c.sharded) AMB_CUDA(ctx, ctx->point_ids.reserve(cap * sizeof(uint64_t)));
    if (timed_upload) AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_BEGIN], ctx->stream));
    if (c.n) {
      const int st = staged_h2d(ctx, ctx->points.ptr, c.xyz, c.n * 3 * sizeof(double), ctx->stream);  // pageable clouds
      if (st != AMB_OK) return st;
      if (c.mode == 1)
        AMB_CUDA(ctx, cudaMemcpyAsync(ctx->intensities.ptr, c.intensities, c.n * sizeof(int32_t), cudaMemcpyHostToDevice,
                                      ctx->stream));
      if (c.sharded)
        AMB_CUDA(ctx, cudaMemcpyAsync(ctx->point_ids.ptr, c.ids, c.n * sizeof(uint64_t), cudaMemcpyHostToDevice,
                                      ctx->stream));
    }
    xyz = ctx->points.as<double>();
    if (c.mode == 1) intensities = ctx->intensities.as<int>();
    if (c.sharded) ids = ctx->point_ids.as<unsigned long long>();
    if (timed_upload) AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_H2D_END], ctx->stream));
  }

  int st;
  if (exchange) {
    // records its own events and sets dsm_timed
    st = sharded_step(ctx, xyz, intensities, reinterpret_cast<const uint64_t*>(ids), c.n, c.radius, c.center_easting,
                      c.center_northing, c.halo_capacity, c.mode);
  } else {
    if (!timed_upload) {  // inputs already on the device: an empty "h2d" phase
      AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_BEGIN], ctx->stream));
      AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_DSM_H2D_END], ctx->stream));
    }
    ctx->dsm_had_h2d = timed_upload;
    float* saved = nullptr;
    if (c.adaptive) {
      const int pst = pcl_adaptive_prepare(ctx, &saved);
      if (pst != AMB_OK)  // frees what prepare made; no pass ran, so the timings of the previous call stay
        return pcl_adaptive_finish(ctx, pst, xyz, ids, intensities, c.n, c.radius, saved);
    }
    st = dsm_run(ctx, xyz, ids, c.n, c.radius, c.center_easting, c.center_northing, c.mode, intensities);
    if (c.adaptive) st = pcl_adaptive_finish(ctx, st, xyz, ids, intensities, c.n, c.radius, saved);
    ctx->dsm_timed = (st == AMB_OK);
  }
  if (st != AMB_OK || !c.host) return st;
  // Host entry points return with their result final on the device.  amb_dsm_process also reports a point on a cell
  // centre at once, as the reference's Dsm::process does (CHECK in dsm.cc); the other host entry points leave their
  // sticky flags to amb_sync.
  if (c.mode == 0 && !c.sharded) return finish_flags(ctx, CTR_DSM_COINCIDENT, AMB_ERR_COINCIDENT_POINT);
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return AMB_OK;
}

// One OrthoBackwardGrid::process, wherever its frames live: every amb_ortho_process* entry point is one call of
// run_ortho.  Every argument is checked before any device work, so a refused call leaves the layers and the previous
// call's timings as they were.
static int run_ortho(amb_ctx* ctx, OrthoCall c) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  if (c.n == 0) return AMB_ERR_EMPTY;  // CHECK(!T_G_Bs.empty()), ortho-backward-grid.cc:225
  const bool jpeg = c.frames == OrthoCall::JPEG;
  if (!c.camera || !c.T_G_B || (jpeg ? !c.files || !c.file_bytes : !c.images)) return AMB_ERR_INVALID_ARGUMENT;
  const amb_camera& cam = *c.camera;
  if (cam.width <= 0 || cam.height <= 0) return AMB_ERR_SIZE_MISMATCH;
  std::vector<JpegFrame> headers(jpeg ? c.n : 0);  // every header before any device work
  for (size_t f = 0; f < c.n && c.frames != OrthoCall::DEVICE; ++f) {  // device frame pointers are not inspected
    if (jpeg ? !c.files[f] : !c.images[f]) return AMB_ERR_INVALID_ARGUMENT;
    if (!jpeg) continue;
    const int st = jpeg_parse(static_cast<const unsigned char*>(c.files[f]), c.file_bytes[f], &headers[f]);
    if (st != AMB_OK) return st;
  }
  for (const JpegFrame& h : headers)
    if (h.width != cam.width || h.height != cam.height) return AMB_ERR_SIZE_MISMATCH;
  c.headers = headers.data();
  if (jpeg) c.row_step = static_cast<size_t>(cam.width) * c.channels;  // decoded bands: rows of width * channels
  if (cam.width > 65535 || cam.height > 65535) return AMB_ERR_UNSUPPORTED;
  if (c.colored_ortho ? c.channels != 3 : c.channels != 1) return AMB_ERR_SIZE_MISMATCH;
  if (c.row_step < static_cast<size_t>(cam.width) * c.channels) return AMB_ERR_SIZE_MISMATCH;
  if (cam.dist_type < AMB_DIST_NONE || cam.dist_type > AMB_DIST_FOV) return AMB_ERR_UNSUPPORTED;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  ctx->ortho_timed = false;  // the events below are this call's: its timings stand only if it succeeds
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_ORTHO_BEGIN], ctx->stream));
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_ORTHO_H2D_END], ctx->stream));
  ctx->ortho_two_phase = c.frames != OrthoCall::DEVICE;
  const int st = ortho_run(ctx, c);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_ORTHO_END], ctx->stream));
  ctx->ortho_timed = true;
  // host and JPEG frames return with their result final and CHECK(alpha > 0) reported; device frames leave it to amb_sync
  return c.frames == OrthoCall::DEVICE ? AMB_OK : finish_flags(ctx, CTR_ORTHO_CHECK, AMB_ERR_CHECK_FAILED);
}

}  // namespace amb

using namespace amb;

extern "C" {

int amb_abi_version(void) { return AMB_ABI_VERSION; }

const char* amb_status_string(int status) {
  switch (status) {
    case AMB_OK: return "ok";
    case AMB_ERR_EMPTY: return "empty input";
    case AMB_ERR_SIZE_MISMATCH: return "size mismatch";
    case AMB_ERR_COINCIDENT_POINT: return "a point coincides with a cell centre (reference CHECK(distances[i] > 0.0))";
    case AMB_ERR_CUDA: return "CUDA error";
    case AMB_ERR_INVALID_ARGUMENT: return "invalid argument";
    case AMB_ERR_CHECK_FAILED: return "reference CHECK(alpha > 0.0) failed";
    case AMB_ERR_NO_DEVICE: return "no CUDA device";
    case AMB_ERR_UNSUPPORTED: return "unsupported configuration";
    case AMB_ERR_CORRUPT_DATA: return "corrupt data";
    default: return "unknown status";
  }
}

const char* amb_last_error(const amb_ctx* ctx) { return ctx ? ctx->last_error.c_str() : ""; }

int amb_device_count(void) {
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return AMB_ERR_NO_DEVICE;
  }
  return n;
}

int amb_geometry_init(double delta_easting, double delta_northing, double resolution, double center_easting,
                      double center_northing, amb_geometry* out) {
  if (!out || !(resolution > 0.0) || !(delta_easting > 0.0) || !(delta_northing > 0.0))
    return AMB_ERR_INVALID_ARGUMENT;
  // grid_map::GridMap::setGeometry: size = round(length / resolution); length = size * resolution.
  out->rows = static_cast<int32_t>(std::round(delta_easting / resolution));
  out->cols = static_cast<int32_t>(std::round(delta_northing / resolution));
  if (out->rows <= 0 || out->cols <= 0) return AMB_ERR_INVALID_ARGUMENT;
  out->resolution = resolution;
  out->length_x = out->rows * resolution;
  out->length_y = out->cols * resolution;
  out->pos_x = center_easting;
  out->pos_y = center_northing;
  return AMB_OK;
}

int amb_geometry_position(const amb_geometry* g, int32_t i, int32_t j, double* x, double* y) {
  if (!g || !x || !y) return AMB_ERR_INVALID_ARGUMENT;
  if (i < 0 || j < 0 || i >= g->rows || j >= g->cols) return AMB_ERR_SIZE_MISMATCH;
  // grid_map::getPositionFromIndex: (mapPosition + (0.5*length - 0.5*res)) + res * (-(double)index)
  *x = (g->pos_x + (0.5 * g->length_x - 0.5 * g->resolution)) + g->resolution * (-static_cast<double>(i));
  *y = (g->pos_y + (0.5 * g->length_y - 0.5 * g->resolution)) + g->resolution * (-static_cast<double>(j));
  return AMB_OK;
}

int amb_create(const amb_geometry* geom, int device, int32_t col_begin, int32_t col_end, amb_ctx** out) {
  if (!geom || !out) return AMB_ERR_INVALID_ARGUMENT;
  if (geom->rows <= 0 || geom->cols <= 0 || !(geom->resolution > 0.0)) return AMB_ERR_INVALID_ARGUMENT;
  if (col_begin < 0 || col_end > geom->cols || col_begin >= col_end) return AMB_ERR_SIZE_MISMATCH;
  if (static_cast<size_t>(geom->rows) * static_cast<size_t>(col_end - col_begin) >= size_t(0xffffffffu))
    return AMB_ERR_UNSUPPORTED;
  int n = amb_device_count();
  if (n <= 0) return AMB_ERR_NO_DEVICE;
  if (device < 0 || device >= n) return AMB_ERR_INVALID_ARGUMENT;
  amb_ctx* ctx = new (std::nothrow) amb_ctx();
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  ctx->geom = *geom;
  ctx->device = device;
  ctx->col_begin = col_begin;
  ctx->col_end = col_end;
  // process-wide override of the gather's default arithmetic (amb_dsm_set_precision still wins per context): lets the
  // same test suite / demo binary run in either mode without code changes
  if (const char* p = std::getenv("AMB_DSM_PRECISION")) {
    if (p[0] == 'f' && p[1] == '6') ctx->dsm_precision = AMB_DSM_F64;
    if (p[0] == 'f' && p[1] == '3') ctx->dsm_precision = AMB_DSM_F32;
  }
  // A/B switch of the deferred reset (amb_init_layers): 1 fills every existing slab at once, as a separate pass
  if (const char* p = std::getenv("AMB_EAGER_LAYER_INIT")) ctx->eager_layer_init = p[0] == '1';
  cudaError_t e = cudaSetDevice(device);
#ifdef AMB_CUDA_EMU  // tests/emu (CPU emulation of the kernel source): grid-stride launches need no more blocks than this
  ctx->num_sms = 2;
#else
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&ctx->num_sms, cudaDevAttrMultiProcessorCount, device);
#endif
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&ctx->scatter_stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->scatter_start, cudaEventDisableTiming);
  for (int k = 0; k < EV_COUNT && e == cudaSuccess; ++k) e = cudaEventCreate(&ctx->events[k]);
  for (int k = 0; k < 2 && e == cudaSuccess; ++k) e = cudaEventCreateWithFlags(&ctx->copy_done[k], cudaEventDisableTiming);
  if (e != cudaSuccess) {
    cudaGetLastError();
    amb_destroy(ctx);
    return AMB_ERR_CUDA;
  }
  *out = ctx;
  return AMB_OK;
}

void amb_destroy(amb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  if (ctx->scatter_stream) cudaStreamSynchronize(ctx->scatter_stream);  // (joined by `stream` unless a DSM call failed)
  amb_comm_destroy(ctx);
  ctx->halo_send.release();
  ctx->halo_recv.release();
  release_compact_mirrors(ctx);
  for (int l = 0; l < AMB_NUM_LAYERS; ++l)
    if (ctx->layers[l]) cudaFree(ctx->layers[l]);
  DeviceBuffer* bufs[] = {&ctx->points,  &ctx->point_ids, &ctx->intensities, &ctx->records, &ctx->records_tmp, &ctx->tile_offsets, &ctx->point_order, &ctx->bucket_flags,
                            &ctx->bin_starts, &ctx->block_sums, &ctx->empty_cells,
                          &ctx->counters, &ctx->dbg_count, &ctx->dbg_level,  &ctx->raster_band, &ctx->raster_taps, &ctx->jpeg_mcu, &ctx->jpeg_spine, &ctx->jpeg_words, &ctx->jpeg_out, &ctx->jdec_files, &ctx->jdec_stream, &ctx->jdec_meta, &ctx->jdec_subs, &ctx->jdec_coef, &ctx->deflate_scratch, &ctx->deflate_words, &ctx->cog_levels, &ctx->cog_tiles, &ctx->tiff_files, &ctx->tiff_inflated, &ctx->tiff_meta, &ctx->frames,     &ctx->frame_table,
                          &ctx->frame_cull, &ctx->frame_rects, &ctx->ortho_pix, &ctx->ortho_bbox};
  for (DeviceBuffer* b : bufs) b->release();
  for (int k = 0; k < EV_COUNT; ++k)
    if (ctx->events[k]) cudaEventDestroy(ctx->events[k]);
  if (ctx->scatter_start) cudaEventDestroy(ctx->scatter_start);
  for (cudaEvent_t e : ctx->band_done) cudaEventDestroy(e);
  for (int k = 0; k < 2; ++k)
    if (ctx->copy_done[k]) cudaEventDestroy(ctx->copy_done[k]);
  for (int l = 0; l < AMB_NUM_LAYERS; ++l)
    if (ctx->layer_copy_event[l]) cudaEventDestroy(ctx->layer_copy_event[l]);
  if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
  for (int k = 0; k < 2; ++k) {
    ctx->stages[k].release();
    if (ctx->stage_events[k]) cudaEventDestroy(ctx->stage_events[k]);
  }
  if (ctx->host_flags) cudaFreeHost(ctx->host_flags);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
  if (ctx->scatter_stream) cudaStreamDestroy(ctx->scatter_stream);
  delete ctx;
}

int amb_sync(amb_ctx* ctx) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
  const int compact_status = join_compact_mirrors(ctx);  // host threads widening one-byte codes (opt-in; none otherwise)
  for (int l = 0; l < AMB_NUM_LAYERS; ++l) ctx->layer_copy_pending[l] = false;
  if (compact_status != AMB_OK) return compact_status;
  // Deferred reference CHECKs of the asynchronous `_device` entry points.
  if (ctx->counters.ptr) {
    unsigned int c[CTR_COUNT];
    AMB_CUDA(ctx, cudaMemcpy(c, ctx->counters.ptr, sizeof(c), cudaMemcpyDeviceToHost));
    if (c[CTR_DSM_COINCIDENT] || c[CTR_ORTHO_CHECK] || c[CTR_HALO_OVERFLOW]) {  // reported once, then cleared
      unsigned int* d = ctx->counters.as<unsigned int>();
      AMB_CUDA(ctx, cudaMemset(d + CTR_DSM_COINCIDENT, 0, sizeof(unsigned int)));
      AMB_CUDA(ctx, cudaMemset(d + CTR_ORTHO_CHECK, 0, sizeof(unsigned int)));
      AMB_CUDA(ctx, cudaMemset(d + CTR_HALO_OVERFLOW, 0, sizeof(unsigned int)));
    }
    if (c[CTR_HALO_OVERFLOW]) {
      ctx->last_error = "a rank's border halo exceeded halo_capacity (amb_dsm_process_sharded_device): result incomplete";
      return AMB_ERR_SIZE_MISMATCH;
    }
    if (c[CTR_DSM_COINCIDENT]) return AMB_ERR_COINCIDENT_POINT;
    if (c[CTR_ORTHO_CHECK]) return AMB_ERR_CHECK_FAILED;
  }
  return AMB_OK;
}

void* amb_stream(amb_ctx* ctx) { return ctx ? static_cast<void*>(ctx->stream) : nullptr; }

int amb_init_layers(amb_ctx* ctx) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  for (int l = 0; l < AMB_NUM_LAYERS; ++l) {
    // Slabs are allocated lazily and start fresh, so only the ones that already exist need resetting.  The reset is
    // deferred: the next ensure_layer fills the slab, and a writer of every cell (ensure_layer_overwrite) stores the
    // initial values itself, which spares a pass over the slab.
    if (!ctx->layers[l]) continue;
    wait_layer_copy(ctx, l);
    ctx->layer_fresh[l] = true;
    if (ctx->eager_layer_init) {
      const int st = ensure_layer(ctx, l);
      if (st != AMB_OK) return st;
    }
  }
  return AMB_OK;
}

int amb_upload_layer(amb_ctx* ctx, int layer, const float* host_slab) {
  if (!ctx || !host_slab) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  bool fresh;  // the copy writes every cell
  int st = ensure_layer_overwrite(ctx, layer, &fresh);
  if (st != AMB_OK) return st;
  wait_layer_copy(ctx, layer);
  st = staged_h2d(ctx, ctx->layers[layer], host_slab, ctx->slab_cells() * sizeof(float), ctx->stream);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return AMB_OK;
}

int amb_upload_layer_device(amb_ctx* ctx, int layer, const float* device_slab) {
  if (!ctx || !device_slab) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  bool fresh;  // the copy writes every cell
  int st = ensure_layer_overwrite(ctx, layer, &fresh);
  if (st != AMB_OK) return st;
  wait_layer_copy(ctx, layer);
  AMB_CUDA(ctx, cudaMemcpyAsync(ctx->layers[layer], device_slab, ctx->slab_cells() * sizeof(float),
                                cudaMemcpyDeviceToDevice, ctx->stream));
  return AMB_OK;
}

int amb_download_layer(amb_ctx* ctx, int layer, float* host_slab) {
  if (!ctx || !host_slab) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  int st = ensure_layer(ctx, layer);
  if (st != AMB_OK) return st;
  return staged_d2h(ctx, host_slab, ctx->layers[layer], ctx->slab_cells() * sizeof(float), ctx->stream);
}

int amb_download_layer_async(amb_ctx* ctx, int layer, float* host_slab) {
  if (!ctx || !host_slab) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  int st = ensure_layer(ctx, layer);
  if (st != AMB_OK) return st;
  return enqueue_layer_download(ctx, layer, host_slab);
}

int amb_set_host_mirror(amb_ctx* ctx, int layer, float* host_slab) {
  if (!ctx || layer < 0 || layer >= AMB_NUM_LAYERS) return AMB_ERR_INVALID_ARGUMENT;
  ctx->host_mirror[layer] = host_slab;
  return AMB_OK;
}

int amb_layer_device_ptr(amb_ctx* ctx, int layer, float** device_slab) {
  if (!ctx || !device_slab) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  int st = ensure_layer(ctx, layer);
  if (st != AMB_OK) return st;
  *device_slab = ctx->layers[layer];
  return AMB_OK;
}

// ---- DSM and OrthoFromPcl ("next" row N1, SURVEY.md §8f) ----
int amb_dsm_process(amb_ctx* ctx, const double* xyz, size_t n, int32_t interpolation_radius,
                    double center_easting, double center_northing) {
  return run_cloud(ctx, {.mode = 0, .host = true, .xyz = xyz, .n = n, .radius = interpolation_radius,
                         .center_easting = center_easting, .center_northing = center_northing});
}

int amb_dsm_process_device(amb_ctx* ctx, const double* d_xyz, size_t n, int32_t interpolation_radius,
                           double center_easting, double center_northing) {
  return run_cloud(ctx, {.mode = 0, .xyz = d_xyz, .n = n, .radius = interpolation_radius,
                         .center_easting = center_easting, .center_northing = center_northing});
}

int amb_dsm_process_device_ids(amb_ctx* ctx, const double* d_xyz, const uint64_t* d_ids, size_t n,
                               int32_t interpolation_radius, double center_easting, double center_northing) {
  return run_cloud(ctx, {.mode = 0, .xyz = d_xyz, .ids = d_ids, .n = n, .radius = interpolation_radius,
                         .center_easting = center_easting, .center_northing = center_northing});
}

int amb_dsm_process_sharded(amb_ctx* ctx, const double* xyz, const uint64_t* ids, size_t n_local,
                            int32_t interpolation_radius, double center_easting, double center_northing,
                            uint32_t halo_capacity) {
  return run_cloud(ctx, {.mode = 0, .host = true, .sharded = true, .need_ids = true, .xyz = xyz, .ids = ids,
                         .n = n_local, .radius = interpolation_radius, .center_easting = center_easting,
                         .center_northing = center_northing, .halo_capacity = halo_capacity});
}

int amb_dsm_process_sharded_device(amb_ctx* ctx, const double* d_xyz, const uint64_t* d_ids, size_t n_local,
                                   int32_t interpolation_radius, double center_easting, double center_northing,
                                   uint32_t halo_capacity) {
  return run_cloud(ctx, {.mode = 0, .sharded = true, .need_ids = true, .xyz = d_xyz, .ids = d_ids, .n = n_local,
                         .radius = interpolation_radius, .center_easting = center_easting,
                         .center_northing = center_northing, .halo_capacity = halo_capacity});
}

int amb_ortho_from_pcl_process(amb_ctx* ctx, const double* xyz, const int32_t* intensities, size_t n,
                               int32_t interpolation_radius, int32_t use_adaptive_interpolation) {
  return run_cloud(ctx, {.mode = 1, .host = true, .xyz = xyz, .intensities = intensities, .n = n,
                         .radius = interpolation_radius, .adaptive = use_adaptive_interpolation});
}

int amb_ortho_from_pcl_process_device(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities, size_t n,
                                      int32_t interpolation_radius, int32_t use_adaptive_interpolation) {
  return run_cloud(ctx, {.mode = 1, .xyz = d_xyz, .intensities = d_intensities, .n = n,
                         .radius = interpolation_radius, .adaptive = use_adaptive_interpolation});
}

int amb_ortho_from_pcl_process_device_ids(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities,
                                          const uint64_t* d_ids, size_t n, int32_t interpolation_radius,
                                          int32_t use_adaptive_interpolation) {
  return run_cloud(ctx, {.mode = 1, .need_ids = true, .xyz = d_xyz, .intensities = d_intensities, .ids = d_ids,
                         .n = n, .radius = interpolation_radius, .adaptive = use_adaptive_interpolation});
}

int amb_ortho_from_pcl_process_sharded(amb_ctx* ctx, const double* xyz, const int32_t* intensities, const uint64_t* ids,
                                       size_t n_local, int32_t interpolation_radius, uint32_t halo_capacity) {
  return run_cloud(ctx, {.mode = 1, .host = true, .sharded = true, .need_ids = true, .xyz = xyz,
                         .intensities = intensities, .ids = ids, .n = n_local, .radius = interpolation_radius,
                         .halo_capacity = halo_capacity});
}

int amb_ortho_from_pcl_process_sharded_device(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities,
                                              const uint64_t* d_ids, size_t n_local, int32_t interpolation_radius,
                                              uint32_t halo_capacity) {
  return run_cloud(ctx, {.mode = 1, .sharded = true, .need_ids = true, .xyz = d_xyz, .intensities = d_intensities,
                         .ids = d_ids, .n = n_local, .radius = interpolation_radius, .halo_capacity = halo_capacity});
}

int amb_ortho_from_pcl_extract_halo(amb_ctx* ctx, const double* d_xyz, const int32_t* d_intensities,
                                    const uint64_t* d_ids, size_t n, double y_lo, double y_hi, double reach,
                                    double* d_out_xyz, int32_t* d_out_intensities, uint64_t* d_out_ids,
                                    uint32_t capacity, uint32_t* d_count) {
  if (!ctx || !d_xyz || !d_intensities || !d_out_xyz || !d_out_intensities || !d_out_ids || !d_count)
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return dsm_extract_halo(ctx, d_xyz, reinterpret_cast<const unsigned long long*>(d_ids), n, y_lo, y_hi, reach, 0.0,
                          d_out_xyz, reinterpret_cast<unsigned long long*>(d_out_ids), capacity, d_count, d_intensities,
                          d_out_intensities);
}

int amb_dsm_set_stream_chunks(amb_ctx* ctx, int chunks) {
  if (!ctx || chunks < 1) return AMB_ERR_INVALID_ARGUMENT;
  ctx->dsm_stream_chunks = chunks;
  return AMB_OK;
}

int amb_dsm_set_precision(amb_ctx* ctx, int precision) {
  if (!ctx || (precision != AMB_DSM_F64 && precision != AMB_DSM_F32)) return AMB_ERR_INVALID_ARGUMENT;
  ctx->dsm_precision = precision;
  return AMB_OK;
}

int amb_dsm_set_density_hint(amb_ctx* ctx, double points_per_cell) {
  if (!ctx || !(points_per_cell >= 0.0)) return AMB_ERR_INVALID_ARGUMENT;
  ctx->dsm_density_hint = points_per_cell;
  return AMB_OK;
}

int amb_stripe_y_interval(const amb_geometry* g, int32_t col_begin, int32_t col_end, double* y_lo, double* y_hi) {
  if (!g || !y_lo || !y_hi || col_begin < 0 || col_end > g->cols || col_begin >= col_end) return AMB_ERR_INVALID_ARGUMENT;
  // cell column j is centred at base_y - res*j; the stripe [col_begin, col_end) covers (y_lo, y_hi]
  const double base_y = g->pos_y + (0.5 * g->length_y - 0.5 * g->resolution);
  *y_hi = base_y - g->resolution * col_begin + 0.5 * g->resolution;
  *y_lo = base_y - g->resolution * (col_end - 1) - 0.5 * g->resolution;
  return AMB_OK;
}

double amb_dsm_halo_reach(const amb_geometry* g, int32_t interpolation_radius) {
  if (!g || interpolation_radius < 1) return -1.0;
  const std::vector<double> thr = dsm_thresholds(interpolation_radius);
  double m = 0.0;
  for (double t : thr) m = std::max(m, t);
  // (i) the largest retry threshold's reach + one cell of slack: what a border CELL can see; (ii) everything a border
  // TILE stages — tiles are aligned to global columns, so a tile cut by the stripe border extends up to tile-width - 1
  // columns beyond it, plus the window apron: with those points present every tile of the stripe stages exactly the
  // point set it stages in the undivided map, so tile-level quantities (shared-memory / warp-per-cell decision, the FP32
  // gather's height offset) are independent of the sharding.
  return std::max(std::sqrt(m) + g->resolution, dsm_tile_reach_cells(g->resolution, interpolation_radius) * g->resolution);
}

int amb_dsm_extract_halo(amb_ctx* ctx, const double* d_xyz, const uint64_t* d_ids, size_t n, double y_lo, double y_hi,
                         double reach, double center_easting, double* d_out_xyz, uint64_t* d_out_ids,
                         uint32_t capacity, uint32_t* d_count) {
  if (!ctx || !d_xyz || !d_out_xyz || !d_out_ids || !d_count) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  return dsm_extract_halo(ctx, d_xyz, reinterpret_cast<const unsigned long long*>(d_ids), n, y_lo, y_hi, reach,
                          center_easting, d_out_xyz, reinterpret_cast<unsigned long long*>(d_out_ids), capacity,
                          d_count);
}

int amb_dsm_enable_debug(amb_ctx* ctx, int enable) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  ctx->dsm_debug = enable != 0;
  if (!enable) ctx->dsm_debug_valid = false;
  return AMB_OK;
}

int amb_dsm_download_debug(amb_ctx* ctx, int32_t* neighbour_count, int8_t* threshold_index) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  if (!ctx->dsm_debug_valid) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t cells = ctx->slab_cells();
  if (neighbour_count)
    AMB_CUDA(ctx, cudaMemcpyAsync(neighbour_count, ctx->dbg_count.ptr, cells * sizeof(int32_t),
                                  cudaMemcpyDeviceToHost, ctx->stream));
  if (threshold_index)
    AMB_CUDA(ctx, cudaMemcpyAsync(threshold_index, ctx->dbg_level.ptr, cells, cudaMemcpyDeviceToHost, ctx->stream));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return AMB_OK;
}

int amb_dsm_download_bins(amb_ctx* ctx, int32_t* layout, uint32_t* bucket_starts, double* records, uint32_t* order) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  if (ctx->last_bin_destinations <= 0 || ctx->last_dsm_plan.size() != sizeof(dsmk::DsmPlan))
    return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  dsmk::DsmPlan plan;
  std::memcpy(&plan, ctx->last_dsm_plan.data(), sizeof(plan));
  unsigned int n_binned = 0;  // counted by the partition kernel, independently of the bucket starts
  AMB_CUDA(ctx, cudaMemcpyAsync(&n_binned, ctx->counters.as<unsigned int>() + CTR_DSM_BINNED, sizeof(n_binned),
                                cudaMemcpyDeviceToHost, ctx->stream));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (layout) {
    const int32_t v[AMB_DSM_BINS_LAYOUT] = {plan.B,   plan.Pa,  plan.BR,      plan.BC,
                                            plan.KR,  plan.KC,  plan.gj0,     plan.tile_j0,
                                            static_cast<int32_t>(n_binned),   ctx->last_bin_destinations};
    std::memcpy(layout, v, sizeof(v));
  }
  const size_t nbk = static_cast<size_t>(plan.KR) * static_cast<size_t>(plan.KC);
  if (bucket_starts)
    AMB_CUDA(ctx, cudaMemcpyAsync(bucket_starts, ctx->bin_starts.ptr, (nbk + 1) * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost, ctx->stream));
  if (records && n_binned)
    AMB_CUDA(ctx, cudaMemcpyAsync(records, ctx->records.ptr, static_cast<size_t>(n_binned) * sizeof(dsmk::PointRec),
                                  cudaMemcpyDeviceToHost, ctx->stream));
  if (order && n_binned)
    AMB_CUDA(ctx, cudaMemcpyAsync(order, ctx->point_order.ptr, static_cast<size_t>(n_binned) * sizeof(uint32_t),
                                  cudaMemcpyDeviceToHost, ctx->stream));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return AMB_OK;
}

int amb_dsm_thresholds(int32_t interpolation_radius, double* thresholds, int32_t capacity) {
  if (interpolation_radius < 1 || !thresholds || capacity <= 0) return AMB_ERR_INVALID_ARGUMENT;
  const std::vector<double> thr = dsm_thresholds(interpolation_radius);
  const int n = static_cast<int>(std::min<size_t>(thr.size(), static_cast<size_t>(capacity)));
  for (int k = 0; k < n; ++k) thresholds[k] = thr[k];
  return n;
}

// ---- Ortho ----
int amb_ortho_process_device(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B,
                             const uint8_t* const* d_images, size_t n, int32_t channels, size_t row_step,
                             int32_t colored_ortho) {
  return run_ortho(ctx, {.frames = OrthoCall::DEVICE, .camera = camera, .T_G_B = T_G_B, .n = n, .channels = channels,
                         .row_step = row_step, .colored_ortho = colored_ortho, .images = d_images});
}

int amb_ortho_process(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B, const uint8_t* const* images,
                      size_t n, int32_t channels, size_t row_step, int32_t colored_ortho) {
  return run_ortho(ctx, {.frames = OrthoCall::HOST, .camera = camera, .T_G_B = T_G_B, .n = n, .channels = channels,
                         .row_step = row_step, .colored_ortho = colored_ortho, .images = images});
}

int amb_ortho_process_jpeg(amb_ctx* ctx, const amb_camera* camera, const double* T_G_B, const void* const* files,
                           const size_t* file_bytes, size_t n, int32_t colored_ortho) {
  return run_ortho(ctx, {.frames = OrthoCall::JPEG, .camera = camera, .T_G_B = T_G_B, .n = n,
                         .channels = colored_ortho ? 3 : 1, .colored_ortho = colored_ortho, .files = files,
                         .file_bytes = file_bytes});
}

int amb_ortho_set_brute_force(amb_ctx* ctx, int brute_force) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  ctx->ortho_brute_force = brute_force != 0;
  return AMB_OK;
}

int amb_ortho_set_dominance_cull(amb_ctx* ctx, int enable) {
  if (!ctx) return AMB_ERR_INVALID_ARGUMENT;
  ctx->ortho_dominance = enable != 0;
  return AMB_OK;
}

// ---- measurement ----
int amb_get_timings(amb_ctx* ctx, amb_timings* out) {
  if (!ctx || !out) return AMB_ERR_INVALID_ARGUMENT;
  AMB_CUDA(ctx, cudaSetDevice(ctx->device));
  AMB_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  std::memset(out, 0, sizeof(*out));
  auto ms = [&](int a, int b) {
    float t = 0.f;
    if (cudaEventElapsedTime(&t, ctx->events[a], ctx->events[b]) != cudaSuccess) {
      cudaGetLastError();
      t = 0.f;
    }
    return t;
  };
  if (ctx->dsm_timed) {
    out->dsm_h2d_ms = ctx->dsm_had_h2d ? ms(EV_DSM_BEGIN, EV_DSM_H2D_END) : 0.f;
    out->dsm_bin_ms = ms(EV_DSM_H2D_END, EV_DSM_BIN_END);
    out->dsm_gather_ms = ms(EV_DSM_BIN_END, EV_DSM_GATHER_END);
    out->dsm_fill_ms = ms(EV_DSM_GATHER_END, EV_DSM_FILL_END);
    out->dsm_total_ms = ms(EV_DSM_BEGIN, EV_DSM_FILL_END);
    out->dsm_kernel_launches = ctx->dsm_launches;
    unsigned int c[CTR_COUNT] = {};
    if (ctx->counters.ptr) {
      AMB_CUDA(ctx, cudaMemcpy(c, ctx->counters.ptr, sizeof(c), cudaMemcpyDeviceToHost));
    }
    out->dsm_cells_empty = static_cast<int64_t>(c[CTR_DSM_LIST]) + c[CTR_DSM_LIST_DONE];
    out->dsm_points_binned = c[CTR_DSM_BINNED];
  }
  if (ctx->ortho_timed) {
    if (ctx->ortho_two_phase) {  // select kernel | sub-rectangle copies | texel kernel
      out->ortho_h2d_ms = ms(EV_ORTHO_SELECT_END, EV_ORTHO_COPY_END);
      out->ortho_kernel_ms = ms(EV_ORTHO_H2D_END, EV_ORTHO_SELECT_END) + ms(EV_ORTHO_COPY_END, EV_ORTHO_END);
      out->ortho_h2d_bytes = ctx->ortho_h2d_bytes;
    } else {
      out->ortho_h2d_ms = 0.f;
      out->ortho_kernel_ms = ms(EV_ORTHO_H2D_END, EV_ORTHO_END);
    }
    out->ortho_total_ms = ms(EV_ORTHO_BEGIN, EV_ORTHO_END);
    out->ortho_kernel_launches = ctx->ortho_launches;
  }
  return AMB_OK;
}

int amb_host_alloc(void** ptr, size_t bytes) {
  if (!ptr) return AMB_ERR_INVALID_ARGUMENT;
  cudaError_t e = cudaHostAlloc(ptr, bytes, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return AMB_ERR_CUDA;
  }
  return AMB_OK;
}

int amb_host_free(void* ptr) {
  if (!ptr) return AMB_OK;
  cudaError_t e = cudaFreeHost(ptr);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return AMB_ERR_CUDA;
  }
  return AMB_OK;
}

}  // extern "C"
