// amb_multi.cu — several GPUs of ONE process behind the C ABI (SURVEY.md §8b "amb_create(geom, n_gpus)"): what a C++
// caller of dsm::Dsm / ortho::OrthoBackwardGrid (the drop-in headers under shim/) gets without any framework.
//
//   amb_multi owns one amb_ctx per device, each with a contiguous column stripe of the map (the same partition as
//   sharding.stripe_range).  The reference's entry points take ONE unsorted host cloud / ONE set of host frames, so:
//     DSM    every device receives the whole cloud over its own PCIe link (the copies run in parallel) and bins what can
//            reach its stripe; point ids are array positions, so each stripe is bit-identical to the same stripe of a
//            single-GPU run.  No exchange step exists on this path: nothing is sharded on the way in.  (A cloud that
//            ARRIVES sharded uses the per-context amb_dsm_process_sharded* with its halo exchange.)
//     ortho  every device evaluates its stripe over all frames; with host frames only the winners' sub-rectangles of the
//            stripe cross that device's PCIe link.
//     OrthoFromPcl  like DSM (whole cloud and intensities to every device); adaptive interpolation included, whose far
//            thresholds read the whole cloud each device holds (pcl_adaptive_kernels.cu).
//   Host layers are full column-major maps; a stripe is a contiguous range of them.
// The blocking host entry points of the stripes run concurrently on one std::thread per device.
#include <thread>

#include "amb_context.h"

struct amb_multi {
  amb_geometry geom;
  std::vector<amb_ctx*> ctx;
  std::string last_error;
};

namespace {

inline void stripe_of(int32_t cols, int rank, int world, int32_t* c0, int32_t* c1) {
  const int32_t w = (cols + world - 1) / world;  // sharding.stripe_range
  *c0 = std::min<int32_t>(rank * w, cols);
  *c1 = std::min<int32_t>(*c0 + w, cols);
}

// run fn(r, ctx) for every stripe concurrently; first non-zero status wins
template <typename F>
int for_each_stripe(amb_multi* m, F fn) {
  const int n = static_cast<int>(m->ctx.size());
  std::vector<int> st(n, AMB_OK);
  if (n == 1) {
    st[0] = fn(0, m->ctx[0]);
  } else {
    std::vector<std::thread> th;
    try {
      for (int r = 0; r < n; ++r) th.emplace_back([&, r] { st[r] = fn(r, m->ctx[r]); });
    } catch (const std::exception&) {
      for (std::thread& t : th) t.join();
      m->last_error = "could not start the per-device host threads";
      return AMB_ERR_UNSUPPORTED;
    }
    for (std::thread& t : th) t.join();
  }
  for (int r = 0; r < n; ++r)
    if (st[r] != AMB_OK) {
      m->last_error = std::string("device ") + std::to_string(m->ctx[r]->device) + ": " + amb_last_error(m->ctx[r]);
      return st[r];
    }
  return AMB_OK;
}

inline float* stripe_ptr(const amb_multi* m, int r, float* full) {
  return full + static_cast<size_t>(m->geom.rows) * static_cast<size_t>(m->ctx[r]->col_begin);
}

// One host cloud of n points to every stripe's host entry point process(ctx).  Bucket size / stage capacity — hence
// every summation order — follow the density of the WHOLE cloud on every device; the adaptive OrthoFromPcl pass's
// whole-map binning also needs it to visit the buckets of a single-GPU run.
template <typename F>
int cloud_to_every_stripe(amb_multi* m, size_t n, bool inputs, F process) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  if (n == 0) return AMB_ERR_EMPTY;  // dsm.cc:189-192, CHECK(!pointcloud.empty()) ortho-from-pcl.cc:23
  if (!inputs) return AMB_ERR_INVALID_ARGUMENT;
  const double per_cell = static_cast<double>(n) / (static_cast<double>(m->geom.rows) * static_cast<double>(m->geom.cols));
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    const int st = amb_dsm_set_density_hint(c, per_cell);
    return st == AMB_OK ? process(c) : st;
  });
}

}  // namespace

extern "C" {

int amb_multi_create(const amb_geometry* geom, int n_gpus, amb_multi** out) {
  if (!geom || !out || n_gpus < 1) return AMB_ERR_INVALID_ARGUMENT;
  const int have = amb_device_count();
  if (have <= 0) return AMB_ERR_NO_DEVICE;
  if (n_gpus > have || n_gpus > geom->cols) return AMB_ERR_INVALID_ARGUMENT;
  amb_multi* m = new (std::nothrow) amb_multi();
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  m->geom = *geom;
  for (int r = 0; r < n_gpus; ++r) {
    int32_t c0, c1;
    stripe_of(geom->cols, r, n_gpus, &c0, &c1);
    if (c1 <= c0) break;  // more devices than stripes of that width: the rest stay idle
    amb_ctx* c = nullptr;
    const int st = amb_create(geom, r, c0, c1, &c);
    if (st != AMB_OK) {
      for (amb_ctx* x : m->ctx) amb_destroy(x);
      delete m;
      return st;
    }
    m->ctx.push_back(c);
  }
  *out = m;
  return AMB_OK;
}

void amb_multi_destroy(amb_multi* m) {
  if (!m) return;
  for (amb_ctx* c : m->ctx) amb_destroy(c);
  delete m;
}

int amb_multi_size(const amb_multi* m) { return m ? static_cast<int>(m->ctx.size()) : 0; }
amb_ctx* amb_multi_context(amb_multi* m, int rank) {
  return (m && rank >= 0 && rank < static_cast<int>(m->ctx.size())) ? m->ctx[rank] : nullptr;
}
const char* amb_multi_last_error(const amb_multi* m) { return m ? m->last_error.c_str() : ""; }

int amb_multi_init_layers(amb_multi* m) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [](int, amb_ctx* c) { return amb_init_layers(c); });
}

int amb_multi_upload_layer(amb_multi* m, int layer, const float* host_full) {
  if (!m || !host_full) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [&](int r, amb_ctx* c) {
    return amb_upload_layer(c, layer, stripe_ptr(m, r, const_cast<float*>(host_full)));
  });
}

int amb_multi_download_layer(amb_multi* m, int layer, float* host_full) {
  if (!m || !host_full) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [&](int r, amb_ctx* c) { return amb_download_layer(c, layer, stripe_ptr(m, r, host_full)); });
}

int amb_multi_export_raster(amb_multi* m, int layer, int format, void* host_image) {
  if (!m || !host_image || layer < 0 || layer >= AMB_NUM_LAYERS || format < AMB_RASTER_F32 || format > AMB_RASTER_MASK8)
    return AMB_ERR_INVALID_ARGUMENT;
  const size_t bpp = format == AMB_RASTER_F32 ? 4 : format == AMB_RASTER_BGR8 ? 3 : 1;
  // stripe r owns image rows [col_begin, col_end) (include/aerial_mapper_b200.h)
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    unsigned char* band = static_cast<unsigned char*>(host_image) +
                          static_cast<size_t>(m->geom.rows) * static_cast<size_t>(c->col_begin) * bpp;
    return amb_export_raster(c, layer, format, band);
  });
}

int amb_multi_import_raster(amb_multi* m, int layer, const float* host_band, int32_t width, int32_t height,
                            size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  // every stripe validates the same arguments before it writes anything, and reads only its own window of the band
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    return amb_import_raster(c, layer, host_band, width, height, row_stride, gt, has_nodata, nodata, resample);
  });
}

int amb_multi_import_tiff(amb_multi* m, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                          const double gt[6], int has_nodata, float nodata, int resample) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  // each stripe decodes the chunks of its own window; a corrupt one stops only that stripe's import
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    return amb_import_tiff(c, layer, file, bytes, layout, gt, has_nodata, nodata, resample);
  });
}

int amb_multi_import_raster_lonlat(amb_multi* m, int layer, const float* host_band, int32_t width, int32_t height,
                                   size_t row_stride, const double gt[6], int has_nodata, float nodata, int resample,
                                   int32_t map_epsg) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    return amb_import_raster_lonlat(c, layer, host_band, width, height, row_stride, gt, has_nodata, nodata, resample,
                                    map_epsg);
  });
}

int amb_multi_import_tiff_lonlat(amb_multi* m, int layer, const void* file, size_t bytes, const amb_tiff_layout* layout,
                                 const double gt[6], int has_nodata, float nodata, int resample, int32_t map_epsg) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    return amb_import_tiff_lonlat(c, layer, file, bytes, layout, gt, has_nodata, nodata, resample, map_epsg);
  });
}

int amb_multi_set_host_mirror(amb_multi* m, int layer, float* host_full) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  for (size_t r = 0; r < m->ctx.size(); ++r) {
    const int st = amb_set_host_mirror(m->ctx[r], layer, host_full ? stripe_ptr(m, static_cast<int>(r), host_full) : nullptr);
    if (st != AMB_OK) return st;
  }
  return AMB_OK;
}

int amb_multi_sync(amb_multi* m) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [](int, amb_ctx* c) { return amb_sync(c); });
}

int amb_multi_dsm_process(amb_multi* m, const double* xyz, size_t n, int32_t interpolation_radius, double center_easting,
                          double center_northing) {
  return cloud_to_every_stripe(m, n, xyz != nullptr, [&](amb_ctx* c) {
    return amb_dsm_process(c, xyz, n, interpolation_radius, center_easting, center_northing);
  });
}

int amb_multi_ortho_from_pcl_process(amb_multi* m, const double* xyz, const int32_t* intensities, size_t n,
                                     int32_t interpolation_radius, int32_t use_adaptive_interpolation) {
  return cloud_to_every_stripe(m, n, xyz && intensities, [&](amb_ctx* c) {
    return amb_ortho_from_pcl_process(c, xyz, intensities, n, interpolation_radius, use_adaptive_interpolation);
  });
}

int amb_multi_ortho_process(amb_multi* m, const amb_camera* camera, const double* T_G_B, const uint8_t* const* images,
                            size_t n, int32_t channels, size_t row_step, int32_t colored_ortho) {
  if (!m) return AMB_ERR_INVALID_ARGUMENT;
  return for_each_stripe(m, [&](int, amb_ctx* c) {
    return amb_ortho_process(c, camera, T_G_B, images, n, channels, row_step, colored_ortho);
  });
}

}  // extern "C"
