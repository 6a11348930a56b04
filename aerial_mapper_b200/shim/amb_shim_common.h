// amb_shim_common.h — glue shared by the two drop-in class headers.
//
// Real build (inside the aerial_mapper catkin workspace): pulls the same third-party headers the reference's own
// headers pull (dsm.h:13-21, ortho-backward-grid.h:14-28).  Stand-alone build (-DAMB_SHIM_MINI, used by this
// repository's tests because Eigen / grid_map / aslam_cv2 / minkindr / OpenCV / glog are absent here): tiny
// stand-ins with the same names and the handful of members the marshalling code touches (mini/amb_mini_deps.h).
#ifndef AMB_SHIM_COMMON_H_
#define AMB_SHIM_COMMON_H_

#include <cstdio>
#include <cstdlib>
#include <ctime>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/aerial_mapper_b200.h"

#ifdef AMB_SHIM_MINI
#include "mini/amb_mini_deps.h"
#else
#include <aerial-mapper-io/aerial-mapper-io.h>            // Pose, Poses, Image, Images
#include <aerial-mapper-utils/utils-nearest-neighbor.h>  // AlignedType
#include <aslam/cameras/camera.h>
#include <aslam/cameras/camera-pinhole.h>
#include <aslam/cameras/ncamera.h>
#include <Eigen/Dense>
#include <glog/logging.h>
#include <grid_map_core/GridMap.hpp>
#endif

namespace amb_shim {

// The reference aborts through glog CHECK on contract violations (SURVEY.md §8b "Error convention"); a non-zero
// status from the C ABI is turned back into that.
inline void checkStatus(int status, const amb_ctx* ctx, const char* what) {
  if (status == AMB_OK) return;
  std::fprintf(stderr, "aerial_mapper_b200: %s failed: %s %s\n", what, amb_status_string(status),
               ctx ? amb_last_error(ctx) : "");
  CHECK(status == AMB_OK);
}

inline amb_geometry geometryOf(const grid_map::GridMap& map) {
  amb_geometry g;
  g.rows = map.getSize()(0);
  g.cols = map.getSize()(1);
  g.resolution = map.getResolution();
  g.length_x = map.getLength()(0);
  g.length_y = map.getLength()(1);
  g.pos_x = map.getPosition()(0);
  g.pos_y = map.getPosition()(1);
  return g;
}

// One device backend per MAP GEOMETRY, shared by every drop-in object of the process that works on a map of that geometry
// (dsm::Dsm and ortho::OrthoBackwardGrid of the batch demo, main-ortho-backward-grid.cc:129-141, end up on the same
// context: one set of device layers, scratch buffers allocated once) — or, with AMB_SHIM_GPUS=N (N > 1) in the
// environment, one amb_multi spreading the map's column stripes over N GPUs of this process (same results bit for bit,
// see include/aerial_mapper_b200.h "several GPUs of one process").
//
// Host layers stay authoritative like in the reference: by default every process() uploads what it reads and downloads
// what it writes (the library stages pageable memory — Eigen / cv::Mat / std::vector storage — through pinned slots
// with a worker pool, csrc/host_staging.cu, so these copies run at the host's memcpy rate rather than the driver's
// single-thread rate).  AMB_SHIM_RESIDENT_LAYERS=1 skips the upload of a layer whose device copy is known to equal the
// caller's buffer because this backend itself downloaded it into that very buffer last — valid when the caller does
// not edit layers between process() calls, which holds for every demo of the reference
// (main-dsm.cc, main-ortho-backward-grid.cc, main-ortho-backward-grid-incremental.cc).
struct Backend {
  amb_ctx* ctx;
  amb_multi* multi;
  amb_geometry geom;
  const float* device_equals[AMB_NUM_LAYERS];  // host buffer the device copy of the layer is known to equal (or nullptr)
  Backend() : ctx(nullptr), multi(nullptr) {
    for (int l = 0; l < AMB_NUM_LAYERS; ++l) device_equals[l] = nullptr;
  }
  ~Backend() {
    if (ctx) amb_destroy(ctx);
    if (multi) amb_multi_destroy(multi);
  }
};

inline bool sameGeometry(const amb_geometry& a, const amb_geometry& b) {
  return a.rows == b.rows && a.cols == b.cols && a.resolution == b.resolution && a.pos_x == b.pos_x &&
         a.pos_y == b.pos_y && a.length_x == b.length_x && a.length_y == b.length_y;
}

inline std::shared_ptr<Backend> acquireBackend(const amb_geometry& g) {
  static std::mutex mu;
  static std::vector<std::weak_ptr<Backend> > live;
  std::lock_guard<std::mutex> lock(mu);
  for (size_t k = 0; k < live.size(); ++k) {
    std::shared_ptr<Backend> b = live[k].lock();
    if (b && sameGeometry(b->geom, g)) return b;
  }
  std::shared_ptr<Backend> b(new Backend());
  b->geom = g;
  int gpus = 1;
  if (const char* e = std::getenv("AMB_SHIM_GPUS")) gpus = std::atoi(e);
  if (gpus > 1) {
    checkStatus(amb_multi_create(&g, gpus, &b->multi), nullptr, "amb_multi_create");
  } else {
    int device = 0;
    if (const char* e = std::getenv("AMB_DEVICE")) device = std::atoi(e);
    checkStatus(amb_create(&g, device, 0, g.cols, &b->ctx), nullptr, "amb_create");
  }
  size_t k = 0;
  while (k < live.size() && !live[k].expired()) ++k;
  if (k < live.size()) live[k] = b; else live.push_back(b);
  return b;
}

// AMB_SHIM_TRACE=1: wall-clock trace of the steps inside a process() call on stderr (development aid)
struct Trace {
  explicit Trace(const char* what) : on_(enabled()), what_(what) {
    if (on_) last_ = now();
  }
  void step(const char* name) {
    if (!on_) return;
    const double t = now();
    std::fprintf(stderr, "[amb shim] %s: %s %.2f ms\n", what_, name, (t - last_) * 1e3);
    last_ = t;
  }
  static bool enabled() {
    static const bool on = [] {
      const char* e = std::getenv("AMB_SHIM_TRACE");
      return e && e[0] == '1';
    }();
    return on;
  }
  static double now() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return static_cast<double>(ts.tv_sec) + 1e-9 * static_cast<double>(ts.tv_nsec);
  }
  bool on_;
  const char* what_;
  double last_;
};

class Context {
 public:
  Context() {}
  // binds to the backend of this map's geometry (creating it if needed); returns the single context (nullptr in multi-GPU mode)
  amb_ctx* get(const grid_map::GridMap& map) {
    const amb_geometry g = geometryOf(map);
    if (!b_ || !sameGeometry(b_->geom, g)) b_ = acquireBackend(g);
    return b_->ctx;
  }
  void upload(grid_map::GridMap* map, const char* layer, int id) {
    const float* host = (*map)[layer].data();
    static const bool resident = [] {
      const char* e = std::getenv("AMB_SHIM_RESIDENT_LAYERS");
      return e && e[0] == '1';
    }();
    if (resident && b_->device_equals[id] == host) return;  // the device copy is what this backend put into `host` last
    if (b_->multi) {
      checkMulti(amb_multi_upload_layer(b_->multi, id, host), "amb_multi_upload_layer");
    } else {
      checkStatus(amb_upload_layer(b_->ctx, id, host), b_->ctx, "amb_upload_layer");
    }
    b_->device_equals[id] = host;
  }
  void download(grid_map::GridMap* map, const char* layer, int id) {
    float* host = (*map)[layer].data();
    if (b_->multi) {
      checkMulti(amb_multi_download_layer(b_->multi, id, host), "amb_multi_download_layer");
    } else {
      checkStatus(amb_download_layer(b_->ctx, id, host), b_->ctx, "amb_download_layer");
    }
    b_->device_equals[id] = host;
  }
  void dsmProcess(const double* xyz, size_t n, int32_t radius, double center_easting, double center_northing) {
    b_->device_equals[AMB_LAYER_ELEVATION] = nullptr;
    if (b_->multi) {
      checkMulti(amb_multi_dsm_process(b_->multi, xyz, n, radius, center_easting, center_northing), "amb_multi_dsm_process");
    } else {
      checkStatus(amb_dsm_process(b_->ctx, xyz, n, radius, center_easting, center_northing), b_->ctx, "amb_dsm_process");
    }
  }
  void orthoProcess(const amb_camera* cam, const double* poses, const uint8_t* const* rasters, size_t n, int32_t channels,
                    size_t row_step, int32_t colored) {
    b_->device_equals[AMB_LAYER_ELEVATION_ANGLE] = nullptr;
    b_->device_equals[AMB_LAYER_OBSERVATION_INDEX] = nullptr;
    b_->device_equals[colored ? AMB_LAYER_COLORED_ORTHO : AMB_LAYER_ORTHO] = nullptr;
    if (b_->multi) {
      checkMulti(amb_multi_ortho_process(b_->multi, cam, poses, rasters, n, channels, row_step, colored),
                 "amb_multi_ortho_process");
    } else {
      checkStatus(amb_ortho_process(b_->ctx, cam, poses, rasters, n, channels, row_step, colored), b_->ctx, "amb_ortho_process");
    }
  }
  void orthoFromPclProcess(const double* xyz, const int32_t* intensities, size_t n, int32_t radius, int32_t adaptive) {
    b_->device_equals[AMB_LAYER_ORTHO] = nullptr;
    if (b_->multi) {
      checkMulti(amb_multi_ortho_from_pcl_process(b_->multi, xyz, intensities, n, radius, adaptive),
                 "amb_multi_ortho_from_pcl_process");
    } else {
      checkStatus(amb_ortho_from_pcl_process(b_->ctx, xyz, intensities, n, radius, adaptive), b_->ctx,
                  "amb_ortho_from_pcl_process");
    }
  }
  // (ortho-from-pcl.h) the output layer of OrthoFromPcl changed on the device
  void invalidate(int id) { b_->device_equals[id] = nullptr; }

 private:
  Context(const Context&);
  Context& operator=(const Context&);
  void checkMulti(int status, const char* what) {
    if (status == AMB_OK) return;
    std::fprintf(stderr, "aerial_mapper_b200: %s failed: %s %s\n", what, amb_status_string(status),
                 amb_multi_last_error(b_->multi));
    CHECK(status == AMB_OK);
  }
  std::shared_ptr<Backend> b_;
};

}  // namespace amb_shim
#endif
