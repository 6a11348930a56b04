// Drop-in replacement of <aerial-mapper-ortho/ortho-from-pcl.h> (reference
// aerial_mapper_ortho/include/aerial-mapper-ortho/ortho-from-pcl.h; caller main-ortho-from-pcl.cc:122-136).
// "Next" row N1 of SURVEY.md §8f.  NB this header defines its OWN ortho::Settings (different members from the
// backward-grid one, as in the reference): never include both in one translation unit.
#ifndef ORTHO_FROM_PCL_H_
#define ORTHO_FROM_PCL_H_

#include "../amb_shim_common.h"

namespace ortho {

struct Settings {  // ortho-from-pcl.h:28-35, field for field
  EIGEN_MAKE_ALIGNED_OPERATOR_NEW
  bool show_orthomosaic_opencv = false;
  int interpolation_radius = 2;
  bool use_adaptive_interpolation = false;
  bool save_orthomosaic_jpg = false;
  std::string orthomosaic_jpg_filename = "";
};

class OrthoFromPcl {
 public:
  EIGEN_MAKE_ALIGNED_OPERATOR_NEW

  explicit OrthoFromPcl(const Settings& settings) : settings_(settings), context_(new amb_shim::Context()) {}

  // ortho-from-pcl.cc:20-113
  void process(const AlignedType<std::vector, Eigen::Vector3d>::type& pointcloud,
               const std::vector<int>& intensities, grid_map::GridMap* map) const {
    CHECK(!pointcloud.empty());
    CHECK(map);
    CHECK(intensities.size() >= pointcloud.size());  // CHECK(i < intensities.size()) for every i, :32
    static_assert(sizeof(int) == sizeof(int32_t), "int32 intensities expected");
    context_->get(*map);
    context_->upload(map, "ortho", AMB_LAYER_ORTHO);  // cells without neighbours keep their value
    // one GPU, or the map's column stripes over AMB_SHIM_GPUS=N GPUs (amb_multi_ortho_from_pcl_process)
    context_->orthoFromPclProcess(&pointcloud[0](0), reinterpret_cast<const int32_t*>(intensities.data()),
                                  pointcloud.size(), settings_.interpolation_radius,
                                  settings_.use_adaptive_interpolation ? 1 : 0);
    context_->download(map, "ortho", AMB_LAYER_ORTHO);
  }

 private:
  Settings settings_;
  std::shared_ptr<amb_shim::Context> context_;  // process() is const in the reference
};

}  // namespace ortho
#endif  // ORTHO_FROM_PCL_H_
