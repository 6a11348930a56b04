/*
 * amb_oracle.h — C ABI of the CPU ORACLE (TEST INFRASTRUCTURE, NOT PRODUCT CODE).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load this.
 * The product library (aerial_mapper_b200/csrc) never links, loads or calls anything under oracle/.
 *
 * PINNING.  The reference (ethz-asl/aerial_mapper @ /root/reference) ships no tests, golden vectors or fixtures for
 * this path (SURVEY.md §4, §8c) and its packages cannot be built as they are (ROS, catkin, grid_map, aslam_cv2,
 * minkindr, Eigen, OpenCV, glog — all absent, no network).  What pins this oracle:
 *   - oracle/_ref/libamb_refsrc_{main,pcl}.so: the reference's OWN dsm.cc, ortho-backward-grid.cc, ortho-from-pcl.cc,
 *     utils-common.cc and the reference headers they include (nanoflann.hpp among them) compiled VERBATIM from where
 *     they lie, against stand-in headers for the absent third-party libraries (refsrc_stubs/amb_refsrc_deps.h lists
 *     exactly what is reference code and what is restated).  tests/test_oracle_refsrc.py: the restated loops are
 *     bit-identical to the reference's own code on every layer; the committed golden fixtures likewise.
 *   - oracle/_ref/libamb_refsrc_stereo.so: the reference's densifier.cpp likewise ("next" row N3); stereo_oracle.cc is
 *     bit-identical to it (tests/test_stereo_reproject.py).
 *   - oracle/_ref/libamb_oracle_ref.so: nanoflann.hpp verbatim around the restated cell loop (exposes neighbour
 *     counts / retry levels); the dependency-free restatement in dsm_oracle.cc is checked against it.
 *   - brute force / scipy.spatial.cKDTree for neighbour sets, cv2.projectPoints for the camera model, scipy Rotation
 *     for the pose algebra (tests/test_oracle_*.py).
 * PARITY UNPINNED for one part only: the arithmetic of the un-vendored, un-versioned dependencies
 * (install/dependencies_https.rosinstall:1,9,11) — grid_map's cell-centre formula and colour packing, aslam_cv2's
 * pinhole/distortion projection, minkindr's pose algebra — is restated from their upstream sources
 * (thirdparty_math.h, oracle_common.h) in both the stand-ins and the restatement.
 */
#ifndef AMB_ORACLE_H_
#define AMB_ORACLE_H_

#include "../include/aerial_mapper_b200.h" /* amb_geometry, amb_camera, amb_status: plain structs only */

#ifdef __cplusplus
extern "C" {
#endif

/*
 * dsm::Dsm::process restated (dsm.cc:186-201 -> :36-52 kd-tree fill, :113-184 cell loop).
 *   elevation      full layer rows*cols, column-major, in/out (cells without neighbours keep their value)
 *   num_threads    >0: that many parFor blocks (utils-common.h:29-59); 0: std::thread::hardware_concurrency()
 *                  (dsm.cc:178); -1: the single-thread twin (dsm.cc:54-111) — same arithmetic
 *   cell_begin/end half-open range of GridMapIterator linear indices k (index = (k % rows, k / rows)) to
 *                  evaluate; 0, rows*cols for the whole map.  A sub-range is the bench's "bounded sample".
 *   neighbour_count / threshold_index   nullable, full-size, filled for evaluated cells
 *                  (result_set.size() dsm.cc:146; k of the threshold lambda_k*radius that produced it, -1 none)
 *   seconds        nullable double[2]: [0] kd-tree/bucket build, [1] cell loop (the reference's own bracket
 *                  dsm.cc:115,181-183)
 */
int ambo_dsm_process(const amb_geometry* geom, float* elevation, const double* xyz, size_t n,
                     int32_t interpolation_radius, double center_easting, double center_northing,
                     int32_t num_threads, int64_t cell_begin, int64_t cell_end, int32_t* neighbour_count,
                     int8_t* threshold_index, double* seconds);

/* Same cell loop around the reference's vendored nanoflann.hpp compiled verbatim; only exported by
 * oracle/_ref/libamb_oracle_ref.so. */
int ambo_ref_dsm_process(const amb_geometry* geom, float* elevation, const double* xyz, size_t n,
                         int32_t interpolation_radius, double center_easting, double center_northing,
                         int32_t num_threads, int64_t cell_begin, int64_t cell_end, int32_t* neighbour_count,
                         int8_t* threshold_index, double* seconds);

/*
 * ortho::OrthoFromPcl::process restated (aerial_mapper_ortho/src/ortho-from-pcl.cc:20-113; "next" row N1):
 * IDW of the point intensities into the `ortho` layer.  Same search back ends as the DSM (bucket restatement here,
 * the reference's nanoflann in oracle/_ref as ambo_ref_ortho_from_pcl_process).  use_adaptive_interpolation != 0
 * (:63-72, thresholds 10^k * radius without bound) is only supported by the nanoflann back end.
 * The reference loop is single-threaded (:52); num_threads > 0 only speeds the checker up (cells are independent).
 */
int ambo_ortho_from_pcl_process(const amb_geometry* geom, float* ortho, const double* xyz, const int32_t* intensities,
                                size_t n, int32_t interpolation_radius, int32_t use_adaptive_interpolation,
                                int32_t num_threads, int64_t cell_begin, int64_t cell_end, double* seconds);
int ambo_ref_ortho_from_pcl_process(const amb_geometry* geom, float* ortho, const double* xyz,
                                    const int32_t* intensities, size_t n, int32_t interpolation_radius,
                                    int32_t use_adaptive_interpolation, int32_t num_threads, int64_t cell_begin,
                                    int64_t cell_end, double* seconds);

/*
 * ortho::OrthoBackwardGrid::process restated (ortho-backward-grid.cc:223-239 -> :128-221).
 * All layers are full rows*cols column-major.  ortho / colored_ortho: the one not selected may be NULL.
 * seconds: nullable double[1] = cell loop (reference bracket ortho-backward-grid.cc:140,218-220).
 */
int ambo_ortho_process(const amb_geometry* geom, const float* elevation, float* elevation_angle,
                       float* observation_index, float* ortho, float* colored_ortho, const amb_camera* camera,
                       const double* T_G_B, const uint8_t* const* images, size_t n, int32_t channels,
                       size_t row_step, int32_t colored_ortho_flag, int32_t num_threads, int64_t cell_begin,
                       int64_t cell_end, double* seconds);

/* stereo::Densifier::computePointCloud restated (densifier.cpp:25-108; "next" row N3): disparity -> world points in
 * raster order.  K = {fx, fy, cx, cy}; strides in elements per row, at least `width` (the product's argument
 * contract, include/aerial_mapper_b200.h). */
int ambo_stereo_reproject(const float* disparity, size_t disparity_stride, const uint8_t* image_left,
                          size_t image_stride, int32_t width, int32_t height, const double* K, double baseline,
                          const double* R_G_C, const double* t_G_C1, float max_invalid_disparity, double* out_xyz,
                          int32_t* out_intensity, size_t capacity, size_t* out_count);

/* stereo::Rectifier::rectifyStereoPair restated (rectifier.cpp:36-107; "next" row N3, second half).  Matrices row-major
 * 3x3.  setup: Fusiello rectification in double -> baseline, R_G_C_rect and the two float32 homographies T_i^-1;
 * maps: the per-pixel fill of the four CV_32FC1 maps (row stride map_stride floats).  remap / mask stay OpenCV. */
int ambo_stereo_rectify_setup(const double* K, const double* R_G_C1, const double* R_G_C2, const double* t_G_C1,
                              const double* t_G_C2, double* baseline, double* R_G_C_rect, float* T1_inv,
                              float* T2_inv);
int ambo_stereo_rectify_maps(const float* T1_inv, const float* T2_inv, int32_t width, int32_t height,
                             size_t map_stride, float* map1_x, float* map1_y, float* map2_x, float* map2_y);

/* Single-point helpers for cross-checks against cv2 / scipy. */
/* aslam::PinholeCamera::project3 restated; returns 1 if the reference's keypoint_visible predicate
 * (ortho-backward-grid.cc:164-171) holds, 0 otherwise. */
int ambo_project3(const amb_camera* camera, const double* p_C, double* keypoint);
/* T_G_C = T_G_B * T_C_B^-1 (ortho-backward-grid.cc:232), then C_p = T_G_C^-1 . G_p (:157-158).
 * T_G_B as x y z qw qx qy qz. */
int ambo_transform_to_camera(const amb_camera* camera, const double* T_G_B, const double* p_G, double* p_C);
/* grid_map::colorVectorToValue on the (R,G,B)/255 vector the reference builds from a BGR pixel
 * (ortho-backward-grid.cc:194-202); returns the float's bit pattern. */
uint32_t ambo_pack_color(uint8_t b, uint8_t g, uint8_t r);
/* Number of hardware threads the MT path would use. */
int ambo_hardware_concurrency(void);

#ifdef __cplusplus
}
#endif
#endif /* AMB_ORACLE_H_ */
