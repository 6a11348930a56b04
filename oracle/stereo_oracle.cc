/*
 * stereo_oracle.cc — CPU restatement of stereo::Densifier::computePointCloud (TEST INFRASTRUCTURE; see
 * amb_oracle.h).  Reference: aerial_mapper_dense_pcl/src/densifier.cpp:25-108 ("next" row N3).  Only the outputs
 * the mapping path consumes are produced (point_cloud_eigen, point_cloud_intensities); the ROS message fill is
 * visualisation transport.
 */
#include <cmath>
#include <cstddef>
#include <cstdint>

#include "amb_oracle.h"

extern "C" int ambo_stereo_reproject(const float* disparity, size_t disparity_stride, const uint8_t* image_left,
                                     size_t image_stride, int32_t width, int32_t height, const double* K,
                                     double baseline, const double* R_G_C, const double* t_G_C1,
                                     float max_invalid_disparity, double* out_xyz, int32_t* out_intensity,
                                     size_t capacity, size_t* out_count) {
  if (!disparity || !image_left || !K || !R_G_C || !t_G_C1 || !out_xyz || !out_intensity || !out_count || width <= 0 ||
      height <= 0 || disparity_stride < static_cast<size_t>(width) || image_stride < static_cast<size_t>(width))
    return AMB_ERR_INVALID_ARGUMENT;
  if (baseline == 0.0) return AMB_ERR_CHECK_FAILED; /* CHECK_NE(baseline, 0.0), :39 */
  const double fx = K[0], fy = K[1], cx = K[2], cy = K[3];
  /* Q = [1 0 0 -cx; 0 fx/fy 0 -cy*(fx/fy); 0 0 0 fx; 0 0 1/baseline 0]  (:45-47) */
  const double q03 = -cx, q11 = fx / fy, q13 = -cy * (fx / fy), q23 = fx, q32 = 1.0 / baseline;
  size_t n = 0;
  for (int v = 0; v < height; ++v) {
    const float* drow = disparity + static_cast<size_t>(v) * disparity_stride;
    const uint8_t* irow = image_left + static_cast<size_t>(v) * image_stride;
    for (int u = 0; u < width; ++u) {
      if (drow[u] > max_invalid_disparity) {          /* :61 */
        const double w = q32 * drow[u];               /* :63 */
        const double x1 = (u + q03) / w;              /* :69-70 */
        const double y1 = (q11 * v + q13) / w;
        const double z1 = q23 / w;
        /* rectified_stereo_pair.R_G_C * point_r1 + stereo_pair.t_G_C1 (:73-74) */
        const double X = ((R_G_C[0] * x1 + R_G_C[1] * y1) + R_G_C[2] * z1) + t_G_C1[0];
        const double Y = ((R_G_C[3] * x1 + R_G_C[4] * y1) + R_G_C[5] * z1) + t_G_C1[1];
        const double Z = ((R_G_C[6] * x1 + R_G_C[7] * y1) + R_G_C[8] * z1) + t_G_C1[2];
        const float z = static_cast<float>(Z);
        if (!std::isinf(z)) {                         /* :78 */
          if (n < capacity) {
            out_xyz[3 * n + 0] = X;                   /* point_cloud_eigen.push_back(point_G), :93 */
            out_xyz[3 * n + 1] = Y;
            out_xyz[3 * n + 2] = Z;
            out_intensity[n] = irow[u];               /* point_cloud_intensities.push_back(gray), :94 */
          }
          ++n;
        }
      }
    }
  }
  *out_count = n;
  return AMB_OK;
}

/* ------------------------------------------------------------------------------------------------------------
 * stereo::Rectifier::rectifyStereoPair restated (aerial_mapper_dense_pcl/src/rectifier.cpp:36-107; "next" row N3,
 * second half): Fusiello's compact rectification on the host in double, then the per-pixel fill of the four
 * CV_32FC1 rectification maps in float.  cv::remap and the contour mask (OpenCV) stay out of scope, like block
 * matching.  Matrices are row-major 3x3.
 *
 * Eigen arithmetic restated (absent, un-versioned dependency): cross products, normalized() = v / sqrt(v.v),
 * 3x3 products as (a0*b0 + a1*b1) + a2*b2, Matrix3d::inverse() through cofactors and 1/det (Eigen LU/InverseImpl.h,
 * compute_inverse<..., 3>).  The float maps depend on these only through the rounded float32 homographies. */
namespace {

inline void cross3(const double* a, const double* b, double* o) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}

inline void normalize3(const double* v, double* o) {
  const double n = std::sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
  o[0] = v[0] / n;
  o[1] = v[1] / n;
  o[2] = v[2] / n;
}

inline void mul33(const double* A, const double* B, double* C) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
}

inline void transpose33(const double* A, double* T) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) T[3 * i + j] = A[3 * j + i];
}

inline double cofactor33(const double* m, int i, int j) {
  const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
  return m[3 * i1 + j1] * m[3 * i2 + j2] - m[3 * i1 + j2] * m[3 * i2 + j1];
}

inline bool inverse33(const double* m, double* inv) {
  const double c00 = cofactor33(m, 0, 0), c10 = cofactor33(m, 1, 0), c20 = cofactor33(m, 2, 0);
  const double det = (c00 * m[0] + c10 * m[3]) + c20 * m[6];
  if (det == 0.0) return false;
  const double invdet = 1.0 / det;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) inv[3 * j + i] = cofactor33(m, i, j) * invdet; /* inverse = adjugate / det */
  return true;
}

}  // namespace

extern "C" int ambo_stereo_rectify_setup(const double* K, const double* R_G_C1, const double* R_G_C2,
                                         const double* t_G_C1, const double* t_G_C2, double* baseline,
                                         double* R_G_C_rect, float* T1_inv, float* T2_inv) {
  if (!K || !R_G_C1 || !R_G_C2 || !t_G_C1 || !t_G_C2 || !baseline || !R_G_C_rect || !T1_inv || !T2_inv)
    return AMB_ERR_INVALID_ARGUMENT;
  /* new x axis = direction of the baseline, t_G_C2 - t_G_C1 (:46-47) */
  const double x[3] = {t_G_C2[0] - t_G_C1[0], t_G_C2[1] - t_G_C1[1], t_G_C2[2] - t_G_C1[2]};
  *baseline = std::sqrt((x[0] * x[0] + x[1] * x[1]) + x[2] * x[2]);
  if (*baseline == 0.0) return AMB_ERR_CHECK_FAILED;
  /* new y = old z of camera 1 (R_G_C1.col(2)) x new x; new z = x cross y (:49-53) */
  const double z1[3] = {R_G_C1[2], R_G_C1[5], R_G_C1[8]};
  double y[3], z[3];
  cross3(z1, x, y);
  cross3(x, y, z);
  /* R_G_C_rect = [x^ y^ z^]^T: rows are the normalised axes (:56-61) */
  normalize3(x, R_G_C_rect + 0);
  normalize3(y, R_G_C_rect + 3);
  normalize3(z, R_G_C_rect + 6);
  /* P_rect.block<3,3>(0,0) = K * R_G_C_rect (:64-71); Q_i = K * R_G_C_i^T (:74-75);
   * T_i_rect = (K R_rect) * Q_i^-1 (:76-77); T_i_inv = T_i_rect^-1 cast to float (:78-79) */
  double KR[9], Rt[9], Q[9], Qinv[9], T[9], Tinv[9];
  mul33(K, R_G_C_rect, KR);
  const double* Rs[2] = {R_G_C1, R_G_C2};
  float* outs[2] = {T1_inv, T2_inv};
  for (int c = 0; c < 2; ++c) {
    transpose33(Rs[c], Rt);
    mul33(K, Rt, Q);
    if (!inverse33(Q, Qinv)) return AMB_ERR_CHECK_FAILED;
    mul33(KR, Qinv, T);
    if (!inverse33(T, Tinv)) return AMB_ERR_CHECK_FAILED;
    for (int k = 0; k < 9; ++k) outs[c][k] = static_cast<float>(Tinv[k]);
  }
  return AMB_OK;
}

/* The per-pixel loop (:80-104): [x y w]^T = T_inv * [u_rect v_rect 1]^T in float, map = (x / w, y / w).
 * Maps are H x W, row stride `map_stride` floats. */
extern "C" int ambo_stereo_rectify_maps(const float* T1_inv, const float* T2_inv, int32_t width, int32_t height,
                                        size_t map_stride, float* map1_x, float* map1_y, float* map2_x,
                                        float* map2_y) {
  if (!T1_inv || !T2_inv || !map1_x || !map1_y || !map2_x || !map2_y || width <= 0 || height <= 0 ||
      map_stride < static_cast<size_t>(width))
    return AMB_ERR_INVALID_ARGUMENT;
  const float* Ts[2] = {T1_inv, T2_inv};
  float* mx[2] = {map1_x, map2_x};
  float* my[2] = {map1_y, map2_y};
  int status = AMB_OK;
  for (int v = 0; v < height; ++v) {
    for (int u = 0; u < width; ++u) {
      const float fu = static_cast<float>(u), fv = static_cast<float>(v);
      for (int c = 0; c < 2; ++c) {
        const float* T = Ts[c];
        const float x = (T[0] * fu + T[1] * fv) + T[2] * 1.0f;
        const float y = (T[3] * fu + T[4] * fv) + T[5] * 1.0f;
        const float w = (T[6] * fu + T[7] * fv) + T[8] * 1.0f;
        if (w == 0.0f) status = AMB_ERR_CHECK_FAILED; /* CHECK_NE(xyw(2), 0.0), :92,:99 */
        mx[c][static_cast<size_t>(v) * map_stride + u] = x / w;
        my[c][static_cast<size_t>(v) * map_stride + u] = y / w;
      }
    }
  }
  return status;
}
