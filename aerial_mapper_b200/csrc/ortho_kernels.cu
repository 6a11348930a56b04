// ortho_kernels.cu — grid-based orthomosaic back-projection on sm_90a.
//
// Replaces ortho::OrthoBackwardGrid::process (reference aerial_mapper_ortho/src/ortho-backward-grid.cc:223-239)
// and its cell loop (:128-221).  Per cell: landmark = (cell centre, (double)elevation); for every frame in
// ascending index: transform into the camera (:157-158), project with the distortion model (:159-161), test
// visibility (:164-171), alpha = asin(|z|/norm) (:173-177); a frame replaces the cell's state iff
// alpha > (double)elevation_angle (float32 layer, :180); the winner's nearest-neighbour texel is written
// (:186-206).  Winner-takes-all with a float-rounded running maximum — a sequential recurrence per cell, so it
// is evaluated by one thread per cell in frame order; frames are the inner loop, cells the parallel axis.
//
// What makes it fast: the reference projects every cell into every frame.  Here a 32x32 cell tile first discards
// the frames whose view cone cannot contain any of its cells (a provably conservative test, see
// compute_view_cone), keeps the survivors as an ascending index list in shared memory, and every thread walks
// that list reading the per-frame constants (R_C_G, t, camera centre) from __constant__ memory — all threads of
// a block read the same frame at the same time, i.e. a constant-cache broadcast.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <mutex>

#include "amb_context.h"
#include "jpeg_header.h"
#include "approx_math.h"

namespace amb {
namespace {

constexpr int kMaxFramesPerLaunch = 512;
#ifndef AMB_OTI
#define AMB_OTI 32
#endif
constexpr int OTI = AMB_OTI;  // tile extent along i (rows; contiguous in memory): a multiple of 32
static_assert(OTI % 32 == 0, "a warp covers 32 consecutive rows");
constexpr int OTJ = 32;  // tile extent along j
#ifndef AMB_OSTRIP
#define AMB_OSTRIP 4
#endif
#ifndef AMB_OBPS
#define AMB_OBPS 3   // H100 SXM (400 W): orthomosaic 2.22 ms at 3 blocks/SM vs 2.44 ms at 4 (ortho_c3_gray)
#endif
constexpr int kOStrip = AMB_OSTRIP;  // cells per thread (adjacent along j); tuning knobs AMB_OSTRIP / AMB_OBPS (resident blocks
                                     // per SM the register allocation targets) are compile-time: see DESIGN.md §4.2
constexpr int kOrthoThreads = OTI * OTJ / kOStrip;

struct FrameConst {
  double m[9];  // R_C_G (row-major): X_c = m * X + t
  double t[3];  // -R_C_G * t_G_C
};
static_assert(sizeof(FrameConst) * kMaxFramesPerLaunch <= 64 * 1024, "constant memory budget");

__constant__ FrameConst c_frames[kMaxFramesPerLaunch];

// c_frames is one symbol per device: launches of different contexts (streams) on the same device must not
// overwrite it while another context's kernel still reads it.  Every upload waits for the previous user's kernel
// (an event per device), whatever stream that was on.
struct ConstantGuard {
  std::mutex mu;
  cudaEvent_t last_use[64] = {};
};
ConstantGuard g_constant_guard;

struct OrthoArgs {
  const float* elevation;
  float* elevation_angle;
  float* observation_index;
  float* out_layer;               // `ortho` (gray) or `colored_ortho` (packed colour bits)
  const uint8_t* const* images;   // device array: frame -> device raster
  const double* cull_data;        // device array [n_frames][12]: camera centre, R_C_G rows (map frame)
  unsigned int* error_flag;
  unsigned int* pix;              // SELECT mode: per cell (py << 16 | px) of the winner, untouched if not updated
  int* bbox;                      // SELECT mode: per frame [xmin, ymin, xmax, ymax] of the winners' pixels
  size_t row_step;
  int n_frames, frame_base;       // frames in this launch; index of its first frame within the process() call
  int rows, cols_slab, col_begin;
  int width, height, channels, colored;
  int dist_type;
  int do_cull;                    // 0: brute force over all frames
  int cone;                       // 1: view-cone test active (else only "behind the camera")
  int rect;                       // 1: view-rectangle test active (bounds on the undistorted normalised keypoint)
  double u_lo, u_hi, v_lo, v_hi;  // visible  =>  u in [u_lo, u_hi], v in [v_lo, v_hi]   (u = x_c/z_c, v = y_c/z_c)
  double nu_lo, nu_hi, nv_lo, nv_hi;  // sqrt(1 + bound^2): norms of the bounding planes' normals
  double base_x, base_y, res;
  double fu, fv, cu, cv;
  double d0, d1, d2, d3;
  double cos_c, sin_c;            // half-angle of the conservative view cone
  // dominance cull, rect: every ray with undistorted normalised keypoint inside [ui_lo, ui_hi] x [vi_lo, vi_hi] (and
  // z_c > 0) IS visible
  double ui_lo, ui_hi, vi_lo, vi_hi;
  double nui_lo, nui_hi, nvi_lo, nvi_hi;  // sqrt(1 + bound^2)
  double dom_cos_in;                      // cone: every ray whose angle to the axis has a larger cosine is imaged
  double dom_cos_margin, dom_sin_margin;  // cos / sin of the dominance margin
  int dominance;                          // 1: per-tile dominance cull of the frame list (needs the inner bounds above)
  const double* exact_data;               // device array [n_frames][8]: inverse(T_G_C) as the reference forms it —
                                          // conjugate quaternion (w, x, y, z), translation -(q^-1).rotate(t), pad
  // scaling of the guards with the inputs' magnitude (see kDeltaUlps): per tile delta = delta_coef * max(t_max, |X|,
  // |Y|, |Z| over the tile's cells) bounds |fast - reference| of each camera coordinate
  double delta_coef;                      // kDeltaUlps * 2^-53 * max(1, |q|^2 over the frames)
  double t_max;                           // largest |component| of t_G_C and of -R_C_G t_G_C over the frames
  double px_coef;                         // max(fu, fv) * J: keypoint error <= px_coef * delta / z_c
};

// Guard bands of the fused fast path.  Its camera coordinates come from a pre-multiplied rotation matrix with FMA
// contraction and a <= 1 ulp reciprocal; the reference (minkindr / Eigen / aslam_cv2, see exact_* below) rotates by the
// quaternion formula and divides.  A decision closer to its boundary than the guard is re-made with the reference's
// own operation sequence, un-contracted, so visibility, winner and pixel are the reference's by construction.
// The two sequences round intermediate values as large as the inputs: with M the largest |X|, |Y|, |Z| of the
// landmark and |t| of the pose, each camera coordinate differs by at most delta = kDeltaUlps * 2^-53 * M.  Counted
// with unit roundoff u = 2^-53 and |q_i| <= 1: the matrix entries carry <= 16 u each (3 of them per coordinate: 48 u M)
// and the three FMAs round values <= 2M, 3M, 4M (9 u M), 57 u M for the fast path; the quaternion formula rounds
// q x v (4 u M, doubled to 8), q x (q x v) (32 u M), the sums (18 u M) and + t (2 u M), 60 u M for the reference.
// Near the map origin M is ~1e3 m and delta ~1e-11 m; at UTM coordinates (5e6 .. 1e7 m) delta is ~1e-7 m.  The guards:
//   keypoint: kGuardPx + px_coef * delta / z_c        (u = x/z moves by <= delta (1 + |u|) / z, times the distortion's
//                                                      row-sum derivative J on the view cone, J including (1 + r_c))
//   camera z: kGuardZ + delta
//   sin^2 of the observation angle: the band of the running best + 2 delta / z_c  (|d(z^2/n^2)| <= sqrt(3) delta / n,
//                                                      n >= z_c), for the candidate and, while pending, for the winner
constexpr double kGuardPx = 1e-9;   // keypoint vs raster edge / half-integer: rounding of the projection itself
constexpr double kGuardZ = 1e-6;    // camera z vs kMinimumDepth (1e-10): anything that close to the camera plane goes exact
constexpr double kDeltaUlps = 128.0;

// ---- the reference's arithmetic, operation by operation (restated third-party code: oracle/thirdparty_math.h cites the
// upstream sources; parity tests compare with it), no FMA contraction, IEEE division ----
// Eigen QuaternionBase::_transformVector: uv = q.vec x v; uv += uv; v + q.w*uv + q.vec x uv
__device__ __forceinline__ void exact_quat_rotate(double qw, double qx, double qy, double qz, double vx, double vy,
                                                  double vz, double* rx, double* ry, double* rz) {
  double ux = __dadd_rn(__dmul_rn(qy, vz), -__dmul_rn(qz, vy));
  double uy = __dadd_rn(__dmul_rn(qz, vx), -__dmul_rn(qx, vz));
  double uz = __dadd_rn(__dmul_rn(qx, vy), -__dmul_rn(qy, vx));
  ux = __dadd_rn(ux, ux);
  uy = __dadd_rn(uy, uy);
  uz = __dadd_rn(uz, uz);
  const double cx = __dadd_rn(__dmul_rn(qy, uz), -__dmul_rn(qz, uy));
  const double cy = __dadd_rn(__dmul_rn(qz, ux), -__dmul_rn(qx, uz));
  const double cz = __dadd_rn(__dmul_rn(qx, uy), -__dmul_rn(qy, ux));
  *rx = __dadd_rn(__dadd_rn(vx, __dmul_rn(qw, ux)), cx);
  *ry = __dadd_rn(__dadd_rn(vy, __dmul_rn(qw, uy)), cy);
  *rz = __dadd_rn(__dadd_rn(vz, __dmul_rn(qw, uz)), cz);
}

// T_G_C.inverse().transform(landmark) (ortho-backward-grid.cc:157-158): q^-1.rotate(p) + t_inv
__device__ __noinline__ void exact_to_camera(const OrthoArgs& a, int f, double X, double Y, double Z, double* xc,
                                                double* yc, double* zc) {
  const double* e = a.exact_data + 8 * static_cast<size_t>(f);
  double rx, ry, rz;
  exact_quat_rotate(__ldg(e + 0), __ldg(e + 1), __ldg(e + 2), __ldg(e + 3), X, Y, Z, &rx, &ry, &rz);
  *xc = __dadd_rn(rx, __ldg(e + 4));
  *yc = __dadd_rn(ry, __ldg(e + 5));
  *zc = __dadd_rn(rz, __ldg(e + 6));
}

// aslam::PinholeCamera::project3Functional + the reference's keypoint_visible predicate (:159-171)
template <int DIST>
__device__ __noinline__ bool exact_project(const OrthoArgs& a, double x, double y, double z, double* kx, double* ky) {
  const double rz = __ddiv_rn(1.0, z);
  double u = __dmul_rn(x, rz);
  double v = __dmul_rn(y, rz);
  if (DIST == AMB_DIST_RADTAN) {
    const double mx2 = __dmul_rn(u, u), my2 = __dmul_rn(v, v), mxy = __dmul_rn(u, v);
    const double rho2 = __dadd_rn(mx2, my2);
    const double rad = __dadd_rn(__dmul_rn(a.d0, rho2), __dmul_rn(__dmul_rn(a.d1, rho2), rho2));
    // x += x*rad + 2*p1*mxy + p2*(rho2 + 2*mx2)   (left to right)
    const double ax = __dadd_rn(__dadd_rn(__dmul_rn(u, rad), __dmul_rn(__dmul_rn(2.0, a.d2), mxy)),
                                __dmul_rn(a.d3, __dadd_rn(rho2, __dmul_rn(2.0, mx2))));
    const double ay = __dadd_rn(__dadd_rn(__dmul_rn(v, rad), __dmul_rn(__dmul_rn(2.0, a.d3), mxy)),
                                __dmul_rn(a.d2, __dadd_rn(rho2, __dmul_rn(2.0, my2))));
    u = __dadd_rn(u, ax);
    v = __dadd_rn(v, ay);
  } else if (DIST == AMB_DIST_EQUIDISTANT) {
    const double r = sqrt(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)));
    if (r > 1e-8) {
      const double th = atan(r);
      const double th2 = __dmul_rn(th, th), th4 = __dmul_rn(th2, th2), th6 = __dmul_rn(th4, th2), th8 = __dmul_rn(th4, th4);
      const double poly = __dadd_rn(__dadd_rn(__dadd_rn(__dadd_rn(1.0, __dmul_rn(a.d0, th2)), __dmul_rn(a.d1, th4)),
                                              __dmul_rn(a.d2, th6)), __dmul_rn(a.d3, th8));
      const double s = __ddiv_rn(__dmul_rn(th, poly), r);
      u = __dmul_rn(u, s);
      v = __dmul_rn(v, s);
    }
  } else if (DIST == AMB_DIST_FOV) {
    // oracle/thirdparty_math.h, FOV branch, operation by operation (tan(w/2) = a.d1, evaluated by the host libm)
    const double r = sqrt(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)));
    const double at = atan(__dmul_rn(__dmul_rn(2.0, a.d1), r));
    double s;
    if (__dmul_rn(a.d0, a.d0) < 1e-5) {
      s = 1.0;
    } else if (__dmul_rn(r, r) < 1e-5) {
      s = __ddiv_rn(__dmul_rn(2.0, a.d1), a.d0);
    } else {
      s = __ddiv_rn(at, __dmul_rn(r, a.d0));
    }
    u = __dmul_rn(u, s);
    v = __dmul_rn(v, s);
  }
  *kx = __dadd_rn(__dmul_rn(a.fu, u), a.cu);
  *ky = __dadd_rn(__dmul_rn(a.fv, v), a.cv);
  return (*kx >= 0.0) && (*ky >= 0.0) && (*kx < static_cast<double>(a.width)) &&
         (*ky < static_cast<double>(a.height)) && (z > 1e-10);
}

__device__ __noinline__ double exact_observation_angle(double xc, double yc, double zc) {
  // u.norm() (:175) = sqrt(x*x + y*y + z*z), then asin(fabs(u(2)) / norm_u) (:177)
  const double n = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(xc, xc), __dmul_rn(yc, yc)), __dmul_rn(zc, zc)));
  return asin(__ddiv_rn(fabs(zc), n));
}

// aslam::PinholeCamera::project3: rz = 1/z; (u,v) = (x,y)*rz; distort; k = f*u + c.  Returns the reference's
// keypoint_visible predicate (ortho-backward-grid.cc:164-171): inside the raster and z > 1e-10
// (POINT_BEHIND_CAMERA is z < 0, PROJECTION_INVALID is 0 <= z <= 1e-10; both rejected).  *rzp: the reciprocal of z
// (of 1e-300 for z <= 0), which scales the guards.
template <int DIST>
__device__ __forceinline__ bool project(const OrthoArgs& a, double x, double y, double z, double* kx, double* ky,
                                        double* rzp) {
  const double rz = fast_rcp(fmax(z, 1e-300));  // 1.0 / z to <= 1 ulp; z <= 1e-10 is rejected below
  *rzp = rz;
  double u = x * rz;
  double v = y * rz;
  if (DIST == AMB_DIST_RADTAN) {
    const double mx2 = u * u, my2 = v * v, mxy = u * v;
    const double rho2 = mx2 + my2;
    const double rad = a.d0 * rho2 + a.d1 * rho2 * rho2;
    const double un = u + (u * rad + 2.0 * a.d2 * mxy + a.d3 * (rho2 + 2.0 * mx2));
    const double vn = v + (v * rad + 2.0 * a.d3 * mxy + a.d2 * (rho2 + 2.0 * my2));
    u = un;
    v = vn;
  } else if (DIST == AMB_DIST_EQUIDISTANT) {
    const double r = sqrt(u * u + v * v);
    if (r > 1e-8) {
      const double th = atan(r);
      const double th2 = th * th, th4 = th2 * th2, th6 = th4 * th2, th8 = th4 * th4;
      const double thd = th * (1.0 + a.d0 * th2 + a.d1 * th4 + a.d2 * th6 + a.d3 * th8);
      const double s = thd / r;
      u *= s;
      v *= s;
    }
  } else if (DIST == AMB_DIST_FOV) {
    // aslam FisheyeDistortion, d0 = w, d1 = tan(w/2) from the HOST libm (restated from recollection of upstream: see
    // AMB_DIST_FOV in include/aerial_mapper_b200.h)
    const double r = sqrt(u * u + v * v);
    double s = 1.0;
    if (!(a.d0 * a.d0 < 1e-5)) s = (r * r < 1e-5) ? 2.0 * a.d1 / a.d0 : atan(2.0 * a.d1 * r) / (r * a.d0);
    u *= s;
    v *= s;
  }
  *kx = a.fu * u + a.cu;
  *ky = a.fv * v + a.cv;
  return (*kx >= 0.0) && (*ky >= 0.0) && (*kx < static_cast<double>(a.width)) &&
         (*ky < static_cast<double>(a.height)) && (z > 1e-10);
}

// X_c = R_C_G X - R_C_G t_G_C for frame f (T_G_C^-1 . landmark, ortho-backward-grid.cc:157-158)
__device__ __forceinline__ void to_camera(int f, double X, double Y, double Z, double* xc, double* yc, double* zc) {
  const FrameConst& fc = c_frames[f];
  *xc = fma(fc.m[1], Y, fma(fc.m[2], Z, fma(fc.m[0], X, fc.t[0])));
  *yc = fma(fc.m[4], Y, fma(fc.m[5], Z, fma(fc.m[3], X, fc.t[1])));
  *zc = fma(fc.m[7], Y, fma(fc.m[8], Z, fma(fc.m[6], X, fc.t[2])));
}

// asin(fabs(u(2)) / norm_u) exactly as the reference evaluates it (ortho-backward-grid.cc:175-177)
__device__ __forceinline__ double observation_angle(double xc, double yc, double zc) {
  return asin(fabs(zc) / sqrt(xc * xc + yc * yc + zc * zc));
}

// Layer value of a texel (:194-206).  Colour: cv::Vec3b is (B,G,R) and grid_map::colorVectorToValue packs 0x00RRGGBB,
// moved as raw bits (int(float(c/255.0)*255.0f) == c for every byte c; tests/test_oracle_ortho.py checks all 256).
__device__ __forceinline__ float texel_value(const uint8_t* texel, int colored) {
  if (colored) {
    const unsigned int b = __ldg(texel), g = __ldg(texel + 1), r = __ldg(texel + 2);
    return __uint_as_float((r << 16) | (g << 8) | b);
  }
  return static_cast<float>(__ldg(texel));
}

// Frame f (index within the launch) won `cell` with angle `angle` and keypoint (kx, ky): write the angle and the frame
// index (:181-182; :183 num_observations += num_observations keeps 0 at 0, the layer is untouched), then the pixel is
// round(keypoint), half away from zero, clamped to the last row / column (:186-193).  SELECT records the pixel and
// grows the frame's bounding box in shared memory; otherwise the texel is fetched.  (The keypoint is taken by reference:
// it may sit in local memory after the exact path, and is then read where the pixel is rounded, not at the call.)
template <bool SELECT>
__device__ __forceinline__ void store_winner(const OrthoArgs& a, int* s_bbox, size_t cell, int f, float angle,
                                             const double& kx, const double& ky) {
  a.elevation_angle[cell] = angle;
  a.observation_index[cell] = static_cast<float>(a.frame_base + f);
  const int py = min(static_cast<int>(round(ky)), a.height - 1);
  const int px = min(static_cast<int>(round(kx)), a.width - 1);
  if (SELECT) {
    a.pix[cell] = (static_cast<unsigned int>(py) << 16) | static_cast<unsigned int>(px);
    atomicMin(&s_bbox[f], px);
    atomicMin(&s_bbox[kMaxFramesPerLaunch + f], py);
    atomicMax(&s_bbox[2 * kMaxFramesPerLaunch + f], px);
    atomicMax(&s_bbox[3 * kMaxFramesPerLaunch + f], py);
  } else {
    const uint8_t* texel = a.images[f] + static_cast<size_t>(py) * a.row_step + static_cast<size_t>(px) * a.channels;
    a.out_layer[cell] = texel_value(texel, a.colored);
  }
}

// The initial values of the layers a cell's winner writes (AerialGridMap's, ensure_layer), for a cell no frame wins in a
// FRESH launch
__device__ __forceinline__ void store_initial(const OrthoArgs& a, size_t cell) {
  a.elevation_angle[cell] = 0.0f;
  a.observation_index[cell] = __int_as_float(0x7fc00000);
  a.out_layer[cell] = a.colored ? __int_as_float(0x7fc00000) : 255.0f;
}

// ... for every cell of a thread's strip inside the slab (a tile that returns before its winner selection)
__device__ __forceinline__ void store_initial_strip(const OrthoArgs& a, int i, int jl0) {
  if (i >= a.rows) return;
#pragma unroll
  for (int m = 0; m < kOStrip; ++m)
    if (jl0 + m < a.cols_slab) store_initial(a, static_cast<size_t>(jl0 + m) * a.rows + i);
}

// One block = one OTI x OTJ cell tile; one thread = a 1 x kOStrip strip of cells (same i, adjacent j): the
// per-frame constants are fetched once per thread and serve four cells, and the tile's cull list is built once
// for 1024 cells.
// SELECT = false: fused kernel, frames resident in HBM, the winner's texel is fetched in the epilogue.
// SELECT = true:  phase A of the host-frame path: no texel access at all; records the winner's pixel per cell and
//                 the bounding box of the winners' pixels per frame, so that only those sub-rectangles of the
//                 host frames have to cross PCIe (phase B: ortho_texel_kernel).
// FRESH = true (fused kernel only): elevation_angle, observation_index and out_layer are fresh (ensure_layer_overwrite):
//                 the running best starts at their known initial 0 without a load, and every cell of the tile that no
//                 frame wins takes the layers' initial values (store_initial).  A template parameter: as a run-time flag
//                 the extra stores doubled the spills of the other instances.
//
// The frame list is culled by conservative view cone / rectangle tests (unless a.do_cull == 0: brute force) and, with
// a.dominance, by the per-tile DOMINANCE cull:
//   alpha = asin(|z_c| / |X - c|) = pi/2 - theta, theta = angle between the ray and the optical axis.  Over the
//   tile's bounding sphere (centre C, radius rho) theta lies in [max(0, theta_c - delta), theta_c + delta],
//   theta_c = angle(axis, C - c), delta = asin(rho / |C - c|).  If a frame g sees EVERY landmark of the tile (sphere
//   in front of the camera and inside the view rectangle shrunk by the distortion bound), any frame f with
//   theta_min(f) > theta_max(g) + margin has a smaller alpha than g in every cell, by far more than the float32
//   rounding of the running best can hide: whether or not f is visited, the reference's sequential recurrence ends
//   in the same (angle, index) — after g has been visited the state is the same, and a frame between them that wins
//   against the state without f also wins against the state with f or loses to g afterwards.  Dropping f therefore
//   changes no output bit (tools/ortho_dominance_study.py checks this against the oracle) and leaves ~1.2 instead of
//   ~8.5 frames per tile at the benchmark geometry.
template <int DIST, bool SELECT, bool FRESH>
__global__ void __launch_bounds__(kOrthoThreads, AMB_OBPS) ortho_kernel_dom(const __grid_constant__ OrthoArgs a) {
  static_assert(!(SELECT && FRESH), "SELECT writes no texel: the host-frame path never runs fresh");
  __shared__ unsigned short s_list[kMaxFramesPerLaunch];
  __shared__ int s_bbox[SELECT ? 4 * kMaxFramesPerLaunch : 4];
  __shared__ float s_red[2][kOrthoThreads / 32];
  __shared__ int s_warp_cnt[kOrthoThreads / 32];
  __shared__ int s_total;

  const int ti = threadIdx.x & 31, tq = threadIdx.x >> 5;
  const int tiles_i = (a.rows + OTI - 1) / OTI;
  const int i0 = (blockIdx.x % tiles_i) * OTI;
  const int j0 = (blockIdx.x / tiles_i) * OTJ;
  // ti / tq = lane / warp; a warp covers 32 consecutive rows of one strip column group (OTI may span several warps)
  const int i = i0 + (tq % (OTI / 32)) * 32 + ti;
  const int jl0 = j0 + kOStrip * (tq / (OTI / 32));

  float elev[kOStrip];
  unsigned int validmask = 0;
  float zmin = FLT_MAX, zmax = -FLT_MAX;
#pragma unroll
  for (int m = 0; m < kOStrip; ++m) {
    elev[m] = __int_as_float(0x7fc00000);
    if (i < a.rows && jl0 + m < a.cols_slab) elev[m] = a.elevation[static_cast<size_t>(jl0 + m) * a.rows + i];
    if (!isnan(elev[m])) {  // NaN elevation: every comparison is false, the cell stays untouched
      validmask |= 1u << m;
      zmin = fminf(zmin, elev[m]);
      zmax = fmaxf(zmax, elev[m]);
    }
  }
  // tile elevation range
  for (int o = 16; o > 0; o >>= 1) {
    zmin = fminf(zmin, __shfl_xor_sync(0xffffffffu, zmin, o));
    zmax = fmaxf(zmax, __shfl_xor_sync(0xffffffffu, zmax, o));
  }
  if (ti == 0) {
    s_red[0][tq] = zmin;
    s_red[1][tq] = zmax;
  }
  if (threadIdx.x == 0) s_total = 0;
  if (SELECT) {
    for (int e = threadIdx.x; e < 2 * kMaxFramesPerLaunch; e += kOrthoThreads) {
      s_bbox[e] = 0x7fffffff;                            // xmin, ymin
      s_bbox[2 * kMaxFramesPerLaunch + e] = -1;          // xmax, ymax
    }
  }
  __syncthreads();
  zmin = s_red[0][0];
  zmax = s_red[1][0];
#pragma unroll
  for (int w = 1; w < kOrthoThreads / 32; ++w) {
    zmin = fminf(zmin, s_red[0][w]);
    zmax = fmaxf(zmax, s_red[1][w]);
  }
  if (zmin > zmax) {  // no cell of this tile has an elevation
    if (FRESH) store_initial_strip(a, i, jl0);
    return;
  }

  // bounding sphere of the tile's landmarks (cell centres x elevation range)
  const int i1 = min(i0 + OTI, a.rows) - 1, j1 = min(j0 + OTJ, a.cols_slab) - 1;
  const double x_hi = a.base_x - a.res * i0, x_lo = a.base_x - a.res * i1;
  const double y_hi = a.base_y - a.res * (a.col_begin + j0), y_lo = a.base_y - a.res * (a.col_begin + j1);
  const double sx = 0.5 * (x_hi + x_lo), sy = 0.5 * (y_hi + y_lo);
  const double sz = 0.5 * (static_cast<double>(zmin) + static_cast<double>(zmax));
  const double ex = 0.5 * (x_hi - x_lo), ey = 0.5 * (y_hi - y_lo);
  const double ez = 0.5 * (static_cast<double>(zmax) - static_cast<double>(zmin));
  const double rho = sqrt(ex * ex + ey * ey + ez * ez) * (1.0 + 1e-9) + 1e-6;
  // bound on |fast path - reference| of a camera coordinate over this tile's cells (see kDeltaUlps)
  const double delta = a.delta_coef * fmax(fmax(a.t_max, fmax(fabs(x_hi), fabs(x_lo))),
                                           fmax(fmax(fabs(y_hi), fabs(y_lo)),
                                                static_cast<double>(fmaxf(fabsf(zmin), fabsf(zmax)))));

  {
    // The angles are compared through their COSINES (cos is decreasing on [0, pi]), built from the sphere centre's camera
    // coordinates with the addition formulas — no atan2 / asin per (tile, frame), which was 23 % of the kernel's
    // instructions (the cull only has to be SOUND, not to reproduce a particular rounding: whichever frames it drops,
    // the output is the same by the argument above):
    //   cos(theta_c) = z_c / |C - c|, sin(theta_c) = perp / |C - c|, sin(delta) = rho / |C - c|
    //   cos(theta_min) = 1 if theta_c <= delta, else cos(theta_c - delta);   cos(theta_max) = cos(theta_c + delta)
    __shared__ double s_cmin[kMaxFramesPerLaunch];     // cos(theta_min) per surviving frame, NaN: not a candidate
    __shared__ unsigned long long s_best_cmax;         // largest cos(theta_max) among the frames that see the whole tile
    // pass 1: the conservative visibility tests, plus cos(theta_min) per surviving frame and (a.dominance) the largest
    // cos(theta_max) among the frames that see the whole tile (doubles > 0 order like their bit patterns: atomicMax)
    if (threadIdx.x == 0) s_best_cmax = 0ull;  // no whole-tile frame yet (theirs are > 0: the sphere is in front of them)
    __syncthreads();
    for (int f = threadIdx.x; f < a.n_frames; f += kOrthoThreads) {
      // per-thread frame index: read from global memory (a divergent __constant__ index would serialise)
      const double* cf = a.cull_data + 12 * static_cast<size_t>(f);
      const double dx = sx - __ldg(cf + 0), dy = sy - __ldg(cf + 1), dz = sz - __ldg(cf + 2);
      const double xp = dx * __ldg(cf + 3) + dy * __ldg(cf + 4) + dz * __ldg(cf + 5);    // x_c of the centre
      const double yp = dx * __ldg(cf + 6) + dy * __ldg(cf + 7) + dz * __ldg(cf + 8);    // y_c
      const double zp = dx * __ldg(cf + 9) + dy * __ldg(cf + 10) + dz * __ldg(cf + 11);  // z_c (optical axis)
      const double dd = dx * dx + dy * dy + dz * dz;
      const double slack = rho + 1e-9 * (fabs(xp) + fabs(yp) + fabs(zp));
      const double perp = sqrt(fmax(dd - zp * zp, 0.0));
      bool keep = true;
      if (zp + rho <= 0.0) {
        keep = false;  // whole sphere behind the camera plane: z_c <= 0 for every landmark
      } else {
        // distance from the sphere centre to the solid cone {angle to axis <= theta_c} is at least
        // perp*cos(theta_c) - zp*sin(theta_c)
        if (a.cone) {
          if (perp * a.cos_c - zp * a.sin_c > slack) keep = false;
        }
        // a landmark with z_c > 0 and u = x_c/z_c > u_hi has x_c - u_hi*z_c > 0: the sphere lies entirely on
        // that side of the plane through the camera centre iff the centre's value exceeds rho*|normal|
        if (a.rect) {
          if (xp - a.u_hi * zp > slack * a.nu_hi) keep = false;
          if (a.u_lo * zp - xp > slack * a.nu_lo) keep = false;
          if (yp - a.v_hi * zp > slack * a.nv_hi) keep = false;
          if (a.v_lo * zp - yp > slack * a.nv_lo) keep = false;
        }
      }
      double c_min = __longlong_as_double(0x7ff8000000000000ll);  // NaN: not a candidate
      if (keep) {
        const double inv = 1.0 / sqrt(dd);  // (dd == 0: inf — the camera sits on the sphere centre)
        double c_max = -1.0;
        c_min = 1.0;  // camera inside the tile's sphere: theta_min = 0 and the frame cannot "see the whole tile"
        if (rho * inv < 1.0) {
          const double cos_t = zp * inv, sin_t = perp * inv;
          const double sin_d = rho * inv;
          const double cos_d = sqrt(fmax(1.0 - sin_d * sin_d, 0.0));
          c_min = cos_t >= cos_d ? 1.0 : cos_t * cos_d + sin_t * sin_d;
          c_max = cos_t * cos_d - sin_t * sin_d;
        }
        // every landmark of the tile is imaged by this frame: pinhole / rad-tan — sphere inside the INNER view rectangle;
        // equidistant / FOV — sphere inside the INNER view cone (every ray whose angle to the axis has a cosine above
        // dom_cos_in lands in the raster; with the sphere in front of the camera theta_c + delta < pi/2, so the cosines
        // compare like the angles)
        const bool whole = a.dominance && zp - rho > 1e-6 && c_max > 0.0 &&
                           (a.rect ? (xp - a.ui_hi * zp < -slack * a.nui_hi && a.ui_lo * zp - xp < -slack * a.nui_lo &&
                                      yp - a.vi_hi * zp < -slack * a.nvi_hi && a.vi_lo * zp - yp < -slack * a.nvi_lo)
                                   : (c_max > a.dom_cos_in + 1e-12));
        if (whole) atomicMax(&s_best_cmax, static_cast<unsigned long long>(__double_as_longlong(c_max)));
      }
      s_cmin[f] = a.do_cull ? c_min : 1.0;  // brute force: every frame is a candidate (and a.dominance is 0)
    }
    __syncthreads();
    // a frame is dropped when theta_min > theta_max(best) + margin, i.e. cos(theta_min) < cos(theta_max + margin)
    // (1e-12 covers the rounding of the products above; the margin itself is 1e-4 rad)
    double c_cut = -2.0;  // no whole-tile frame (always so without a.dominance): nothing is dropped
    if (s_best_cmax != 0ull) {
      const double c = __longlong_as_double(static_cast<long long>(s_best_cmax));
      c_cut = c * a.dom_cos_margin - sqrt(fmax(1.0 - c * c, 0.0)) * a.dom_sin_margin - 1e-12;
    }
    // pass 2: ascending list of the candidates no whole-tile frame dominates
    for (int f0 = 0; f0 < a.n_frames; f0 += kOrthoThreads) {
      const int f = f0 + threadIdx.x;
      bool keep = false;
      if (f < a.n_frames) {
        const double c_min = s_cmin[f];
        keep = c_min == c_min && !(c_min < c_cut);
      }
      const unsigned int mk = __ballot_sync(0xffffffffu, keep);
      if (ti == 0) s_warp_cnt[tq] = __popc(mk);
      __syncthreads();
      int before = s_total;
      for (int w = 0; w < tq; ++w) before += s_warp_cnt[w];
      if (keep) s_list[before + __popc(mk & ((1u << ti) - 1u))] = static_cast<unsigned short>(f);
      __syncthreads();
      if (threadIdx.x == 0) {
        int t = s_total;
        for (int w = 0; w < kOrthoThreads / 32; ++w) t += s_warp_cnt[w];
        s_total = t;
      }
      __syncthreads();
    }
  }
  const int n_list = s_total;
#ifdef AMB_CUDA_EMU  // tests/emu only: how many frames the tile keeps (plain vs dominance cull)
  if (threadIdx.x == 0) emu::note(a.dominance ? "ortho_dom_list" : "ortho_list", n_list);
#endif
  if (n_list == 0) {
    if (FRESH) store_initial_strip(a, i, jl0);
    return;
  }
  if (!SELECT && !validmask) {  // (SELECT: every thread reaches the block-wide bbox flush below)
    if (FRESH) store_initial_strip(a, i, jl0);
    return;
  }

  // ---- winner selection: the reference's recurrence  `alpha_f > (double)best_f32  =>  best_f32 = (float)alpha_f`
  // with alpha = asin(|z|/norm)  (ortho-backward-grid.cc:173-183), evaluated WITHOUT an asin per candidate.
  // asin is increasing with slope >= 1, so comparing s2 = z^2/norm^2 = sin^2(alpha) decides the comparison
  // whenever the gap is larger than what the float32 rounding of the running best can hide:
  //   running best known exactly (layer value b):          ref2 = sin^2(b), band 1e-11
  //   running best = (float)asin(s_p) of a pending winner: ref2 = s_p^2,    band 2e-7
  //       (|(float)a - a| <= 6.0e-8 * a <= 9.4e-8;  s2_f - s2_p > 2e-7  =>  s_f - s_p > 1e-7  =>  alpha_f - alpha_p > 1e-7)
  // Inside the band the decision is made exactly as the reference does (asin of both, float-rounded best).
  const double X = __dadd_rn(a.base_x, __dmul_rn(a.res, -static_cast<double>(i)));
  double Y[kOStrip], Z[kOStrip], thr_hi[kOStrip], thr_lo[kOStrip];
  float best[kOStrip];
  int best_f[kOStrip];
  unsigned int pending = 0;  // bit m: best_f[m] won but (float)asin(...) has not been evaluated yet
#pragma unroll
  for (int m = 0; m < kOStrip; ++m) {
    Y[m] = __dadd_rn(a.base_y, __dmul_rn(a.res, -static_cast<double>(a.col_begin + jl0 + m)));
    Z[m] = static_cast<double>(elev[m]);
    best[m] = 0.0f;
    best_f[m] = -1;
    double ref2 = 4.0, band = 0.0;  // invalid cell: nothing can win
    if ((validmask >> m) & 1u) {
      best[m] = FRESH ? 0.0f : a.elevation_angle[static_cast<size_t>(jl0 + m) * a.rows + i];
      if (best[m] > 0.0f) {
        const double sb = sin(static_cast<double>(best[m]));
        ref2 = sb * sb;
        band = 1e-11;
      } else if (best[m] == 0.0f) {
        ref2 = 0.0;  // any visible frame has alpha > 0
      } else if (best[m] < 0.0f) {
        ref2 = -1.0;  // a negative layer value is beaten by anything; NaN (ref2 = 4) by nothing
      }
    }
    thr_hi[m] = ref2 + band;
    thr_lo[m] = ref2 - band;
  }
  bool check_failed = false;
  unsigned int dirty = 0;  // bit m: a candidate fell inside a band (angle tie / raster edge / camera plane) -> redo exactly
  const double wd = static_cast<double>(a.width), hd = static_cast<double>(a.height);
  // the guards at this tile's magnitude: per candidate, pixel guard = kGuardPx + gpx_c / z_c, sin^2 band + band_c / z_c
  const double guard_z = kGuardZ + delta;
  const double gpx_c = a.px_coef * delta;
  const double band_c = 2.0 * delta;

  // ---- one candidate frame (after the dominance cull: ~4 of 5 tiles at the benchmark geometry) ----
  // The frame loop below projects the winner a second time after its frame loop (like the reference, :186-188) because
  // keeping every cell's winning keypoint across the loop costs registers; with a single candidate there is no loop state:
  // each cell is evaluated, decided (exact re-evaluation included) and written in one go, from the SAME camera
  // coordinates and keypoint (to_camera / project are the expressions of the loop body: identical bits).  The winner's
  // re-projection was a third of the kernel's instructions.
  if (n_list == 1) {  // block-uniform
    const int f = s_list[0];
    const FrameConst& fc = c_frames[f];
    const double cx = fma(fc.m[0], X, fc.t[0]);
    const double cy = fma(fc.m[3], X, fc.t[1]);
    const double cz = fma(fc.m[6], X, fc.t[2]);
#pragma unroll
    for (int m = 0; m < kOStrip; ++m) {
      if (!((validmask >> m) & 1u)) {  // no elevation / beyond the map edge: untouched, nothing is read
        if (FRESH && i < a.rows && jl0 + m < a.cols_slab) store_initial(a, static_cast<size_t>(jl0 + m) * a.rows + i);
        continue;
      }
      double xc = fma(fc.m[1], Y[m], fma(fc.m[2], Z[m], cx));
      double yc = fma(fc.m[4], Y[m], fma(fc.m[5], Z[m], cy));
      double zc = fma(fc.m[7], Y[m], fma(fc.m[8], Z[m], cz));
      double kx, ky, rz;
      project<DIST>(a, xc, yc, zc, &kx, &ky, &rz);
      const double gpx = fma(gpx_c, rz, kGuardPx);
      const bool vis = kx >= gpx && ky >= gpx && kx < wd - gpx && ky < hd - gpx && zc > guard_z;
      const bool out = kx < -gpx || ky < -gpx || kx >= wd + gpx || ky >= hd + gpx || zc < -guard_z;
      const double z2 = zc * zc;
      const double n2 = fma(xc, xc, fma(yc, yc, z2));
      const double en2 = band_c * rz * n2;   // the candidate's own sin^2 error, times n2
      bool win = vis && (z2 - en2 > thr_hi[m] * n2);
      const bool unc = (vis && !win && (z2 + en2 >= thr_lo[m] * n2)) || (!vis && !out);
#ifdef AMB_CUDA_EMU  // tests/emu only: share of cell decisions the guards hand to the exact path
      emu::note("ortho_exact_decision", unc ? 1 : 0);
#endif
      bool pend = win;
      float b = best[m];
      if (unc) {  // too close to call: the reference's own operation sequence decides (as in the general path's dirty branch)
        win = false;
        pend = false;
        double ex, ey, ez, ekx, eky;
        exact_to_camera(a, f, X, Y[m], Z[m], &ex, &ey, &ez);
        if (exact_project<DIST>(a, ex, ey, ez, &ekx, &eky)) {
          const double alpha = exact_observation_angle(ex, ey, ez);
          if (!(alpha > 0.0)) check_failed = true;  // reference: CHECK(alpha > 0.0), :178
          if (alpha > static_cast<double>(b)) {     // :180
            b = static_cast<float>(alpha);          // :181
            win = true;
          }
        }
      }
      if (!win) {
        if (FRESH) store_initial(a, static_cast<size_t>(jl0 + m) * a.rows + i);
        continue;
      }
      const size_t cell = static_cast<size_t>(jl0 + m) * a.rows + i;
      // the pixel is round(keypoint) (:186-193): within the guard of a half-integer (or for a cell that took the exact
      // path) the keypoint is recomputed with the reference's operation sequence
      const bool near_half = fabs((kx - floor(kx)) - 0.5) < gpx || fabs((ky - floor(ky)) - 0.5) < gpx;
#ifdef AMB_CUDA_EMU  // tests/emu only: share of winners whose pixel is rounded from the exact keypoint
      emu::note("ortho_exact_pixel", near_half ? 1 : 0);
#endif
      if (near_half || unc || !(kx == kx) || !(ky == ky)) {
        exact_to_camera(a, f, X, Y[m], Z[m], &xc, &yc, &zc);
        exact_project<DIST>(a, xc, yc, zc, &kx, &ky);
      }
      if (pend) {
        const double alpha = observation_angle(xc, yc, zc);
        if (!(alpha > 0.0)) check_failed = true;
        b = static_cast<float>(alpha);
      }
      store_winner<SELECT>(a, s_bbox, cell, f, b, kx, ky);
    }
    // Own exit rather than a fall-through into the shared flush below: joining the two paths keeps n_list and the flag
    // live across this block, and ptxas then spills more in three of the SELECT instances and reschedules this block.
    if (check_failed) atomicExch(a.error_flag, 1u);
    if (SELECT) {
      __syncthreads();
      if (threadIdx.x == 0 && s_bbox[2 * kMaxFramesPerLaunch + f] >= 0) {
        int* g = a.bbox + 4 * (a.frame_base + f);
        atomicMin(g + 0, s_bbox[f]);
        atomicMin(g + 1, s_bbox[kMaxFramesPerLaunch + f]);
        atomicMax(g + 2, s_bbox[2 * kMaxFramesPerLaunch + f]);
        atomicMax(g + 3, s_bbox[3 * kMaxFramesPerLaunch + f]);
      }
    }
    return;
  }

  // Hot loop: straight-line code, four independent dependency chains per thread (one per cell of the strip).
  for (int l = 0; l < n_list; ++l) {
    const int f = s_list[l];
    const FrameConst& fc = c_frames[f];
    const double cx = fma(fc.m[0], X, fc.t[0]);
    const double cy = fma(fc.m[3], X, fc.t[1]);
    const double cz = fma(fc.m[6], X, fc.t[2]);
#pragma unroll
    for (int m = 0; m < kOStrip; ++m) {
      const double xc = fma(fc.m[1], Y[m], fma(fc.m[2], Z[m], cx));
      const double yc = fma(fc.m[4], Y[m], fma(fc.m[5], Z[m], cy));
      const double zc = fma(fc.m[7], Y[m], fma(fc.m[8], Z[m], cz));
      double kx, ky, rz;
      project<DIST>(a, xc, yc, zc, &kx, &ky, &rz);
      // visibility with a guard band (gpx / guard_z): certainly inside, certainly not visible, or too close to call
      // with FMA-contracted coordinates (NaN keypoints compare false everywhere: too close to call) -> exact path
      const double gpx = fma(gpx_c, rz, kGuardPx);
      const bool vis = kx >= gpx && ky >= gpx && kx < wd - gpx && ky < hd - gpx && zc > guard_z;
      const bool out = kx < -gpx || ky < -gpx || kx >= wd + gpx || ky >= hd + gpx || zc < -guard_z;
      const double z2 = zc * zc;
      const double n2 = fma(xc, xc, fma(yc, yc, z2));
      const double e = band_c * rz;   // bound on this candidate's |sin^2 fast - sin^2 reference|
      const bool win = vis && (fma(-e, n2, z2) > thr_hi[m] * n2);
      // (cells without an elevation — NaN, or beyond the map edge in a partial tile — have NaN keypoints: never "too
      // close to call", nothing can win there and their layer entries must not even be read)
      const bool unc = (vis && !win && (fma(e, n2, z2) >= thr_lo[m] * n2)) || (!vis && !out && ((validmask >> m) & 1u));
      dirty |= (unc ? 1u : 0u) << m;
      const double ref2 = z2 * fast_rcp(n2);
      best_f[m] = win ? f : best_f[m];
      thr_hi[m] = win ? ref2 + (2e-7 + e) : thr_hi[m];   // a pending winner's band carries its own error bound too
      thr_lo[m] = win ? ref2 - (2e-7 + e) : thr_lo[m];
      pending |= (win ? 1u : 0u) << m;
    }
  }

#ifdef AMB_CUDA_EMU
  for (int m = 0; m < kOStrip; ++m)
    if ((validmask >> m) & 1u) emu::note("ortho_exact_decision", (dirty >> m) & 1u);
#endif
  if (dirty) {
    // Rare (a near-tie within the float32 rounding of the running best, a keypoint within 1e-9 px of the raster edge, a
    // landmark on the camera plane): evaluate the reference's recurrence literally for those cells, with the
    // reference's own operation sequence (exact_*: quaternion rotation, IEEE division, no contraction) — asin for
    // every visible frame, float-rounded best (:173-183).
#pragma unroll
    for (int m = 0; m < kOStrip; ++m) {  // unrolled: the per-cell arrays must stay in registers
      if (!((dirty >> m) & 1u)) continue;
      float b = FRESH ? 0.0f : a.elevation_angle[static_cast<size_t>(jl0 + m) * a.rows + i];
      int bf = -1;
      for (int l = 0; l < n_list; ++l) {
        const int f = s_list[l];
        double xc, yc, zc, kx, ky;
        exact_to_camera(a, f, X, Y[m], Z[m], &xc, &yc, &zc);
        if (!exact_project<DIST>(a, xc, yc, zc, &kx, &ky)) continue;
        const double alpha = exact_observation_angle(xc, yc, zc);
        if (!(alpha > 0.0)) check_failed = true;  // reference: CHECK(alpha > 0.0), :178
        if (alpha > static_cast<double>(b)) {     // :180
          b = static_cast<float>(alpha);          // :181
          bf = f;
        }
      }
      best[m] = b;
      best_f[m] = bf;
      pending &= ~(1u << m);
    }
  }

#pragma unroll
  for (int m = 0; m < kOStrip; ++m) {
    if (best_f[m] < 0) {
      if (FRESH && i < a.rows && jl0 + m < a.cols_slab) store_initial(a, static_cast<size_t>(jl0 + m) * a.rows + i);
      continue;
    }
    const size_t cell = static_cast<size_t>(jl0 + m) * a.rows + i;
    // the winner's camera coordinates and keypoint, recomputed (the reference projects a second time too, :186-188)
    double xc, yc, zc, kx, ky, rz;
    to_camera(best_f[m], X, Y[m], Z[m], &xc, &yc, &zc);
    project<DIST>(a, xc, yc, zc, &kx, &ky, &rz);
    // the pixel is round(keypoint) (:186-193): within the guard of a half-integer (or for a cell that already took the
    // exact path) the keypoint is recomputed with the reference's operation sequence
    const double gpx = fma(gpx_c, rz, kGuardPx);
    const bool near_half = fabs((kx - floor(kx)) - 0.5) < gpx || fabs((ky - floor(ky)) - 0.5) < gpx;
#ifdef AMB_CUDA_EMU
    emu::note("ortho_exact_pixel", near_half ? 1 : 0);
#endif
    if (near_half || ((dirty >> m) & 1u) || !(kx == kx) || !(ky == ky)) {
      exact_to_camera(a, best_f[m], X, Y[m], Z[m], &xc, &yc, &zc);
      exact_project<DIST>(a, xc, yc, zc, &kx, &ky);
    }
    if ((pending >> m) & 1u) {
      const double alpha = observation_angle(xc, yc, zc);
      if (!(alpha > 0.0)) check_failed = true;
      best[m] = static_cast<float>(alpha);
    }
    store_winner<SELECT>(a, s_bbox, cell, best_f[m], best[m], kx, ky);
  }
  if (check_failed) atomicExch(a.error_flag, 1u);
  if (SELECT) {
    __syncthreads();
    for (int l = threadIdx.x; l < n_list; l += kOrthoThreads) {
      const int f = s_list[l];
      if (s_bbox[2 * kMaxFramesPerLaunch + f] >= 0) {
        int* g = a.bbox + 4 * (a.frame_base + f);
        atomicMin(g + 0, s_bbox[f]);
        atomicMin(g + 1, s_bbox[kMaxFramesPerLaunch + f]);
        atomicMax(g + 2, s_bbox[2 * kMaxFramesPerLaunch + f]);
        atomicMax(g + 3, s_bbox[3 * kMaxFramesPerLaunch + f]);
      }
    }
  }
}

template <bool SELECT, bool FRESH>
void launch_ortho_kernel(const OrthoArgs& a, int grid, cudaStream_t s) {
  switch (a.dist_type) {
    case AMB_DIST_RADTAN: ortho_kernel_dom<AMB_DIST_RADTAN, SELECT, FRESH><<<grid, kOrthoThreads, 0, s>>>(a); break;
    case AMB_DIST_EQUIDISTANT:
      ortho_kernel_dom<AMB_DIST_EQUIDISTANT, SELECT, FRESH><<<grid, kOrthoThreads, 0, s>>>(a);
      break;
    case AMB_DIST_FOV: ortho_kernel_dom<AMB_DIST_FOV, SELECT, FRESH><<<grid, kOrthoThreads, 0, s>>>(a); break;
    default: ortho_kernel_dom<AMB_DIST_NONE, SELECT, FRESH><<<grid, kOrthoThreads, 0, s>>>(a);
  }
}

// Bounding boxes device -> HOST-MAPPED pinned memory with plain stores: the read-back must not queue behind the
// result layers that are streaming to the host on the device->host copy engine.
__global__ void copy_to_mapped_kernel(const int* __restrict__ src, int* __restrict__ dst, int n) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) dst[k] = src[k];
  __threadfence_system();
}

// Phase B of the host-frame path: one thread per cell fetches the winner's texel from the uploaded sub-rectangle.
struct FrameRect {
  const uint8_t* ptr;  // device copy of rows [y0, y1] x columns [x0, x1] of the frame
  int x0, y0;
  int pitch;           // bytes per row of the device copy
  int pad_;
};

__global__ void __launch_bounds__(256) ortho_texel_kernel(const unsigned int* __restrict__ pix,
                                                          const float* __restrict__ observation_index,
                                                          const FrameRect* __restrict__ rects, float* out_layer,
                                                          size_t cells, int channels, int colored) {
  for (size_t cell = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; cell < cells;
       cell += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const unsigned int p = pix[cell];
    if (p == 0xffffffffu) continue;  // not updated by this process() call
    const int f = static_cast<int>(observation_index[cell]);  // index within this call (exact in float32)
    const FrameRect r = rects[f];
    const int px = static_cast<int>(p & 0xffffu), py = static_cast<int>(p >> 16);
    const uint8_t* texel = r.ptr + static_cast<size_t>(py - r.y0) * r.pitch + static_cast<size_t>(px - r.x0) * channels;
    out_layer[cell] = texel_value(texel, colored);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Host side: pose algebra (kindr::minimal::QuatTransformation / Eigen quaternion formulas, restated)
struct Quat {
  double w, x, y, z;
};
struct V3 {
  double x, y, z;
};
inline Quat qmul(const Quat& a, const Quat& b) {
  return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
          a.w * b.y + a.y * b.w + a.z * b.x - a.x * b.z, a.w * b.z + a.z * b.w + a.x * b.y - a.y * b.x};
}
inline V3 cross(const V3& a, const V3& b) {
  return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
inline V3 qrot(const Quat& q, const V3& v) {
  const V3 qv = {q.x, q.y, q.z};
  V3 uv = cross(qv, v);
  uv.x += uv.x;
  uv.y += uv.y;
  uv.z += uv.z;
  const V3 c = cross(qv, uv);
  return {(v.x + q.w * uv.x) + c.x, (v.y + q.w * uv.y) + c.y, (v.z + q.w * uv.z) + c.z};
}

// Conservative view cone of camera 0: the smallest half-angle theta_c (about the optical axis) such that NO ray
// further off-axis can project inside the raster, for the given distortion model.  A point at normalised radius
// r = tan(theta) is imaged at D(u,v); it is inside the raster only if |D| <= Dmax (the farthest raster corner
// from the principal point, in normalised units).  We lower-bound |D| on intervals of r (or theta) with a
// Lipschitz bound on the radial polynomial and scan from far off-axis inwards; the first interval that might
// reach |D| <= Dmax ends the scan.  If even the outermost interval might (fold-back of a non-monotone
// polynomial, or pure tangential distortion), the cone is disabled and only "behind the camera" culls.
bool compute_view_cone(const amb_camera& cam, double* cos_c, double* sin_c, double* tan_c) {
  const double ax = std::max(cam.cu, cam.width - cam.cu) / std::fabs(cam.fu);
  const double ay = std::max(cam.cv, cam.height - cam.cv) / std::fabs(cam.fv);
  const double dmax = std::sqrt(ax * ax + ay * ay) * (1.0 + 1e-9);
  double rc = -1.0;  // tan(theta_c)
  const double* k = cam.dist;
  if (cam.dist_type == AMB_DIST_NONE || (cam.dist_type == AMB_DIST_RADTAN && k[0] == 0 && k[1] == 0 &&
                                          k[2] == 0 && k[3] == 0)) {
    rc = dmax;
  } else if (cam.dist_type == AMB_DIST_RADTAN) {
    const double k1 = k[0], k2 = k[1], T = std::fabs(k[2]) + std::fabs(k[3]);
    // |D| >= r*|1 + k1 r^2 + k2 r^4| - 4 T r^2   (|tangential| <= 4 T r^2)
    const double rmax = 1.0e3;
    // tail r >= rmax: the leading radial term must dominate and keep growing
    bool tail_ok = false;
    {
      const double r = rmax;
      if (k2 != 0.0) {
        const double low = r * (std::fabs(k2) * r * r * r * r - std::fabs(k1) * r * r - 1.0) - 4.0 * T * r * r;
        const double slope_ok = 5.0 * std::fabs(k2) * r * r * r * r >= 2.0 * (3.0 * std::fabs(k1) * r * r + 1.0 + 8.0 * T * r);
        tail_ok = slope_ok && low > dmax;
      } else if (k1 != 0.0) {
        const double low = r * (std::fabs(k1) * r * r - 1.0) - 4.0 * T * r * r;
        const double slope_ok = 3.0 * std::fabs(k1) * r * r >= 2.0 * (1.0 + 8.0 * T * r);
        tail_ok = slope_ok && low > dmax;
      }
    }
    if (!tail_ok) return false;
    double b = rmax;
    rc = 0.0;
    while (b > 1e-4) {
      const double a = b / 1.0005;
      const double poly_a = std::fabs(1.0 + k1 * a * a + k2 * a * a * a * a);
      const double lip = std::fabs(2.0 * k1 * b) + std::fabs(4.0 * k2 * b * b * b);
      const double low = a * std::max(0.0, poly_a - lip * (b - a)) - 4.0 * T * b * b;
      if (low <= dmax) {
        rc = b;
        break;
      }
      b = a;
    }
    if (rc >= rmax) return false;
    if (rc == 0.0) rc = 1e-4;
  } else if (cam.dist_type == AMB_DIST_EQUIDISTANT) {
    // |D| = |theta * (1 + k1 th^2 + k2 th^4 + k3 th^6 + k4 th^8)|, theta = atan(r) in [0, pi/2)
    const double half_pi = 1.5707963267948966;
    const double step = 1e-4;
    double b = half_pi + step;
    double thc = -1.0;
    bool first = true;
    while (b > 0.0) {
      const double a = std::max(0.0, b - step);
      const double a2 = a * a;
      const double poly_a = std::fabs(1.0 + k[0] * a2 + k[1] * a2 * a2 + k[2] * a2 * a2 * a2 + k[3] * a2 * a2 * a2 * a2);
      const double lip = std::fabs(2 * k[0] * b) + std::fabs(4 * k[1] * b * b * b) + std::fabs(6 * k[2] * std::pow(b, 5)) +
                         std::fabs(8 * k[3] * std::pow(b, 7));
      const double low = a * std::max(0.0, poly_a - lip * (b - a));
      if (low <= dmax) {
        if (first) return false;
        thc = b;
        break;
      }
      first = false;
      b = a;
    }
    if (thc < 0.0) thc = step;
    if (thc >= half_pi - 1e-3) return false;
    rc = std::tan(thc);
  } else if (cam.dist_type == AMB_DIST_FOV) {
    // |D| = atan(2 tan(w/2) r) / w (or r itself for w^2 < 1e-5): increasing in r, bounded by (pi/2)/w.  A ray lands inside
    // the raster only if |D| <= dmax, i.e. r <= tan(w dmax) / (2 tan(w/2)) — when w dmax reaches pi/2 every ray might.
    const double w = k[0];
    if (w * w < 1e-5) {
      rc = dmax;
    } else {
      const double wd = std::fabs(w) * dmax;
      if (!(wd < 1.5707963267948966 - 1e-3)) return false;
      rc = std::tan(wd) / (2.0 * std::fabs(std::tan(w / 2.)));
      if (!(rc > 0.0) || !std::isfinite(rc)) return false;
    }
  } else {
    return false;
  }
  rc *= (1.0 + 1e-6);
  const double h = std::sqrt(1.0 + rc * rc);
  *cos_c = 1.0 / h;
  *sin_c = rc / h;
  *tan_c = rc;
  return true;
}

// Conservative bounds on the UNDISTORTED normalised keypoint (u, v) of any visible ray.  Inside the view cone
// (r <= rc) the rad-tan model moves a point by at most  E = |k1| rc^3 + |k2| rc^5 + 4 (|p1|+|p2|) rc^2, and a
// visible ray's distorted keypoint lies in the raster, so  u in [-cu/fu - E, (W-cu)/fu + E]  (same for v).
bool compute_view_rect(const amb_camera& cam, double rc, double* u_lo, double* u_hi, double* v_lo, double* v_hi) {
  double E = 0.0;
  if (cam.dist_type == AMB_DIST_RADTAN) {
    const double* k = cam.dist;
    E = std::fabs(k[0]) * rc * rc * rc + std::fabs(k[1]) * std::pow(rc, 5) +
        4.0 * (std::fabs(k[2]) + std::fabs(k[3])) * rc * rc;
  } else if (cam.dist_type != AMB_DIST_NONE) {
    return false;  // equidistant: the cone is the natural bound
  }
  E = E * (1.0 + 1e-9) + 1e-12;
  *u_lo = -cam.cu / cam.fu - E;
  *u_hi = (cam.width - cam.cu) / cam.fu + E;
  *v_lo = -cam.cv / cam.fv - E;
  *v_hi = (cam.height - cam.cv) / cam.fv + E;
  return cam.fu > 0.0 && cam.fv > 0.0;
}

// Bound J on how far a keypoint moves, in units of f, per unit of camera-coordinate error times z_c, for rays with
// undistorted normalised radius <= r: |du|, |dv| <= delta (1 + r) / z_c, and a row of the distortion's Jacobian sums to
// at most the bound below (rad-tan: differentiate u (1 + k1 rho^2 + k2 rho^4) + 2 p1 u v + p2 (rho^2 + 2 u^2); equidistant:
// D = u theta_d(theta) / r with theta = atan(r), |theta_d / r| <= P and |d theta_d / d theta| <= Q; FOV: D = u s(r)
// with |s| <= 2 tan(w/2) / w and |r s'| <= 2 |s|).
double distortion_slope(const amb_camera& cam, double r) {
  const double* k = cam.dist;
  double J = 1.0;
  if (cam.dist_type == AMB_DIST_RADTAN) {
    J = 1.0 + 5.0 * std::fabs(k[0]) * r * r + 9.0 * std::fabs(k[1]) * r * r * r * r +
        8.0 * (std::fabs(k[2]) + std::fabs(k[3])) * r;
  } else if (cam.dist_type == AMB_DIST_EQUIDISTANT) {
    const double t2 = std::atan(r) * std::atan(r);
    const double P = 1.0 + std::fabs(k[0]) * t2 + std::fabs(k[1]) * t2 * t2 + std::fabs(k[2]) * t2 * t2 * t2 +
                     std::fabs(k[3]) * t2 * t2 * t2 * t2;
    const double Q = 1.0 + 3.0 * std::fabs(k[0]) * t2 + 5.0 * std::fabs(k[1]) * t2 * t2 +
                     7.0 * std::fabs(k[2]) * t2 * t2 * t2 + 9.0 * std::fabs(k[3]) * t2 * t2 * t2 * t2;
    J = 3.0 * P + 2.0 * Q;
  } else if (cam.dist_type == AMB_DIST_FOV) {
    const double w = k[0];
    const double s = (w * w < 1e-5) ? 1.0 : std::fabs(2.0 * std::tan(w / 2.) / w);
    J = 4.0 * std::max(1.0, s);
  }
  return J * (1.0 + r);
}

// T_G_C = T_G_B * T_C_B^-1 (ortho-backward-grid.cc:230-233), then the per-frame constants of
// X_c = T_G_C^-1 . X = R_C_G X - R_C_G t_G_C, and the guards' scale with the inputs' magnitude (a->delta_coef, a->t_max).
void frame_tables(const amb_camera& cam, const double* T_G_B, size_t n, FrameConst* fcs, double* cull, double* exact,
                  OrthoArgs* a) {
  const Quat q_C_B = {cam.q_C_B[0], cam.q_C_B[1], cam.q_C_B[2], cam.q_C_B[3]};
  const Quat q_B_C = {q_C_B.w, -q_C_B.x, -q_C_B.y, -q_C_B.z};
  const V3 t_C_B = {cam.t_C_B[0], cam.t_C_B[1], cam.t_C_B[2]};
  const V3 r_tmp = qrot(q_B_C, t_C_B);
  const V3 t_B_C = {-r_tmp.x, -r_tmp.y, -r_tmp.z};
  double q_norm2 = 1.0, t_max = 0.0;
  for (size_t f = 0; f < n; ++f) {
    const double* p = T_G_B + 7 * f;
    const Quat q_G_B = {p[3], p[4], p[5], p[6]};
    const V3 t_G_B = {p[0], p[1], p[2]};
    const Quat q = qmul(q_G_B, q_B_C);
    const V3 rt = qrot(q_G_B, t_B_C);
    const V3 t = {t_G_B.x + rt.x, t_G_B.y + rt.y, t_G_B.z + rt.z};
    // rows of R_C_G = images of the map axes under q^-1, i.e. columns of R_G_C transposed
    const Quat qi = {q.w, -q.x, -q.y, -q.z};
    const V3 ex = qrot(qi, V3{1, 0, 0}), ey = qrot(qi, V3{0, 1, 0}), ez = qrot(qi, V3{0, 0, 1});
    FrameConst& fc = fcs[f];
    fc.m[0] = ex.x; fc.m[1] = ey.x; fc.m[2] = ez.x;
    fc.m[3] = ex.y; fc.m[4] = ey.y; fc.m[5] = ez.y;
    fc.m[6] = ex.z; fc.m[7] = ey.z; fc.m[8] = ez.z;
    const V3 ti = qrot(qi, t);
    fc.t[0] = -ti.x; fc.t[1] = -ti.y; fc.t[2] = -ti.z;
    double* cf = &cull[12 * f];
    cf[0] = t.x; cf[1] = t.y; cf[2] = t.z;
    for (int k = 0; k < 9; ++k) cf[3 + k] = fc.m[k];
    // inverse(T_G_C) as minkindr forms it: (q^-1, -(q^-1).rotate(t)) — for the exact re-evaluation path
    double* ef = &exact[8 * f];
    ef[0] = qi.w; ef[1] = qi.x; ef[2] = qi.y; ef[3] = qi.z;
    ef[4] = -ti.x; ef[5] = -ti.y; ef[6] = -ti.z; ef[7] = 0.0;
    q_norm2 = std::max(q_norm2, q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    t_max = std::max({t_max, std::fabs(t.x), std::fabs(t.y), std::fabs(t.z), std::fabs(ti.x), std::fabs(ti.y),
                      std::fabs(ti.z)});
  }
  a->delta_coef = kDeltaUlps * std::ldexp(1.0, -53) * q_norm2;
  a->t_max = t_max;
}

// The camera's cull bounds (the fields of `a` from `cone` to the dominance cull's) and px_coef.  `cull`: not brute force.
void camera_bounds(const amb_camera& cam, bool cull, bool dominance, OrthoArgs* a) {
  double cc = 0.0, sc = 1.0, tc = 0.0;
  a->cone = compute_view_cone(cam, &cc, &sc, &tc) ? 1 : 0;
  a->cos_c = cc;
  a->sin_c = sc;
  a->rect = 0;
  if (a->cone && compute_view_rect(cam, tc, &a->u_lo, &a->u_hi, &a->v_lo, &a->v_hi)) {
    a->rect = 1;
    a->nu_lo = std::sqrt(1.0 + a->u_lo * a->u_lo);
    a->nu_hi = std::sqrt(1.0 + a->u_hi * a->u_hi);
    a->nv_lo = std::sqrt(1.0 + a->v_lo * a->v_lo);
    a->nv_hi = std::sqrt(1.0 + a->v_hi * a->v_hi);
  }
  // without a view cone the normalised radius of an imaged ray is bounded by nothing better than the cone scan's limit
  a->px_coef = std::max(std::fabs(cam.fu), std::fabs(cam.fv)) * distortion_slope(cam, a->cone ? tc : 1.0e3);

  // Dominance cull: needs an INNER bound, a set of rays that are certainly imaged inside the raster.  r_in: normalised
  // distance from the principal point to the nearest raster edge.
  if (!(dominance && cull && a->cone && cam.fu > 0.0 && cam.fv > 0.0)) return;
  const double r_in = std::min(std::min(cam.cu, cam.width - cam.cu) / cam.fu,
                               std::min(cam.cv, cam.height - cam.cv) / cam.fv) * (1.0 - 1e-9);
  bool inner = false;
  double th = 0.0;  // inner view cone (equidistant, FOV): every ray with angle-to-axis below th is imaged
  if (a->rect) {
    // Pinhole / rad-tan: the INNER rectangle, the raster's normalised extent shrunk by the same distortion bound E the
    // outer rectangle was grown by: a ray with an undistorted keypoint inside it is imaged inside the raster.
    const double E_u = a->u_hi - (cam.width - cam.cu) / cam.fu;   // what compute_view_rect added
    const double E_v = a->v_hi - (cam.height - cam.cv) / cam.fv;
    const double E = std::max(E_u, E_v) * (1.0 + 1e-9) + 1e-9;
    a->ui_lo = -cam.cu / cam.fu + E;
    a->ui_hi = (cam.width - cam.cu) / cam.fu - E;
    a->vi_lo = -cam.cv / cam.fv + E;
    a->vi_hi = (cam.height - cam.cv) / cam.fv - E;
    a->nui_lo = std::sqrt(1.0 + a->ui_lo * a->ui_lo);
    a->nui_hi = std::sqrt(1.0 + a->ui_hi * a->ui_hi);
    a->nvi_lo = std::sqrt(1.0 + a->vi_lo * a->vi_lo);
    a->nvi_hi = std::sqrt(1.0 + a->vi_hi * a->vi_hi);
    inner = a->ui_lo < a->ui_hi && a->vi_lo < a->vi_hi;
  } else if (cam.dist_type == AMB_DIST_EQUIDISTANT) {
    // Equidistant: the keypoint's distance from the principal point (normalised) is |theta * poly(theta^2)| whatever
    // the azimuth, so every ray with theta <= th is imaged if that radius stays below r_in on [0, th].  Scan outwards
    // with a Lipschitz bound on the radius; stop at the first step that might leave the inscribed circle.
    const double* k = cam.dist;
    const double step = 1e-4;
    while (th < 1.5) {
      const double b = th + step, b2 = b * b;
      const double lip = 1.0 + 3.0 * std::fabs(k[0]) * b2 + 5.0 * std::fabs(k[1]) * b2 * b2 +
                         7.0 * std::fabs(k[2]) * b2 * b2 * b2 + 9.0 * std::fabs(k[3]) * b2 * b2 * b2 * b2;  // >= |dr/dtheta|
      const double t2 = th * th;
      const double r_th = std::fabs(th * (1.0 + k[0] * t2 + k[1] * t2 * t2 + k[2] * t2 * t2 * t2 + k[3] * t2 * t2 * t2 * t2));
      if (r_th + lip * step >= r_in) break;
      th = b;
    }
    inner = th > 1e-3;
  } else if (cam.dist_type == AMB_DIST_FOV) {
    // FOV: radius atan(2 tan(w/2) tan(theta)) / w, increasing — every ray with that radius below r_in is imaged:
    // tan(th) = tan(w r_in) / (2 tan(w/2))
    const double w = std::fabs(cam.dist[0]);
    double tan_in = r_in;
    if (w * w >= 1e-5) tan_in = (w * r_in < 1.5) ? std::tan(w * r_in) / (2.0 * std::fabs(std::tan(w / 2.))) : -1.0;
    th = tan_in > 0.0 ? std::atan(tan_in) * (1.0 - 1e-9) : 0.0;
    inner = th > 1e-3;
  }
  if (inner) {
    const double margin = 1e-4;  // rad; the float32 rounding of an angle <= pi/2 is < 1.2e-7
    a->dominance = 1;
    a->dom_cos_in = std::cos(th);
    a->dom_cos_margin = std::cos(margin);
    a->dom_sin_margin = std::sin(margin);
  }
}

// One launch per chunk of frames, whose constants take their turn in c_frames (ConstantGuard).
int launch_chunks(amb_ctx* ctx, OrthoArgs& a, const FrameConst* fcs, size_t n, bool select_only, bool fresh) {
  cudaStream_t s = ctx->stream;
  const int tiles_i = (a.rows + OTI - 1) / OTI, tiles_j = (a.cols_slab + OTJ - 1) / OTJ;
  ctx->ortho_launches = 0;
  for (size_t f0 = 0; f0 < n; f0 += kMaxFramesPerLaunch) {  // ascending chunks keep the frame order
    const size_t nf = std::min<size_t>(kMaxFramesPerLaunch, n - f0);
    std::lock_guard<std::mutex> lock(g_constant_guard.mu);  // held until this chunk's kernel has been enqueued
    cudaEvent_t& guard_event = g_constant_guard.last_use[ctx->device & 63];
    if (!guard_event) AMB_CUDA(ctx, cudaEventCreateWithFlags(&guard_event, cudaEventDisableTiming));
    AMB_CUDA(ctx, cudaStreamWaitEvent(s, guard_event, 0));
    AMB_CUDA(ctx, cudaMemcpyToSymbolAsync(c_frames, fcs + f0, nf * sizeof(FrameConst), 0,
                                          cudaMemcpyHostToDevice, s));
    a.n_frames = static_cast<int>(nf);
    a.frame_base = static_cast<int>(f0);
    a.images = ctx->frame_table.as<const uint8_t*>() + f0;
    a.cull_data = ctx->frame_cull.as<double>() + 12 * f0;
    a.exact_data = ctx->frame_cull.as<double>() + 12 * n + 8 * f0;
    if (select_only) {
      launch_ortho_kernel<true, false>(a, tiles_i * tiles_j, s);
    } else if (fresh) {
      launch_ortho_kernel<false, true>(a, tiles_i * tiles_j, s);
    } else {
      launch_ortho_kernel<false, false>(a, tiles_i * tiles_j, s);
    }
    ctx->ortho_launches += 1;
    AMB_CUDA(ctx, cudaEventRecord(guard_event, s));
  }
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

// The two texel sources of host frames fill the FrameRect table and ctx->ortho_h2d_bytes from the per-frame bounding
// boxes of the winners' pixels.  Rasters: the sub-rectangle of each frame's box is copied to the device.
int rect_source(amb_ctx* ctx, const OrthoCall& c, const int* bbox, FrameRect* rects) {
  // bytes per row and rows of frame f's box; the rows of its device copy are 256-byte aligned
  auto row_bytes = [&](size_t f) { return static_cast<size_t>(bbox[4 * f + 2] - bbox[4 * f + 0] + 1) * c.channels; };
  auto rows = [&](size_t f) { return static_cast<size_t>(bbox[4 * f + 3] - bbox[4 * f + 1] + 1); };
  auto pitch = [&](size_t f) { return (row_bytes(f) + 255) & ~static_cast<size_t>(255); };
  size_t total = 0;
  for (size_t f = 0; f < c.n; ++f)
    if (bbox[4 * f + 2] >= 0) total += pitch(f) * rows(f);  // xmax < 0: no cell takes its pixel from this frame
  AMB_CUDA(ctx, ctx->frames.reserve(total + 256));
  uint8_t* dst = ctx->frames.as<uint8_t>();
  std::vector<StagedRect> copies;
  copies.reserve(c.n);
  for (size_t f = 0; f < c.n; ++f) {
    rects[f] = FrameRect{nullptr, 0, 0, 0, 0};
    if (bbox[4 * f + 2] < 0) continue;
    const int x0 = bbox[4 * f + 0], y0 = bbox[4 * f + 1];
    rects[f] = FrameRect{dst, x0, y0, static_cast<int>(pitch(f)), 0};
    const uint8_t* src = c.images[f] + static_cast<size_t>(y0) * c.row_step + static_cast<size_t>(x0) * c.channels;
    // (frames in pageable memory — cv::Mat storage — are packed into pinned slots by the worker pool: host_staging.cu)
    copies.push_back(StagedRect{dst, pitch(f), src, c.row_step, row_bytes(f), rows(f)});
    ctx->ortho_h2d_bytes += static_cast<int64_t>(row_bytes(f) * rows(f));
    dst += pitch(f) * rows(f);
  }
  return staged_h2d_rects(ctx, copies.data(), copies.size(), ctx->stream);
}

// JPEG files: the rows of each frame's box, every column, decoded on the device (frames without a winner are neither
// copied nor decoded)
int jpeg_source(amb_ctx* ctx, const OrthoCall& c, const int* bbox, FrameRect* rects) {
  const size_t n = c.n;
  std::vector<int32_t> row0(n), row1(n);
  std::vector<unsigned char*> ptr(n);
  std::vector<int> pitch(n);
  for (size_t f = 0; f < n; ++f) {
    row0[f] = bbox[4 * f + 2] < 0 ? 0 : bbox[4 * f + 1];
    row1[f] = bbox[4 * f + 2] < 0 ? 0 : bbox[4 * f + 3] + 1;
  }
  const JpegBands bands{c.files, c.file_bytes, c.headers, row0.data(), row1.data(), n, c.channels};
  const int st = jpeg_decode_bands(ctx, bands, ptr.data(), pitch.data());
  if (st != AMB_OK) return st;
  for (size_t f = 0; f < n; ++f) {
    rects[f] = FrameRect{ptr[f], 0, row0[f], pitch[f], 0};
    if (ptr[f]) ctx->ortho_h2d_bytes += static_cast<int64_t>(c.file_bytes[f]);
  }
  return AMB_OK;
}

// ---- host frames: bounding boxes back, texels up from their source, texel gather ----
int host_frames_texels(amb_ctx* ctx, const OrthoCall& c, const OrthoArgs& a, HostStage& stage, int* bbox) {
  cudaStream_t s = ctx->stream;
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_ORTHO_SELECT_END], s));
  ctx->ortho_h2d_bytes = 0;
  int* mapped = nullptr;
  AMB_CUDA(ctx, cudaHostGetDevicePointer(reinterpret_cast<void**>(&mapped), bbox, 0));
  copy_to_mapped_kernel<<<8, 256, 0, s>>>(ctx->ortho_bbox.as<int>(), mapped, static_cast<int>(4 * c.n));
  AMB_CUDA(ctx, cudaStreamSynchronize(s));
  FrameRect* rects = stage.take<FrameRect>(c.n);
  AMB_CUDA(ctx, ctx->frame_rects.reserve(c.n * sizeof(FrameRect)));
  const int st = c.frames == OrthoCall::JPEG ? jpeg_source(ctx, c, bbox, rects) : rect_source(ctx, c, bbox, rects);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaMemcpyAsync(ctx->frame_rects.ptr, rects, c.n * sizeof(FrameRect), cudaMemcpyHostToDevice, s));
  AMB_CUDA(ctx, cudaEventRecord(ctx->events[EV_ORTHO_COPY_END], s));
  ortho_texel_kernel<<<ctx->num_sms * 8, 256, 0, s>>>(a.pix, a.observation_index, ctx->frame_rects.as<FrameRect>(),
                                                    a.out_layer, ctx->slab_cells(), c.channels, a.colored);
  ctx->ortho_launches += 1;
  AMB_CUDA(ctx, cudaGetLastError());
  return AMB_OK;
}

}  // namespace

// Device frames: one fused kernel per chunk of frames.
// Host and JPEG frames: phase A selects the winners without touching any pixel, the host reads back the per-frame
// bounding boxes of the winners' pixels, only those parts of the frames reach the device, phase B fetches the texels.
// Same results, a fraction of the PCIe traffic: a cell is seen by ~8 frames but takes its pixel from one.
int ortho_run(amb_ctx* ctx, const OrthoCall& c) {
  const amb_camera& cam = *c.camera;
  const size_t n = c.n;
  const bool select_only = c.frames != OrthoCall::DEVICE;
  const int out_layer = c.colored_ortho ? AMB_LAYER_COLORED_ORTHO : AMB_LAYER_ORTHO;
  const int need[4] = {AMB_LAYER_ELEVATION, AMB_LAYER_ELEVATION_ANGLE, AMB_LAYER_OBSERVATION_INDEX, out_layer};
  // One fused launch (frames on the device, at most one chunk of them) writes every cell of the slab: when all three
  // layers it writes are fresh, it stores their initial values itself instead of reading them after a fill.  Otherwise
  // (host frames, several chunks, a layer an earlier call wrote) the layers are filled first and read as before.
  bool fresh = !select_only && n <= static_cast<size_t>(kMaxFramesPerLaunch);
  for (int k = 1; k < 4; ++k) fresh = fresh && layer_is_fresh(ctx, need[k]);
  for (int l : need) {
    bool overwritten = false;
    const int st = fresh && l != AMB_LAYER_ELEVATION ? ensure_layer_overwrite(ctx, l, &overwritten) : ensure_layer(ctx, l);
    if (st != AMB_OK) return st;
    if (l != AMB_LAYER_ELEVATION) wait_layer_copy(ctx, l);  // written here; elevation is only read
  }
  const amb_geometry& g = ctx->geom;
  cudaStream_t s = ctx->stream;

  // per-call tables live in pinned staging (see HostStage); the previous call's copies must have left it
  const int turn = static_cast<int>(ctx->stage_turn++ & 1u);
  HostStage& stage = ctx->stages[turn];
  cudaEvent_t& stage_event = ctx->stage_events[turn];
  if (!stage_event) AMB_CUDA(ctx, cudaEventCreateWithFlags(&stage_event, cudaEventDisableTiming));
  AMB_CUDA(ctx, cudaEventSynchronize(stage_event));   // the call before the previous one: long finished in practice
  AMB_CUDA(ctx, stage.reserve(n * (sizeof(FrameConst) + 20 * sizeof(double) + 8 * sizeof(int) +
                                        sizeof(FrameRect) + sizeof(uint8_t*)) + 1024));
  stage.used = 0;
  FrameConst* fcs = stage.take<FrameConst>(n);
  double* cull = stage.take<double>(12 * n);
  double* exact = stage.take<double>(8 * n);
  OrthoArgs a;
  std::memset(&a, 0, sizeof(a));
  frame_tables(cam, c.T_G_B, n, fcs, cull, exact, &a);

  AMB_CUDA(ctx, ctx->frame_table.reserve(n * sizeof(uint8_t*)));
  {
    const int cst = ensure_counters(ctx);  // born zeroed; the CHECK(alpha > 0) flag is sticky until reported
    if (cst != AMB_OK) return cst;
  }
  unsigned int* counters = ctx->counters.as<unsigned int>();
  if (!select_only) {
    const uint8_t** table = stage.take<const uint8_t*>(n);
    for (size_t f = 0; f < n; ++f) table[f] = c.images[f];
    AMB_CUDA(ctx, cudaMemcpyAsync(ctx->frame_table.ptr, table, n * sizeof(uint8_t*), cudaMemcpyHostToDevice, s));
  }
  AMB_CUDA(ctx, ctx->frame_cull.reserve(20 * n * sizeof(double)));   // [12 n cull | 8 n exact]
  AMB_CUDA(ctx, cudaMemcpyAsync(ctx->frame_cull.ptr, cull, 12 * n * sizeof(double), cudaMemcpyHostToDevice, s));
  AMB_CUDA(ctx, cudaMemcpyAsync(ctx->frame_cull.as<double>() + 12 * n, exact, 8 * n * sizeof(double),
                                cudaMemcpyHostToDevice, s));

  a.elevation = ctx->layers[AMB_LAYER_ELEVATION];
  a.elevation_angle = ctx->layers[AMB_LAYER_ELEVATION_ANGLE];
  a.observation_index = ctx->layers[AMB_LAYER_OBSERVATION_INDEX];
  a.out_layer = ctx->layers[out_layer];
  a.error_flag = counters + CTR_ORTHO_CHECK;
  int* bbox_back = nullptr;  // pinned and mapped: the select kernel's bounding boxes come back here
  if (select_only) {
    const size_t cells = ctx->slab_cells();
    AMB_CUDA(ctx, ctx->ortho_pix.reserve(cells * sizeof(unsigned int)));
    AMB_CUDA(ctx, ctx->ortho_bbox.reserve(n * 4 * sizeof(int)));
    AMB_CUDA(ctx, cudaMemsetAsync(ctx->ortho_pix.ptr, 0xff, cells * sizeof(unsigned int), s));
    int* bbox = stage.take<int>(4 * n);
    bbox_back = stage.take<int>(4 * n);
    for (size_t f = 0; f < n; ++f) {
      bbox[4 * f + 0] = bbox[4 * f + 1] = 0x7fffffff;
      bbox[4 * f + 2] = bbox[4 * f + 3] = -1;
    }
    AMB_CUDA(ctx, cudaMemcpyAsync(ctx->ortho_bbox.ptr, bbox, 4 * n * sizeof(int), cudaMemcpyHostToDevice, s));
    a.pix = ctx->ortho_pix.as<unsigned int>();
    a.bbox = ctx->ortho_bbox.as<int>();
  }
  a.row_step = c.row_step;
  a.rows = g.rows;
  a.cols_slab = ctx->col_end - ctx->col_begin;
  a.col_begin = ctx->col_begin;
  a.width = cam.width;
  a.height = cam.height;
  a.channels = c.channels;
  a.colored = c.colored_ortho ? 1 : 0;
  a.dist_type = cam.dist_type;
  a.base_x = g.pos_x + (0.5 * g.length_x - 0.5 * g.resolution);
  a.base_y = g.pos_y + (0.5 * g.length_y - 0.5 * g.resolution);
  a.res = g.resolution;
  a.fu = cam.fu; a.fv = cam.fv; a.cu = cam.cu; a.cv = cam.cv;
  a.d0 = cam.dist[0]; a.d1 = cam.dist[1]; a.d2 = cam.dist[2]; a.d3 = cam.dist[3];
  if (cam.dist_type == AMB_DIST_FOV) a.d1 = std::tan(cam.dist[0] / 2.);  // FOV: the kernels take tan(w/2) from here
  a.do_cull = ctx->ortho_brute_force ? 0 : 1;
  camera_bounds(cam, a.do_cull != 0, ctx->ortho_dominance, &a);

  int st = launch_chunks(ctx, a, fcs, n, select_only, fresh);
  // elevation_angle and observation_index are final here: start streaming them to their host mirrors
  if (st == AMB_OK) st = mirror_layer(ctx, AMB_LAYER_ELEVATION_ANGLE);
  if (st == AMB_OK) st = mirror_layer(ctx, AMB_LAYER_OBSERVATION_INDEX);
  if (st == AMB_OK && select_only) st = host_frames_texels(ctx, c, a, stage, bbox_back);
  if (st != AMB_OK) return st;
  AMB_CUDA(ctx, cudaEventRecord(stage_event, s));
  return mirror_layer(ctx, out_layer);
}

}  // namespace amb
