// stereo_kernels.cu — "next" row N3 (SURVEY.md §8f): disparity map -> world points, the step right before
// dsm::Dsm::process in the incremental pipeline (stereo.cpp:149-193).
//
// Replaces the per-pixel loop of stereo::Densifier::computePointCloud (reference
// aerial_mapper_dense_pcl/src/densifier.cpp:25-108): for every pixel (v, u) in raster order with
// disparity > kMaxInvalidDisparity:  w = (1/baseline) * d;  p = ((u - cx)/w, (fx/fy*v - cy*fx/fy)/w, fx/w);
// P = R_G_C * p + t_G_C1; kept unless (float)P.z is infinite; the kept points (double) and their gray values are
// appended IN RASTER ORDER to point_cloud_eigen / point_cloud_intensities — the vectors Dsm::process and
// OrthoFromPcl::process consume.  Block matching itself (OpenCV StereoBM/SGBM) stays out of scope.
//
// Three kernels: per-block valid count -> exclusive scan of the block counts -> ordered write (stable compaction:
// output order == raster order, so the DSM's canonical "original index" order is the reference's).
// Every arithmetic step uses un-contracted IEEE operations in the reference's order: results are bit-identical.
#include <cmath>

#include "amb_context.h"

namespace amb {
namespace {

constexpr int kRpThreads = 256;

struct ReprojectParams {
  const float* disparity;   // H x W, row stride `disp_stride` floats
  const uint8_t* image;     // H x W gray, row stride `img_stride` bytes
  int width, height;
  size_t disp_stride, img_stride;
  float max_invalid_disparity;
  double q03, q11, q13, q23, q32;  // Q = [1 0 0 -cx; 0 fx/fy 0 -cy*fx/fy; 0 0 0 fx; 0 0 1/baseline 0]
  double r[9], t[3];               // R_G_C (row-major), t_G_C1
};

__device__ __forceinline__ bool reproject_pixel(const ReprojectParams& p, size_t pix, double* X, double* Y, double* Z,
                                                int* gray) {
  const int v = static_cast<int>(pix / p.width), u = static_cast<int>(pix - static_cast<size_t>(v) * p.width);
  const float d = p.disparity[static_cast<size_t>(v) * p.disp_stride + u];
  if (!(d > p.max_invalid_disparity)) return false;  // densifier.cpp:61
  const double w = __dmul_rn(p.q32, static_cast<double>(d));                                  // :63
  const double x1 = __ddiv_rn(__dadd_rn(static_cast<double>(u), p.q03), w);                   // :69-70
  const double y1 = __ddiv_rn(__dadd_rn(__dmul_rn(p.q11, static_cast<double>(v)), p.q13), w);
  const double z1 = __ddiv_rn(p.q23, w);
  // R_G_C * point_r1 + t_G_C1 (:73-74): (r0*x + r1*y) + r2*z, then + t
  *X = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p.r[0], x1), __dmul_rn(p.r[1], y1)), __dmul_rn(p.r[2], z1)), p.t[0]);
  *Y = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p.r[3], x1), __dmul_rn(p.r[4], y1)), __dmul_rn(p.r[5], z1)), p.t[1]);
  *Z = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(p.r[6], x1), __dmul_rn(p.r[7], y1)), __dmul_rn(p.r[8], z1)), p.t[2]);
  if (isinf(__double2float_rn(*Z))) return false;  // `if (!std::isinf(z))` on the float copy (:75-78)
  *gray = p.image[static_cast<size_t>(v) * p.img_stride + u];
  return true;
}

__global__ void __launch_bounds__(kRpThreads) reproject_count_kernel(const ReprojectParams p, size_t n_pixels,
                                                                     unsigned int* __restrict__ block_counts) {
  const size_t pix = static_cast<size_t>(blockIdx.x) * kRpThreads + threadIdx.x;
  double X, Y, Z;
  int gray;
  const bool valid = pix < n_pixels && reproject_pixel(p, pix, &X, &Y, &Z, &gray);
  const int c = __syncthreads_count(valid ? 1 : 0);
  if (threadIdx.x == 0) block_counts[blockIdx.x] = static_cast<unsigned int>(c);
}

// exclusive scan of block_counts in place (one block); *total = sum
__global__ void __launch_bounds__(1024) reproject_scan_kernel(unsigned int* __restrict__ counts, int n,
                                                              unsigned long long* __restrict__ total) {
  __shared__ unsigned int warp_sums[32];
  __shared__ unsigned int carry_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int k = base + threadIdx.x;
    const unsigned int v = k < n ? counts[k] : 0u;
    unsigned int inc = v;
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
      const unsigned int w = warp_sums[lane];
      unsigned int winc = w;
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned int t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
      }
      warp_sums[lane] = winc - w;
    }
    __syncthreads();
    const unsigned int carry = carry_s;
    const unsigned int ex = carry + warp_sums[warp] + inc - v;
    if (k < n) counts[k] = ex;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = ex + v;  // last thread holds the running total of this chunk
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry_s;
}

__global__ void __launch_bounds__(kRpThreads) reproject_write_kernel(const ReprojectParams p, size_t n_pixels,
                                                                     const unsigned int* __restrict__ block_offsets,
                                                                     double* __restrict__ out_xyz,
                                                                     int* __restrict__ out_intensity,
                                                                     size_t capacity) {
  __shared__ unsigned int warp_counts[kRpThreads / 32];
  const size_t pix = static_cast<size_t>(blockIdx.x) * kRpThreads + threadIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double X = 0, Y = 0, Z = 0;
  int gray = 0;
  const bool valid = pix < n_pixels && reproject_pixel(p, pix, &X, &Y, &Z, &gray);
  const unsigned int m = __ballot_sync(0xffffffffu, valid);
  if (lane == 0) warp_counts[warp] = __popc(m);
  __syncthreads();
  unsigned int before = block_offsets[blockIdx.x];
  for (int w = 0; w < warp; ++w) before += warp_counts[w];
  if (valid) {
    const size_t pos = static_cast<size_t>(before) + __popc(m & ((1u << lane) - 1u));  // raster order preserved
    if (pos < capacity) {
      out_xyz[3 * pos + 0] = X;
      out_xyz[3 * pos + 1] = Y;
      out_xyz[3 * pos + 2] = Z;
      out_intensity[pos] = gray;
    }
  }
}

}  // namespace
}  // namespace amb

using namespace amb;

extern "C" int amb_stereo_reproject_device(int device, void* stream, const float* d_disparity, size_t disparity_stride,
                                           const uint8_t* d_image_left, size_t image_stride, int32_t width,
                                           int32_t height, const double* K, double baseline, const double* R_G_C,
                                           const double* t_G_C1, float max_invalid_disparity, double* d_out_xyz,
                                           int32_t* d_out_intensity, size_t capacity, uint32_t* d_block_scratch,
                                           unsigned long long* d_count) {
  if (!d_disparity || !d_image_left || !K || !R_G_C || !t_G_C1 || !d_out_xyz || !d_out_intensity || !d_block_scratch ||
      !d_count || width <= 0 || height <= 0 || disparity_stride < static_cast<size_t>(width) ||
      image_stride < static_cast<size_t>(width))
    return AMB_ERR_INVALID_ARGUMENT;
  if (baseline == 0.0) return AMB_ERR_CHECK_FAILED;  // CHECK_NE(baseline, 0.0), densifier.cpp:39
  if (cudaSetDevice(device) != cudaSuccess) {
    cudaGetLastError();
    return AMB_ERR_NO_DEVICE;
  }
  ReprojectParams p;
  p.disparity = d_disparity;
  p.image = d_image_left;
  p.width = width;
  p.height = height;
  p.disp_stride = disparity_stride;
  p.img_stride = image_stride;
  p.max_invalid_disparity = max_invalid_disparity;
  const double fx = K[0], fy = K[1], cx = K[2], cy = K[3];
  p.q03 = -cx;                // densifier.cpp:45-47
  p.q11 = fx / fy;
  p.q13 = -cy * (fx / fy);
  p.q23 = fx;
  p.q32 = 1.0 / baseline;
  for (int k = 0; k < 9; ++k) p.r[k] = R_G_C[k];
  for (int k = 0; k < 3; ++k) p.t[k] = t_G_C1[k];
  const size_t n_pixels = static_cast<size_t>(width) * height;
  const int blocks = static_cast<int>((n_pixels + kRpThreads - 1) / kRpThreads);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  reproject_count_kernel<<<blocks, kRpThreads, 0, s>>>(p, n_pixels, d_block_scratch);
  reproject_scan_kernel<<<1, 1024, 0, s>>>(d_block_scratch, blocks, d_count);
  reproject_write_kernel<<<blocks, kRpThreads, 0, s>>>(p, n_pixels, d_block_scratch, d_out_xyz, d_out_intensity, capacity);
  if (cudaGetLastError() != cudaSuccess) return AMB_ERR_CUDA;
  return AMB_OK;
}

extern "C" int amb_stereo_reproject(int device, const float* disparity, size_t disparity_stride,
                                    const uint8_t* image_left, size_t image_stride, int32_t width, int32_t height,
                                    const double* K, double baseline, const double* R_G_C, const double* t_G_C1,
                                    float max_invalid_disparity, double* out_xyz, int32_t* out_intensity,
                                    size_t capacity, size_t* out_count) {
  if (!disparity || !image_left || !out_xyz || !out_intensity || !out_count || width <= 0 || height <= 0 ||
      disparity_stride < static_cast<size_t>(width) || image_stride < static_cast<size_t>(width))
    return AMB_ERR_INVALID_ARGUMENT;
  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0) {
    cudaGetLastError();
    return AMB_ERR_NO_DEVICE;
  }
  if (cudaSetDevice(device) != cudaSuccess) {
    cudaGetLastError();
    return AMB_ERR_NO_DEVICE;
  }
  const size_t n_pixels = static_cast<size_t>(width) * height;
  const size_t blocks = (n_pixels + kRpThreads - 1) / kRpThreads;
  float* d_disp = nullptr;
  uint8_t* d_img = nullptr;
  double* d_xyz = nullptr;
  int32_t* d_int = nullptr;
  uint32_t* d_scratch = nullptr;
  unsigned long long* d_count = nullptr;
  int st = AMB_OK;
  cudaStream_t s = nullptr;
  auto ok = [&](cudaError_t e) {
    if (e != cudaSuccess && st == AMB_OK) {
      cudaGetLastError();
      st = AMB_ERR_CUDA;
    }
    return e == cudaSuccess;
  };
  ok(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  ok(cudaMalloc(&d_disp, n_pixels * sizeof(float)));
  ok(cudaMalloc(&d_img, n_pixels));
  ok(cudaMalloc(&d_xyz, std::max<size_t>(capacity, 1) * 3 * sizeof(double)));
  ok(cudaMalloc(&d_int, std::max<size_t>(capacity, 1) * sizeof(int32_t)));
  ok(cudaMalloc(&d_scratch, blocks * sizeof(uint32_t)));
  ok(cudaMalloc(&d_count, sizeof(unsigned long long)));
  unsigned long long count = 0;
  if (st == AMB_OK) {
    ok(cudaMemcpy2DAsync(d_disp, width * sizeof(float), disparity, disparity_stride * sizeof(float),
                         width * sizeof(float), height, cudaMemcpyHostToDevice, s));
    ok(cudaMemcpy2DAsync(d_img, width, image_left, image_stride, width, height, cudaMemcpyHostToDevice, s));
  }
  if (st == AMB_OK)
    st = amb_stereo_reproject_device(device, s, d_disp, width, d_img, width, width, height, K, baseline, R_G_C, t_G_C1,
                                     max_invalid_disparity, d_xyz, d_int, capacity, d_scratch, d_count);
  if (st == AMB_OK) {
    ok(cudaMemcpyAsync(&count, d_count, sizeof(count), cudaMemcpyDeviceToHost, s));
    ok(cudaStreamSynchronize(s));
  }
  if (st == AMB_OK) {
    *out_count = static_cast<size_t>(count);
    const size_t n_out = std::min<size_t>(count, capacity);
    if (n_out) {
      ok(cudaMemcpyAsync(out_xyz, d_xyz, n_out * 3 * sizeof(double), cudaMemcpyDeviceToHost, s));
      ok(cudaMemcpyAsync(out_intensity, d_int, n_out * sizeof(int32_t), cudaMemcpyDeviceToHost, s));
      ok(cudaStreamSynchronize(s));
    }
  }
  cudaFree(d_disp);
  cudaFree(d_img);
  cudaFree(d_xyz);
  cudaFree(d_int);
  cudaFree(d_scratch);
  cudaFree(d_count);
  if (s) cudaStreamDestroy(s);
  return st;
}
