// approx_math.h — the MUFU-seeded reciprocals of the DSM, OrthoFromPcl and orthomosaic kernels, and the error each of
// their callers relies on.  Self-contained (tests/cuda/approx_probe.cu includes this header alone and sweeps the
// domains below on the device).  Under AMB_CUDA_EMU (tests/emu: the kernel sources compiled as plain C++) there is no
// MUFU: the seeds are IEEE divisions and square roots.
#ifndef AMB_APPROX_MATH_H_
#define AMB_APPROX_MATH_H_

#include <cuda_runtime.h>

#include <cmath>

namespace amb {

// Reciprocal of a double in [2^-1022, 2^1022), within 1 ulp of 1/x: MUFU.RCP64H seed (rcp.approx.ftz.f64, relative
// error <= 2^-20 from the operand's high word alone) + one cubic correction step.  Replaces the two IEEE divisions per
// neighbour of the reference (heights/d2 and 1/d2) by one reciprocal and one FMA; the IDW height changes by O(1e-16)
// relative, far inside the float32 layer's rounding.
// Outside that domain the seed is flushed (.ftz) and the result is wrong:
//   x                     fast_rcp(x)            1.0 / x
//   [2^-1074, 2^-1022)    NaN                    inf below 2^-1024, else finite above 2^1022
//   2^-1022               within 1 ulp           2^1022
//   (2^1022, DBL_MAX]     up to 0 (flushed)      subnormal
// A subnormal x never gives a value below 2^1022: the FP64 DSM gather relies on that to hand a cell with such a
// distance to dsm_cell_kernel, which divides as the reference does.  A guard for the other inputs would cost the FP64
// gather a fifth of its time.
__device__ __forceinline__ double fast_rcp(double x) {
  double r;
#ifdef AMB_CUDA_EMU  // no MUFU: an exact seed, same correction
  r = 1.0 / x;
#else
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
#endif
  const double e = fma(-x, r, 1.0);  // |e| <= 2^-20
  const double t = fma(e, e, e);     // e + e^2: r*(1 + e + e^2) leaves a relative error e^3 <= 2^-60
  return fma(r, t, r);
}

// 1 / x for a positive normal float, |rcp_f32(x) x - 1| <= 2^-23 (within 1 ulp of 1/x): the bound the FP32 gather's
// weights assume (DESIGN.md §4.1).  A subnormal x is flushed to zero and gives +inf.
__device__ __forceinline__ float rcp_f32(float x) {
#ifdef AMB_CUDA_EMU
  return 1.0f / x;
#else
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#endif
}

// 1 / sqrt(x) for a positive normal float, to ~2 ulp (the FP32 height bound's per-neighbour form only).  A subnormal x
// is flushed to zero and gives +inf.
__device__ __forceinline__ float rsqrt_f32(float x) {
#ifdef AMB_CUDA_EMU
  return 1.0f / std::sqrt(x);
#else
  float r;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
#endif
}

// rsqrt_f32(d2) (1 + kRsqrtSlackUlps u) >= sqrt(rcp_f32(d2)), u = 2^-24, for every positive normal float d2: the
// height bound's per-neighbour form takes sqrt(w) of a computed weight w = rcp_f32(d2) from one rsqrt; the slack is
// sqrt(w) <= (1 + 5u) rsqrt_f32(d2) and 3u for the rounding of t = Delta sqrt(w) (1 + 3u) + u.
constexpr float kRsqrtSlackUlps = 8.0f;

// Factor of the FP32 height bound E (DESIGN.md §4.1): covers E's second-order terms and the rounding of its own
// evaluation, three rcp_f32 (each within 2^-23 relative, above) among a dozen float32 operations.
constexpr float kHeightBoundFactor = 1.1f;

}  // namespace amb
#endif  // AMB_APPROX_MATH_H_
