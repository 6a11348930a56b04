// approx_probe.cu — device sweeps of the approximations in aerial_mapper_b200/csrc/approx_math.h, for
// tests/test_gpu_approx_math.py.  It includes that header and nothing else of the product, so it measures exactly the
// code the kernels inline.  Built by __graft_entry__.build() into tests/cuda/libamb_approx_probe.so with the product's
// compiler flags; test code only, the product library does not link it.
//
// Every sweep runs on the device and returns a ProbeResult: the largest error, the number of inputs whose result is not
// the correctly rounded one, and how many inputs break the sweep's claim, with the smallest of them.
#include <cuda_runtime.h>

#include "approx_math.h"

struct ProbeResult {
  double max_err;                 // largest error, in the unit the sweep documents
  double aux;                     // a second, sweep-specific maximum (documented per sweep)
  unsigned long long n_not_rn;    // inputs whose result differs from the correctly rounded one
  unsigned long long n_bad;       // inputs that break the claim
  unsigned long long first_bad;   // the smallest such input (its bit pattern); ~0 if none
};

namespace {

constexpr double kU = 0x1p-24;   // unit roundoff of float32
constexpr int kThreads = 256;

struct Acc {
  double max_err = 0.0, aux = 0.0;
  unsigned long long n_not_rn = 0, n_bad = 0, first_bad = ~0ull;
  __device__ void add(double err, double a, bool not_rn, bool bad, unsigned long long input) {
    max_err = fmax(max_err, err);   // (fmax drops a NaN operand: a NaN error is counted through `bad`)
    aux = fmax(aux, a);
    n_not_rn += not_rn ? 1 : 0;
    if (bad) {
      ++n_bad;
      first_bad = min(first_bad, input);
    }
  }
  // the warp's totals to `out` (every lane calls it); non-negative doubles order like their bit patterns
  __device__ void flush(ProbeResult* out) {
    for (int o = 16; o > 0; o >>= 1) {
      max_err = fmax(max_err, __shfl_xor_sync(0xffffffffu, max_err, o));
      aux = fmax(aux, __shfl_xor_sync(0xffffffffu, aux, o));
      n_not_rn += __shfl_xor_sync(0xffffffffu, n_not_rn, o);
      n_bad += __shfl_xor_sync(0xffffffffu, n_bad, o);
      first_bad = min(first_bad, __shfl_xor_sync(0xffffffffu, first_bad, o));
    }
    if ((threadIdx.x & 31) == 0) {
      atomicMax(reinterpret_cast<unsigned long long*>(&out->max_err), __double_as_longlong(max_err));
      atomicMax(reinterpret_cast<unsigned long long*>(&out->aux), __double_as_longlong(aux));
      if (n_not_rn) atomicAdd(&out->n_not_rn, n_not_rn);
      if (n_bad) atomicAdd(&out->n_bad, n_bad);
      if (first_bad != ~0ull) atomicMin(&out->first_bad, first_bad);
    }
  }
};

// rcp_f32 on the floats with bit patterns [lo, hi].  Claim: |rcp_f32(x) x - 1| <= 2^-23.  max_err: that relative
// error in units of u = 2^-24 (exact: the product of two floats is exact in double).  Reference: __frcp_rn.
__global__ void rcp_f32_sweep(unsigned int lo, unsigned long long n, ProbeResult* out) {
  Acc acc;
  for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
       k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const unsigned int b = lo + static_cast<unsigned int>(k);
    const float x = __uint_as_float(b);
    const float r = amb::rcp_f32(x);
    const double rel = fabs(fma(static_cast<double>(r), static_cast<double>(x), -1.0));
    acc.add(rel / kU, 0.0, __float_as_uint(r) != __float_as_uint(__frcp_rn(x)), !(rel <= 2.0 * kU), b);
  }
  acc.flush(out);
}

// rsqrt_f32 on the floats with bit patterns [lo, hi].  max_err: |rsqrt_f32(x) sqrt(x) - 1| in units of u; not correctly
// rounded: differs from 1 / sqrt(x) evaluated in double and rounded to float.  Claim (the per-neighbour height bound):
// rsqrt_f32(x) (1 + kRsqrtSlackUlps u) >= sqrt(rcp_f32(x)), decided exactly by the sign of one fma; aux: the slack
// that takes, (sqrt(rcp_f32(x)) / rsqrt_f32(x) - 1) / u.
__global__ void rsqrt_f32_sweep(unsigned int lo, unsigned long long n, ProbeResult* out) {
  const float slack = 1.0f + amb::kRsqrtSlackUlps * static_cast<float>(kU);   // as the kernel evaluates it
  Acc acc;
  for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < n;
       k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const unsigned int b = lo + static_cast<unsigned int>(k);
    const float x = __uint_as_float(b);
    const float rs = amb::rsqrt_f32(x);
    const double s = sqrt(static_cast<double>(x));
    const double err = fabs(fma(static_cast<double>(rs), s, -1.0)) / kU;
    const bool not_rn = __float_as_uint(rs) != __float_as_uint(__double2float_rn(1.0 / s));
    const double w = static_cast<double>(amb::rcp_f32(x));
    const double a = static_cast<double>(rs) * static_cast<double>(slack);   // exact: 24 x 25 significant bits
    const bool ok = fma(a, a, -w) >= 0.0;                                     // the sign of a^2 - w, exactly
    acc.add(err, (sqrt(w) / static_cast<double>(rs) - 1.0) / kU, not_rn, !ok, b);
  }
  acc.flush(out);
}

__device__ __forceinline__ unsigned int hash32(unsigned int h) {
  h ^= h >> 16;
  h *= 0x7feb352du;
  h ^= h >> 15;
  h *= 0x846ca68bu;
  h ^= h >> 16;
  return h;
}

// fast_rcp on the doubles with high words [lo, hi], each with the low words 0, 0xffffffff and one hashed word (the
// MUFU.RCP64H seed reads the high word only).  max_err: distance to __drcp_rn in ulps (bit patterns of two positive
// doubles).  Claim: at most 1 ulp.
__global__ void fast_rcp_sweep(unsigned int lo, unsigned long long n, ProbeResult* out) {
  Acc acc;
  for (unsigned long long k = blockIdx.x * static_cast<unsigned long long>(blockDim.x) + threadIdx.x; k < 3 * n;
       k += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
    const unsigned int hi = lo + static_cast<unsigned int>(k / 3);
    const int variant = static_cast<int>(k % 3);
    const unsigned int low = variant == 0 ? 0u : (variant == 1 ? 0xffffffffu : hash32(hi));
    const unsigned long long bits = (static_cast<unsigned long long>(hi) << 32) | low;
    const double x = __longlong_as_double(static_cast<long long>(bits));
    const long long r = __double_as_longlong(amb::fast_rcp(x));
    const long long ref = __double_as_longlong(__drcp_rn(x));
    const unsigned long long d = static_cast<unsigned long long>(r > ref ? r - ref : ref - r);
    acc.add(static_cast<double>(d), 0.0, d != 0, d > 1, bits);
  }
  acc.flush(out);
}

__global__ void values_kernel(int which, const double* x, double* y, int n) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float xf = static_cast<float>(x[k]);
  y[k] = which == 0 ? amb::fast_rcp(x[k]) : (which == 1 ? amb::rcp_f32(xf) : amb::rsqrt_f32(xf));
}

typedef void (*SweepKernel)(unsigned int, unsigned long long, ProbeResult*);

int run_sweep(SweepKernel kernel, unsigned int lo, unsigned int hi, ProbeResult* host, float* ms) {
  ProbeResult init = {0.0, 0.0, 0, 0, ~0ull};
  ProbeResult* d = nullptr;
  cudaEvent_t e0 = nullptr, e1 = nullptr;
  cudaError_t st = cudaMalloc(&d, sizeof(ProbeResult));
  if (st == cudaSuccess) st = cudaMemcpy(d, &init, sizeof(init), cudaMemcpyHostToDevice);
  if (st == cudaSuccess) st = cudaEventCreate(&e0);
  if (st == cudaSuccess) st = cudaEventCreate(&e1);
  int sms = 0;
  if (st == cudaSuccess) st = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  if (st == cudaSuccess) {
    cudaEventRecord(e0);
    kernel<<<sms * 8, kThreads>>>(lo, static_cast<unsigned long long>(hi - lo) + 1, d);
    cudaEventRecord(e1);
    st = cudaGetLastError();
  }
  if (st == cudaSuccess) st = cudaEventSynchronize(e1);
  if (st == cudaSuccess) st = cudaEventElapsedTime(ms, e0, e1);
  if (st == cudaSuccess) st = cudaMemcpy(host, d, sizeof(ProbeResult), cudaMemcpyDeviceToHost);
  if (e0) cudaEventDestroy(e0);
  if (e1) cudaEventDestroy(e1);
  if (d) cudaFree(d);
  return static_cast<int>(st);
}

}  // namespace

// Each returns a cudaError_t (0 on success); [lo, hi] are inclusive bit-pattern bounds (float bits, or the high words
// of doubles for fast_rcp); *ms is the sweep kernel's time from CUDA events.
extern "C" int amb_probe_rcp_f32(unsigned int lo, unsigned int hi, ProbeResult* out, float* ms) {
  return run_sweep(rcp_f32_sweep, lo, hi, out, ms);
}
extern "C" int amb_probe_rsqrt_f32(unsigned int lo, unsigned int hi, ProbeResult* out, float* ms) {
  return run_sweep(rsqrt_f32_sweep, lo, hi, out, ms);
}
extern "C" int amb_probe_fast_rcp(unsigned int lo, unsigned int hi, ProbeResult* out, float* ms) {
  return run_sweep(fast_rcp_sweep, lo, hi, out, ms);
}

// y[k] = fast_rcp(x[k]) (which == 0), rcp_f32((float)x[k]) (1) or rsqrt_f32((float)x[k]) (2), on the device.
extern "C" int amb_probe_values(int which, const double* x, double* y, int n) {
  double* d = nullptr;
  cudaError_t st = cudaMalloc(&d, 2 * sizeof(double) * (n > 0 ? n : 1));
  if (st == cudaSuccess) st = cudaMemcpy(d, x, sizeof(double) * n, cudaMemcpyHostToDevice);
  if (st == cudaSuccess) {
    values_kernel<<<(n + 255) / 256, 256>>>(which, d, d + n, n);
    st = cudaGetLastError();
  }
  if (st == cudaSuccess) st = cudaMemcpy(y, d + n, sizeof(double) * n, cudaMemcpyDeviceToHost);
  if (d) cudaFree(d);
  return static_cast<int>(st);
}

// The constants of approx_math.h whose claims the sweeps check.
extern "C" void amb_probe_constants(float* rsqrt_slack_ulps, float* height_bound_factor) {
  *rsqrt_slack_ulps = amb::kRsqrtSlackUlps;
  *height_bound_factor = amb::kHeightBoundFactor;
}
