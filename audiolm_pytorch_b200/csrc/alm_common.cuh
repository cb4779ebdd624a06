// Host-side plumbing shared by every translation unit of libalm_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/alm_b200.h"

namespace alm {

// Every kernel launch of this library goes through ALM_LAUNCHED() so the host can report
// "gpu_launches" per step (bench.py) without a profiler.
extern unsigned long long g_launch_count;
#define ALM_LAUNCHED(n) (::alm::g_launch_count += (n))

#define ALM_CUDA_OK(expr)                                                                         \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      fprintf(stderr, "[alm] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__, \
              cudaGetErrorString(_e));                                                            \
      return ALM_ERR_CUDA;                                                                        \
    }                                                                                             \
  } while (0)

#define ALM_REQUIRE(cond, code)                                                            \
  do {                                                                                     \
    if (!(cond)) {                                                                         \
      fprintf(stderr, "[alm] argument check failed (%s) at %s:%d\n", #cond, __FILE__, __LINE__); \
      return (code);                                                                       \
    }                                                                                      \
  } while (0)

#define ALM_CHECK_LAUNCH() ALM_CUDA_OK(cudaGetLastError())

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

// Build a (up to) 3-D bf16/fp32 tiled tensor map with 128-B swizzle. dims/strides innermost first;
// strides in BYTES for dims 1.. (dim 0 is contiguous). Returns ALM_OK or an error code.
int make_tensor_map(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128);

template <typename T>
__host__ __device__ constexpr T ceil_div(T a, T b) {
  return (a + b - 1) / b;
}

// ---- device helpers ------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float bf16_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }

// Phi(x) = 0.5 (1 + erf(x / sqrt2)) and x * phi(x) for the erf GELU (audiolm_pytorch.py:246-249: F.gelu default)
// with ONE exponential: erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, two orders below the bf16 outputs'
// rounding), whose exp(-(x/sqrt2)^2) is also the Gaussian density.  ~14 instructions vs ~35 for erff + __expf.
__device__ __forceinline__ void gelu_parts(float x, float& cdf, float& xpdf) {
  const float ax = fabsf(x) * 0.7071067811865476f;
  const float t = __frcp_rn(fmaf(0.3275911f, ax, 1.f));
  float e;
  const float arg = -0.7213475204444817f * x * x;  // -x^2/2 * log2(e)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(arg));
  float p = fmaf(t, 1.061405429f, -1.453152027f);
  p = fmaf(t, p, 1.421413741f);
  p = fmaf(t, p, -0.284496736f);
  p = fmaf(t, p, 0.254829592f);
  const float half_tail = 0.5f * p * t * e;          // 0.5 * (1 - erf(|x|/sqrt2))
  cdf = x >= 0.f ? 1.f - half_tail : half_tail;
  xpdf = 0.3989422804014327f * x * e;
}

}  // namespace alm
