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

// Build a (up to) 3-D bf16/fp32 tiled tensor map. dims/strides innermost first; strides in BYTES for dims 1..
// (dim 0 is contiguous); swizzle_bytes is 128, 64 or 0 (none). Returns ALM_OK or an error code.
int make_tensor_map(CUtensorMap* out, const void* base, int elem_bytes, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes);

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

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Device-wide barrier: monotonic arrival counter, red.release / ld.acquire at gpu scope (the CTA's own writes are ordered
// before the release by the __syncthreads).  A bounded spin (about 2 s) turns a lost CTA into an error flag instead of a
// hung GPU.
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned& epoch, int* err) {
  __syncthreads();
  if (threadIdx.x == 0) {
    epoch += gridDim.x;
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
    const long long t0 = clock64();
    while (ld_acquire(counter) < epoch) {
      if (clock64() - t0 > 4000000000LL) {
        *err = 1;
        break;
      }
    }
  }
  __syncthreads();
}

// ---- dropout mask ------------------------------------------------------------------------------
// Every dropout decision of the library is keep(seed, site, row, col): a pure function of its arguments, so the
// backward regenerates the forward's mask instead of storing it.  Coordinates: elementwise sites on an [M, C]
// activation use (token b*n + i, channel); attention probabilities use ((b*H + h) * n_q_pad + i, key j), with
// n_q_pad = n_q rounded up to 128 (the LSE row stride), so that 16-row groups never straddle two heads.
//
// Generator: Philox4x32-10 (Salmon et al., SC'11; the generator of torch's CUDA RNG), key = the 64-bit seed.
// One draw gives four 32-bit words = eight 16-bit uniforms.  They decide the 8 elements
//     rows {i0, i0+1, i0+8, i0+9} x cols {j0, j0+8},   i0 % 16 in {0, 2, 4, 6},  j0 % 16 < 8,
// counter = (row / 16, col / 16, site, 8 * ((row % 8) / 2) + col % 8); row i0 + r1 + 8 r8 takes word r1 + 2 r8
// and col j0 + 8 c8 takes its low (c8 = 0) or high half.  This group lies inside what one thread of the attention
// backward holds of dP^T / P^T (two key rows j0, j0 + 8 by query columns {2c, 2c+1} mod 8), so there every draw
// is used in full.  The attention forward holds rows {r, r+8} by the same columns: a lane pair (r, r^1) splits
// the draws and swaps halves with one shuffle per word.  Keep iff the 16-bit uniform < thr, thr = round(65536 (1-p)),
// so the keep probability is exact to 2^-17.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

struct DropoutArgs {
  uint64_t seed;
  uint32_t site;
  uint32_t thr;   // keep iff the 16-bit uniform < thr (65536: keep all)
  float scale;    // 1 / (1 - p)
};

// the draw of the 8-element group that holds (row, col)
__device__ __forceinline__ uint4 dropout_draw(const DropoutArgs& d, uint32_t row, uint32_t col) {
  const uint4 ctr = make_uint4(row >> 4, col >> 4, d.site, ((row & 7u) >> 1) * 8u + (col & 7u));
  return philox4x32_10(ctr, (uint32_t)d.seed, (uint32_t)(d.seed >> 32));
}

// the word of a draw that holds `row`'s two elements
__device__ __forceinline__ uint32_t dropout_word(const uint4& draw, uint32_t row) {
  return (row & 1u) ? ((row & 8u) ? draw.w : draw.y) : ((row & 8u) ? draw.z : draw.x);
}

// the decision for (row, col) inside its group's draw (only the word of `row` is read)
__device__ __forceinline__ bool dropout_pick(const DropoutArgs& d, const uint4& draw, uint32_t row, uint32_t col) {
  const uint32_t w = dropout_word(draw, row);
  const uint32_t u = (col & 8u) ? (w >> 16) : (w & 0xFFFFu);
  return u < d.thr;
}

__device__ __forceinline__ bool dropout_keep(const DropoutArgs& d, uint32_t row, uint32_t col) {
  return dropout_pick(d, dropout_draw(d, row, col), row, col);
}

inline DropoutArgs make_dropout_args(float p, uint64_t seed, uint32_t site) {
  DropoutArgs a;
  a.seed = seed;
  a.site = site;
  const double keep = 1.0 - (double)p;
  a.thr = (uint32_t)(keep * 65536.0 + 0.5);
  a.scale = (float)(1.0 / keep);
  return a;
}

}  // namespace alm
