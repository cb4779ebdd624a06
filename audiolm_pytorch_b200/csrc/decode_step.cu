// One-token decode step of the whole hyper-connection transformer stack as ONE persistent kernel (config C5:
// AudioLM.generate with use_kv_cache, audiolm_pytorch.py:1406-1511, 1608-1740, 1896-2039; the stack itself is
// audiolm_pytorch.py:446-560 with Attention :293-406 and FeedForward :246-260).
//
// The graph engine of decode.py used to replay ~11 small kernels per layer (hyper-connection pre, q / kv GEMVs, value
// residual, cache append, decode attention (+combine), out GEMV, hyper-connection pre, W1 GEMV, GEGLU+LN, W2 GEMV):
// ~70 dependent launches per token, each 3-5 us of launch + drain latency around a few hundred nanoseconds of work.
// Here one cooperative grid (one CTA per SM, 512 threads) walks the whole stack and only meets at a device-wide barrier
// where a matrix-vector product needs every CTA's output columns:
//
//   per layer   A  [every CTA, redundantly: depth(prev) + width + pre-LN of the attention branch, state in SHARED memory]
//                  q / kv columns of this CTA                                                        -> barrier
//               B  flash-decoding slices of the cache (b x splits CTAs; CTA 0 appends the new k / v)  -> barrier
//               C  [every CTA: merge the slices]  out-projection columns                              -> barrier
//               D  [every CTA: depth + width + pre-LN of the feed-forward branch]  W1 columns         -> barrier
//               E  [every CTA: GEGLU + LayerNorm(inner)]  W2 columns                                  -> barrier
//   end            CTA 0: depth of the last branch + stream sum + final LayerNorm, len += 1
//
// The residual streams never leave shared memory (every CTA carries an identical bf16 copy, rounded exactly where the
// multi-kernel path rounds when it stores R_out) and the small vectors between phases go through L2 (ld.global.cg).
// The WEIGHTS are decoupled from that dependency chain: a CTA owns the same output columns of every layer, so as soon as
// it has used its rows of one projection it starts ONE bulk (TMA) copy of the same rows of the NEXT layer (the engine
// keeps the operands regrouped per CTA, so they are one contiguous block) into the same shared-memory slot (about 130 KB
// per SM per layer at d = 1024), completion counted on an mbarrier per slot.  The HBM
// stream of the 115 MB of weights therefore runs a full layer ahead of the arithmetic, and the matrix-vector phases read
// shared memory only.
//
// What is left is a chain of short latency-bound steps, so the code is written against round trips, not bandwidth:
// every global load of a phase is issued before its first use, the layer's pointer table sits in shared memory, block
// reductions need ONE __syncthreads (every warp finishes the cross-warp sum itself), the barrier is a red.release +
// ld.acquire pair, and the phases are __noinline__ so that the layer loop stays small for the instruction cache.
//
// Arithmetic follows the kernels this replaces step by step (hc2::pre_fwd_kernel, gemv_bf16_kernel,
// mqa_attn_decode_kernel, geglu_ln_fwd_kernel, hc_post_fwd_kernel): same bf16 rounding points, fp32 accumulation; the
// summation order inside dot products differs and 1/sqrt, 1/d use the fast units.  tests/test_decode_gpu.py compares
// the two paths.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace dstep {

constexpr int NT = 512, NW = NT / 32;
constexpr int MAXB = 4;            // rows (sequences) per step
constexpr int HS = 4, HT = 5;      // residual streams, streams + 1
constexpr int NPTR = 24;           // pointers per layer in the table
constexpr int DH = 64;             // head width
constexpr int PART_W = DH + 2;     // flash-decoding slice state: m, l, acc[64]
constexpr int MAX_SLOTS = 256;     // split-K partial sums per CTA
constexpr int MAX_SPLITS = 16;     // flash-decoding slices per sequence
constexpr int KEYS_PER_SPLIT = 32; // a slice is only opened per this many cached keys
constexpr int MAXP = 2;            // channel pairs per thread in the hyper-connection: d <= 2 * MAXP * NT
constexpr int MAXG = 2;            // 8-channel chunks per thread in GEGLU: pad8(inner) <= 8 * MAXG * NT
constexpr int MAXL = 64;

// layer table entries
enum {
  A_GAMMA = 0, A_DALPHA, A_DBETA, A_SALPHA, A_SBETA, A_ASCALE, A_BSCALE, A_LN,
  F_GAMMA, F_DALPHA, F_DBETA, F_SALPHA, F_SBETA, F_ASCALE, F_BSCALE, F_LN,
  P_WA, P_UNUSED, P_WC, P_WD, P_WE, P_LN2, P_KC, P_VC   // regrouped q|kv, out, W1, W2 operands (see Job)
};

struct Args {
  const unsigned long long* table;  // [L][NPTR] device pointers
  const float* x;            // [b, d] fp32: embedding of the token that was sampled last
  __nv_bfloat16* out;        // [b, d] final-normed stack output
  const float* final_gamma;
  int* len;                  // cache fill level (the new token goes to position *len; incremented at the end)
  const uint8_t* key_mask;   // [b, mask_bstride] 1 = attend, or null
  long long mask_bstride, cache_bstride;
  unsigned* counter;         // grid barrier (zeroed by the host before the launch)
  int* err;
  __nv_bfloat16* q;          // [b, H*64]
  __nv_bfloat16* kvn;        // [b, 128]
  float* part;               // [b, splits, H, PART_W]
  __nv_bfloat16* Y;          // [b, d] attention branch output
  __nv_bfloat16* Y2;         // [b, d] feed-forward branch output
  __nv_bfloat16* h;          // [b, 2*ip]
  int L, b, d, H, inner, ip, max_len, splits, value_residual;
  float scale_log2, inv_d, inv_inner;
  long long* trace;          // [L][16] clock64 stamps of CTA 0 (only with -DALM_DSTEP_TRACE)
  int st_off[4];             // byte offsets of the staged weight rows of phases A, C, D, E in shared memory, -1 = read from L2
};

// shared-memory views + per-launch values every phase needs
struct Ctx {
  __nv_bfloat16 *sR, *sBin, *sXn, *sGn, *sO, *sKV;
  float *sVfirst, *sBeta, *sRed32, *sRed2, *sStat, *sGacc, *sMerge;
  const unsigned long long* sTbl;  // [L][NPTR]
  uint64_t* sBar;                  // [4]
  __nv_bfloat16* slot[4];
  int pos, n_all, splits;
  bool has_new;
};

#ifdef ALM_DSTEP_TRACE
#define DSTEP_STAMP(i)                                                              \
  do {                                                                              \
    __syncthreads();                                                                \
    if (blockIdx.x == 0 && threadIdx.x == 0) a.trace[layer * 16 + (i)] = clock64(); \
  } while (0)
__device__ long long* g_sub_trace;   // sub-phase stamps of gemv_phase (CTA 0): rows 32.. of the trace area
__device__ int g_sub_count;
#define DSTEP_SUB()                                                     \
  do {                                                                  \
    __syncthreads();                                                    \
    if (blockIdx.x == 0 && threadIdx.x == 0) {                          \
      if (g_sub_count < 512) g_sub_trace[g_sub_count] = clock64();      \
      ++g_sub_count;                                                    \
    }                                                                   \
  } while (0)
#else
#define DSTEP_STAMP(i)
#define DSTEP_SUB()
#endif

// ---- small device helpers -----------------------------------------------------------------------------------------
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));  // same MUFU.TANH as hc2::tanh_fast
  return y;
}
__device__ __forceinline__ uint4 ldg_nc(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ float ld_bf16_cg(const __nv_bfloat16* p) {
  unsigned short u;
  asm volatile("ld.global.cg.u16 %0, [%1];" : "=h"(u) : "l"(p));
  return __uint_as_float((uint32_t)u << 16);
}
__device__ __forceinline__ float bf16r(float v) { return __bfloat162float(__float2bfloat16(v)); }
template <typename T>
__device__ __forceinline__ T* tptr(const unsigned long long* lp, int i) {
  return reinterpret_cast<T*>(lp[i]);
}

// 32 values per lane -> lane L holds the warp total of value L (31 shuffles instead of 160)
__device__ __forceinline__ float warp_reduce32(float (&v)[32], int lane) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = up ? v[i] : v[i + o];
      const float keep = up ? v[i + o] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return v[0];
}
// lane L of EVERY warp gets the block total of value L; one __syncthreads.  `red` ([NW][32]) may be reused after the
// next __syncthreads of the caller.
__device__ __forceinline__ float block_total32(float (&v)[32], float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  red[warp * 32 + lane] = warp_reduce32(v, lane);
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int w = 0; w < NW; ++w) s += red[w * 32 + lane];
  return s;
}
// block sums of two values, one __syncthreads; `red2` is a double buffer ([2][NW][2]) toggled by the caller's counter
__device__ __forceinline__ void block_sum2(float& a, float& b, float* red2, int& which) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float* buf = red2 + which * (NW * 2);
  which ^= 1;
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane == 0) *reinterpret_cast<float2*>(buf + warp * 2) = make_float2(a, b);
  __syncthreads();
  float2 p = lane < NW ? *reinterpret_cast<const float2*>(buf + lane * 2) : make_float2(0.f, 0.f);
#pragma unroll
  for (int o = NW / 2; o >= 1; o >>= 1) {
    p.x += __shfl_xor_sync(0xffffffffu, p.x, o);
    p.y += __shfl_xor_sync(0xffffffffu, p.y, o);
  }
  a = __shfl_sync(0xffffffffu, p.x, 0);
  b = __shfl_sync(0xffffffffu, p.y, 0);
}

// ---- hyper-connection depth(prev) + width + branch pre-LayerNorm for one row (hc2::pre_fwd_kernel) -----------------
// Rrow: this row's residual streams as stored by the previous width connection (bf16, [HS][d], shared memory);
// updated in place.  beta (shared, [HS]): in = beta of the previous branch, out = beta of this branch.
// A thread owns MAXP pairs of adjacent channels; every global load of the row is issued up front.
__device__ __noinline__ void hc_pre_row(const Ctx& cx, const bool first, const unsigned long long* lp, int base, int d,
                                        float inv_d, int r, const float* x, const __nv_bfloat16* Yprev, int& which) {
  const float* gamma_hc = tptr<const float>(lp, base + 0);
  const float* dyn_alpha = tptr<const float>(lp, base + 1);
  const float* dyn_beta = tptr<const float>(lp, base + 2);
  const float* ln_gamma = tptr<const float>(lp, base + 7);
  __nv_bfloat16* Rrow = cx.sR + (size_t)r * HS * d;
  __nv_bfloat16* bin = cx.sBin + (size_t)r * d;
  __nv_bfloat16* xn = cx.sXn + (size_t)r * d;
  float* beta = cx.sBeta + r * HS;
  const int lane = threadIdx.x & 31;
  {  // static_alpha[20] static_beta[4] alpha_scale beta_scale -> shared (read after the reduction's barrier)
    const int t = threadIdx.x;
    if (t < HS * HT) cx.sStat[t] = __ldg(tptr<const float>(lp, base + 3) + t);
    else if (t < HS * HT + HS) cx.sStat[t] = __ldg(tptr<const float>(lp, base + 4) + (t - HS * HT));
    else if (t == HS * HT + HS) cx.sStat[t] = __ldg(tptr<const float>(lp, base + 5));
    else if (t == HS * HT + HS + 1) cx.sStat[t] = __ldg(tptr<const float>(lp, base + 6));
  }
  const float sqrt_d = sqrtf((float)d);
  float bp[HS];
#pragma unroll
  for (int s = 0; s < HS; ++s) bp[s] = first ? 0.f : beta[s];

  float2 rr[HS][MAXP], lng[MAXP];
  float w[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) w[i] = 0.f;
#pragma unroll
  for (int k = 0; k < MAXP; ++k) {
    const int c = 2 * (threadIdx.x + k * NT);
    lng[k] = make_float2(0.f, 0.f);
#pragma unroll
    for (int s = 0; s < HS; ++s) rr[s][k] = make_float2(0.f, 0.f);
    if (c < d) {
      const float2 g = __ldg(reinterpret_cast<const float2*>(gamma_hc + c));
      const float2 bf = __ldg(reinterpret_cast<const float2*>(dyn_beta + c));
      lng[k] = __ldg(reinterpret_cast<const float2*>(ln_gamma + c));
      const float2* ap = reinterpret_cast<const float2*>(dyn_alpha + (size_t)c * HT);  // 2 channels x 5 maps, contiguous
      const float2 a0 = __ldg(ap), a1 = __ldg(ap + 1), a2 = __ldg(ap + 2), a3 = __ldg(ap + 3), a4 = __ldg(ap + 4);
      if (first) {
        const float2 xv = __ldg(reinterpret_cast<const float2*>(x + c));
#pragma unroll
        for (int s = 0; s < HS; ++s) rr[s][k] = xv;
      } else {
        const uint32_t yu = __ldcg(reinterpret_cast<const uint32_t*>(Yprev + c));
        const float y0 = bf16_lo(yu), y1 = bf16_hi(yu);
#pragma unroll
        for (int s = 0; s < HS; ++s) {
          const uint32_t ru = *reinterpret_cast<const uint32_t*>(Rrow + s * d + c);
          rr[s][k] = make_float2(fmaf(bp[s], y0, bf16_lo(ru)), fmaf(bp[s], y1, bf16_hi(ru)));
        }
      }
      const float g0 = (g.x + 1.f) * sqrt_d, g1 = (g.y + 1.f) * sqrt_d;
      const float av0[HT] = {a0.x, a0.y, a1.x, a1.y, a2.x};
      const float av1[HT] = {a2.y, a3.x, a3.y, a4.x, a4.y};
#pragma unroll
      for (int s = 0; s < HS; ++s) {
        const float n0 = rr[s][k].x * g0, n1 = rr[s][k].y * g1;
        w[HS * HT + HS + s] = fmaf(rr[s][k].x, rr[s][k].x, fmaf(rr[s][k].y, rr[s][k].y, w[HS * HT + HS + s]));
#pragma unroll
        for (int t = 0; t < HT; ++t) w[s * HT + t] = fmaf(n0, av0[t], fmaf(n1, av1[t], w[s * HT + t]));
        w[HS * HT + s] = fmaf(n0, bf.x, fmaf(n1, bf.y, w[HS * HT + s]));
      }
    }
  }
  // lane L < 24 finishes map entry L (its own tanh), then the 24 entries are broadcast inside the warp
  const float tot = block_total32(w, cx.sRed32);
  float alpha[HS][HT], beta_new[HS];
  {
    const int s_of = lane < HS * HT ? lane / HT : (lane < HS * HT + HS ? lane - HS * HT : 0);
    const float ss = __shfl_sync(0xffffffffu, tot, HS * HT + HS + s_of);
    const float inv = rsqrtf(fmaxf(ss, 1e-24f));
    const float z = tanh_approx(tot * inv);
    const float scale = lane < HS * HT ? cx.sStat[HS * HT + HS] : cx.sStat[HS * HT + HS + 1];
    const float mine = fmaf(z, scale, cx.sStat[lane < HS * HT + HS ? lane : 0]);
#pragma unroll
    for (int s = 0; s < HS; ++s) {
#pragma unroll
      for (int t = 0; t < HT; ++t) alpha[s][t] = __shfl_sync(0xffffffffu, mine, s * HT + t);
      beta_new[s] = __shfl_sync(0xffffffffu, mine, HS * HT + s);
    }
  }
  // mix the streams; the branch input stays in registers for the LayerNorm
  float2 bi[MAXP];
  float s1 = 0.f, s2 = 0.f, dummy = 0.f;
#pragma unroll
  for (int k = 0; k < MAXP; ++k) {
    const int c = 2 * (threadIdx.x + k * NT);
    bi[k] = make_float2(0.f, 0.f);
    if (c < d) {
      float2 acc = make_float2(0.f, 0.f);
#pragma unroll
      for (int s = 0; s < HS; ++s) {
        acc.x = fmaf(alpha[s][0], rr[s][k].x, acc.x);
        acc.y = fmaf(alpha[s][0], rr[s][k].y, acc.y);
      }
      bi[k] = acc;
      s1 += acc.x + acc.y;
      *reinterpret_cast<__nv_bfloat162*>(bin + c) = __floats2bfloat162_rn(acc.x, acc.y);
#pragma unroll
      for (int t = 1; t < HT; ++t) {
        float2 o = make_float2(0.f, 0.f);
#pragma unroll
        for (int s = 0; s < HS; ++s) {
          o.x = fmaf(alpha[s][t], rr[s][k].x, o.x);
          o.y = fmaf(alpha[s][t], rr[s][k].y, o.y);
        }
        *reinterpret_cast<__nv_bfloat162*>(Rrow + (t - 1) * d + c) = __floats2bfloat162_rn(o.x, o.y);
      }
    }
  }
  block_sum2(s1, dummy, cx.sRed2, which);
  const float mean = s1 * inv_d;
  // the variance in a second pass over the registers (as hc2::pre_fwd_kernel)
#pragma unroll
  for (int k = 0; k < MAXP; ++k)
    if (2 * (threadIdx.x + k * NT) < d)
      s2 = fmaf(bi[k].x - mean, bi[k].x - mean, fmaf(bi[k].y - mean, bi[k].y - mean, s2));
  dummy = 0.f;
  block_sum2(s2, dummy, cx.sRed2, which);
  const float rstd = rsqrtf(s2 * inv_d + 1e-5f);
#pragma unroll
  for (int k = 0; k < MAXP; ++k) {
    const int c = 2 * (threadIdx.x + k * NT);
    if (c < d)
      *reinterpret_cast<__nv_bfloat162*>(xn + c) =
          __floats2bfloat162_rn((bi[k].x - mean) * rstd * lng[k].x, (bi[k].y - mean) * rstd * lng[k].y);
  }
#pragma unroll
  for (int s = 0; s < HS; ++s)
    if (threadIdx.x == s) beta[s] = beta_new[s];
  __syncthreads();
}

// ---- matrix-vector products: this CTA's output columns (column n -> CTA n mod grid) ----------------------------------
// The decode engine keeps a copy of every projection with its rows regrouped per CTA: row (c * per_cta + lc) of the copy
// is row (c + lc * grid) of the operand (zero rows past N).  A CTA's rows of a phase are therefore ONE contiguous block:
// one bulk (TMA) copy per phase and layer, issued by one thread.
struct Job {
  const __nv_bfloat16* W;    // regrouped operand [grid * per_cta, K] bf16
  int N, K, per_cta;         // N = N0 + N1 true output columns, K % 8 == 0
  int N0;                    // columns [0, N0) use xs0 / out0, the rest xs1 / out1 (q | kv share one phase)
  const __nv_bfloat16* xs0;  // shared memory [b][K]
  const __nv_bfloat16* xs1;
  __nv_bfloat16* out0;       // global [b][ldo0]
  __nv_bfloat16* out1;
  int ldo0, ldo1;
};

__device__ __forceinline__ int cols_of_cta(int ntot) {
  return ((int)blockIdx.x < ntot) ? (ntot - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
}

// start the asynchronous copy of this CTA's rows of a phase into its shared-memory slot ([local column][K] bf16),
// completion counted in bytes on the slot's mbarrier
__device__ __forceinline__ void stage_rows(const Job& j, __nv_bfloat16* dst, uint64_t* bar) {
  const __nv_bfloat16* src = j.W + (size_t)blockIdx.x * j.per_cta * j.K;
  const uint32_t bytes = (uint32_t)j.per_cta * (uint32_t)j.K * 2u;
  if (dst != nullptr) {
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(bar, bytes);
      bulk_copy_g2s(dst, src, bytes, bar);
    }
  } else {  // not staged (shared memory is needed for more rows): at least pull the rows into L2 early
    for (uint32_t l = threadIdx.x; l * 128u < bytes; l += NT) prefetch_l2(reinterpret_cast<const char*>(src) + (size_t)l * 128);
  }
}

// this CTA's output columns: consume the phase's rows (waiting for their copy if staged), then start the copy of the
// NEXT layer's rows of the same phase into the slot that has just been read.
// The phase is instruction-bound, not bandwidth-bound (the rows are in shared memory), so the mapping minimises work per
// thread: a thread owns ONE 8-channel chunk of K for a subset of the columns - its x chunk is converted to fp32 once and
// stays in registers - and a column costs one 16-byte load, 8 conversions, 8 FMAs per row and a warp reduction.
// Threads are grouped per K (gsize = K/8 rounded up to warps); group g takes the local columns g, g + groups, ...
__device__ __forceinline__ void load_x8(const __nv_bfloat16* xs, int K, int tl, int b, float (&xf)[MAXB][8]) {
#pragma unroll
  for (int r = 0; r < MAXB; ++r) {
    if (r < b) {
      const uint4 u = *reinterpret_cast<const uint4*>(xs + (size_t)r * K + tl * 8);
      xf[r][0] = bf16_lo(u.x); xf[r][1] = bf16_hi(u.x); xf[r][2] = bf16_lo(u.y); xf[r][3] = bf16_hi(u.y);
      xf[r][4] = bf16_lo(u.z); xf[r][5] = bf16_hi(u.z); xf[r][6] = bf16_lo(u.w); xf[r][7] = bf16_hi(u.w);
    }
  }
}
__device__ __noinline__ void gemv_phase(const Job& jref, const Job& nxt, bool has_next, int b, float* gacc,
                                        __nv_bfloat16* staged, uint64_t* bar, uint32_t parity) {
  const Job j = jref;
  const bool STAGED = staged != nullptr;
  DSTEP_SUB();
  if (STAGED) mbar_wait(bar, parity);
  DSTEP_SUB();
  const int lane = threadIdx.x & 31;
  const int G = gridDim.x;
  const int ncol = cols_of_cta(j.N);
  const int K8 = j.K >> 3;                              // <= NT (checked by the host)
  const int gsize = max(32, (K8 + 31) & ~31);
  const int groups = NT / gsize, wpg = gsize >> 5;
  const int g = threadIdx.x / gsize, tl = threadIdx.x - g * gsize;
  const int wig = tl >> 5;                              // warp inside the group
  const bool active = g < groups && tl < K8;
  const __nv_bfloat16* wbase = STAGED ? staged : j.W + (size_t)blockIdx.x * j.per_cta * j.K;
  if (g < groups) {
    float xf[MAXB][8];
#pragma unroll
    for (int r = 0; r < MAXB; ++r)
#pragma unroll
      for (int e = 0; e < 8; ++e) xf[r][e] = 0.f;   // (threads past K keep zeros: they still take part in the shuffles)
    // NC columns per pass: their dot products are independent chains, and ONE butterfly (9 shuffles per row) reduces all
    // of them over the warp instead of 5 dependent shuffles per column
    constexpr int NC = 8;
    const int idx = ((lane >> 4) & 1) * 4 + ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);   // column of the pass this lane ends up with
    const int nq = cols_of_cta(j.N0);   // local columns [0, nq) belong to the first x vector, [nq, ncol) to the second
#pragma unroll 1
    for (int sweep = 0; sweep < 2; ++sweep) {
    const int lo = sweep == 0 ? 0 : nq, hi = sweep == 0 ? nq : ncol;
    if (lo >= hi) continue;
    if (active) load_x8(sweep == 0 ? j.xs0 : j.xs1, j.K, tl, b, xf);
    if ((hi - lo + groups - 1) / groups < 3) {   // one or two columns per group: plain per-column warp reduction
#pragma unroll 1
      for (int lc = lo + g; lc < hi; lc += groups) {
        float acc1[MAXB];
#pragma unroll
        for (int r = 0; r < MAXB; ++r) acc1[r] = 0.f;
        if (active) {
          const uint4* wp = reinterpret_cast<const uint4*>(wbase + (size_t)lc * j.K) + tl;
          const uint4 w = STAGED ? *wp : ldg_nc(wp);
          const float wf[8] = {bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y),
                               bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w)};
#pragma unroll
          for (int r = 0; r < MAXB; ++r) {
            if (r < b) {
              float s0 = wf[0] * xf[r][0], s1 = wf[1] * xf[r][1];
              s0 = fmaf(wf[2], xf[r][2], s0); s1 = fmaf(wf[3], xf[r][3], s1);
              s0 = fmaf(wf[4], xf[r][4], s0); s1 = fmaf(wf[5], xf[r][5], s1);
              s0 = fmaf(wf[6], xf[r][6], s0); s1 = fmaf(wf[7], xf[r][7], s1);
              acc1[r] = s0 + s1;
            }
          }
        }
#pragma unroll
        for (int r = 0; r < MAXB; ++r) {
          if (r < b) {
            const float v = warp_sum(acc1[r]);
            if (lane == 0) gacc[(lc * wpg + wig) * MAXB + r] = v;
          }
        }
      }
      continue;
    }
#pragma unroll 1
    for (int base = lo + g; base < hi; base += NC * groups) {
      float acc[MAXB][NC];
#pragma unroll
      for (int i = 0; i < NC; ++i) {
        const int lc = base + i * groups;
        uint4 w = make_uint4(0u, 0u, 0u, 0u);
        if (active && lc < hi) {
          const uint4* wp = reinterpret_cast<const uint4*>(wbase + (size_t)lc * j.K) + tl;
          w = STAGED ? *wp : ldg_nc(wp);
        }
        const float wf[8] = {bf16_lo(w.x), bf16_hi(w.x), bf16_lo(w.y), bf16_hi(w.y),
                             bf16_lo(w.z), bf16_hi(w.z), bf16_lo(w.w), bf16_hi(w.w)};
#pragma unroll
        for (int r = 0; r < MAXB; ++r) {
          acc[r][i] = 0.f;
          if (r < b) {
            float s0 = wf[0] * xf[r][0], s1 = wf[1] * xf[r][1];
            s0 = fmaf(wf[2], xf[r][2], s0); s1 = fmaf(wf[3], xf[r][3], s1);
            s0 = fmaf(wf[4], xf[r][4], s0); s1 = fmaf(wf[5], xf[r][5], s1);
            s0 = fmaf(wf[6], xf[r][6], s0); s1 = fmaf(wf[7], xf[r][7], s1);
            acc[r][i] = s0 + s1;
          }
        }
      }
#pragma unroll
      for (int r = 0; r < MAXB; ++r) {
        if (r < b) {
#pragma unroll
          for (int o = 16, n = NC / 2; o >= 4; o >>= 1, n >>= 1) {
            const bool up = (lane & o) != 0;
#pragma unroll
            for (int i = 0; i < n; ++i) {
              const float send = up ? acc[r][i] : acc[r][i + n];
              const float keep = up ? acc[r][i + n] : acc[r][i];
              acc[r][i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
            }
          }
          float v = acc[r][0];
          v += __shfl_xor_sync(0xffffffffu, v, 2);
          v += __shfl_xor_sync(0xffffffffu, v, 1);
          const int lc = base + idx * groups;
          if ((lane & 3) == 0 && lc < hi) gacc[(lc * wpg + wig) * MAXB + r] = v;
        }
      }
    }
    }
  }
  __syncthreads();   // every warp is done with the slot and with the x vectors; per-warp partial sums are in gacc
  DSTEP_SUB();
  if (has_next) stage_rows(nxt, staged, bar);
  for (int i = threadIdx.x; i < ncol * b; i += NT) {
    const int lc = i / b, r = i - lc * b;
    float v = 0.f;
    for (int p2 = 0; p2 < wpg; ++p2) v += gacc[(lc * wpg + p2) * MAXB + r];
    const int n = blockIdx.x + lc * G;
    if (n >= j.N0) j.out1[(size_t)r * j.ldo1 + (n - j.N0)] = __float2bfloat16(v);
    else j.out0[(size_t)r * j.ldo0 + n] = __float2bfloat16(v);
  }
  DSTEP_SUB();
}

// ---- phase B: new k / v (value residual), cache append by CTA 0, flash-decoding slices ----------------------------------
__device__ __noinline__ void attn_slices(const Args& a, const Ctx& cx, int layer, __nv_bfloat16* kc, __nv_bfloat16* vc) {
  const int b = a.b, H = a.H, HD = a.H * DH;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int pos = cx.pos, n_all = cx.n_all, splits = cx.splits;
  for (int i = threadIdx.x; i < b * 2 * DH; i += NT) {
    const int r = i / (2 * DH), c = i - r * 2 * DH;
    float v = ld_bf16_cg(a.kvn + (size_t)r * 2 * DH + c);
    if (c >= DH && a.value_residual) {
      if (layer == 0) cx.sVfirst[r * DH + (c - DH)] = v;
      else v = bf16r(0.5f * v + 0.5f * cx.sVfirst[r * DH + (c - DH)]);
    }
    const __nv_bfloat16 vb = __float2bfloat16(v);
    cx.sKV[i] = vb;
    if (blockIdx.x == 0 && cx.has_new) {
      if (c < DH) kc[(size_t)r * a.cache_bstride + (size_t)pos * DH + c] = vb;
      else vc[(size_t)r * a.cache_bstride + (size_t)pos * DH + (c - DH)] = vb;
    }
  }
  __syncthreads();
  if ((int)blockIdx.x >= b * splits) {
    // an idle CTA pulls the per-channel parameters of the next two hyper-connections (this layer's feed-forward branch,
    // the next layer's attention branch) towards L2: by then the weight stream has pushed them out
    if (blockIdx.x == gridDim.x - 1) {
      const unsigned long long* lp = cx.sTbl + (size_t)layer * NPTR;
      const int lines = (a.d * 4 + 127) / 128;
      for (int which_hc = 0; which_hc < 2; ++which_hc) {
        if (which_hc == 1 && layer + 1 >= a.L) break;
        const unsigned long long* q = which_hc == 0 ? lp + F_GAMMA : lp + NPTR + A_GAMMA;
        for (int i = threadIdx.x; i < lines; i += NT) {
          prefetch_l2(tptr<const char>(q, 0) + (size_t)i * 128);
          prefetch_l2(tptr<const char>(q, 2) + (size_t)i * 128);
          prefetch_l2(tptr<const char>(q, 7) + (size_t)i * 128);
        }
        for (int i = threadIdx.x; i < lines * HT; i += NT) prefetch_l2(tptr<const char>(q, 1) + (size_t)i * 128);
      }
    }
    return;
  }
  const int r = blockIdx.x / splits, sp = blockIdx.x - r * splits;
  const int chunk = ((n_all + splits - 1) / splits + 3) & ~3;
  const int j_begin = sp * chunk, j_end = min(n_all, j_begin + chunk);
  const int wph = H <= NW ? NW / H : 1;            // warps per head
  const int heads_per_pass = NW / wph;
  const __nv_bfloat16* kb = kc + (size_t)r * a.cache_bstride;
  const __nv_bfloat16* vb = vc + (size_t)r * a.cache_bstride;
  const uint8_t* mrow = a.key_mask ? a.key_mask + (size_t)r * a.mask_bstride : nullptr;
  const int grp = lane >> 3, l8 = lane & 7;        // 4 keys per warp step, 8 lanes x 8 channels per key
#pragma unroll 1
  for (int h0 = 0; h0 < H; h0 += heads_per_pass) {
    const int head = h0 + warp / wph, sub = warp % wph;
    if (head < H && warp < heads_per_pass * wph) {
      const uint4 qu = __ldcg(reinterpret_cast<const uint4*>(a.q + (size_t)r * HD + head * DH + l8 * 8));
      float m = -INFINITY, l = 0.f, acc[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = 0.f;
      const int step = 4 * wph;
      // 4 warp steps (16 keys of this warp) per round trip: all their K / V rows are requested before the first use
#pragma unroll 1
      for (int jb = j_begin + sub * 4; jb < j_end; jb += 4 * step) {
        uint4 ku[4], vu[4];
        bool valid[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int j = jb + u * step + grp;
          valid[u] = j < j_end;
          if (valid[u] && mrow != nullptr) valid[u] = mrow[j] != 0;
          ku[u] = make_uint4(0u, 0u, 0u, 0u);
          vu[u] = ku[u];
          if (valid[u]) {
            if (j == pos) {
              ku[u] = *reinterpret_cast<const uint4*>(cx.sKV + (size_t)r * 2 * DH + l8 * 8);
              vu[u] = *reinterpret_cast<const uint4*>(cx.sKV + (size_t)r * 2 * DH + DH + l8 * 8);
            } else {
              ku[u] = *reinterpret_cast<const uint4*>(kb + (size_t)j * DH + l8 * 8);
              vu[u] = *reinterpret_cast<const uint4*>(vb + (size_t)j * DH + l8 * 8);
            }
          }
        }
        const float qv[8] = {bf16_lo(qu.x) * a.scale_log2, bf16_hi(qu.x) * a.scale_log2, bf16_lo(qu.y) * a.scale_log2,
                             bf16_hi(qu.y) * a.scale_log2, bf16_lo(qu.z) * a.scale_log2, bf16_hi(qu.z) * a.scale_log2,
                             bf16_lo(qu.w) * a.scale_log2, bf16_hi(qu.w) * a.scale_log2};
        // the 4 steps of the batch share ONE running-maximum update (4 independent score chains, one rescale)
        float sc[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          float s = 0.f;
          s = fmaf(qv[0], bf16_lo(ku[u].x), s); s = fmaf(qv[1], bf16_hi(ku[u].x), s);
          s = fmaf(qv[2], bf16_lo(ku[u].y), s); s = fmaf(qv[3], bf16_hi(ku[u].y), s);
          s = fmaf(qv[4], bf16_lo(ku[u].z), s); s = fmaf(qv[5], bf16_hi(ku[u].z), s);
          s = fmaf(qv[6], bf16_lo(ku[u].w), s); s = fmaf(qv[7], bf16_hi(ku[u].w), s);
          s += __shfl_xor_sync(0xffffffffu, s, 1);
          s += __shfl_xor_sync(0xffffffffu, s, 2);
          s += __shfl_xor_sync(0xffffffffu, s, 4);
          sc[u] = valid[u] ? s : -INFINITY;
        }
        const float m_new = fmaxf(fmaxf(m, sc[0]), fmaxf(fmaxf(sc[1], sc[2]), sc[3]));
        if (m_new > -INFINITY) {   // (uniform over the 8 lanes of a key group)
          const float al = exp2f(m - m_new);
          l *= al;
#pragma unroll
          for (int e = 0; e < 8; ++e) acc[e] *= al;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float p = exp2f(sc[u] - m_new);   // 0 for an invalid key
            l += p;
            acc[0] = fmaf(p, bf16_lo(vu[u].x), acc[0]); acc[1] = fmaf(p, bf16_hi(vu[u].x), acc[1]);
            acc[2] = fmaf(p, bf16_lo(vu[u].y), acc[2]); acc[3] = fmaf(p, bf16_hi(vu[u].y), acc[3]);
            acc[4] = fmaf(p, bf16_lo(vu[u].z), acc[4]); acc[5] = fmaf(p, bf16_hi(vu[u].z), acc[5]);
            acc[6] = fmaf(p, bf16_lo(vu[u].w), acc[6]); acc[7] = fmaf(p, bf16_hi(vu[u].w), acc[7]);
          }
          m = m_new;
        }
      }
      // merge the 4 key groups of the warp
#pragma unroll
      for (int off = 8; off <= 16; off <<= 1) {
        const float mo = __shfl_xor_sync(0xffffffffu, m, off);
        const float lo = __shfl_xor_sync(0xffffffffu, l, off);
        const float mn = fmaxf(m, mo);
        const float f0 = (m == -INFINITY) ? 0.f : exp2f(m - mn);
        const float f1 = (mo == -INFINITY) ? 0.f : exp2f(mo - mn);
        l = l * f0 + lo * f1;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float ao = __shfl_xor_sync(0xffffffffu, acc[e], off);
          acc[e] = acc[e] * f0 + ao * f1;
        }
        m = mn;
      }
      float* ms = cx.sMerge + (size_t)warp * PART_W;
      if (lane == 0) { ms[0] = m; ms[1] = l; }
      if (lane < 8) {
#pragma unroll
        for (int e = 0; e < 8; ++e) ms[2 + lane * 8 + e] = acc[e];
      }
    }
    __syncthreads();
    // merge the warps of a head and publish the slice state
    for (int i = threadIdx.x; i < heads_per_pass * DH; i += NT) {
      const int hl = i / DH, dd = i - hl * DH;
      const int head2 = h0 + hl;
      if (head2 < H) {
        const float* ms = cx.sMerge + (size_t)(hl * wph) * PART_W;
        float mm = -INFINITY;
        for (int s2 = 0; s2 < wph; ++s2) mm = fmaxf(mm, ms[s2 * PART_W]);
        float ll = 0.f, aa = 0.f;
        for (int s2 = 0; s2 < wph; ++s2) {
          const float m2 = ms[s2 * PART_W];
          const float f = (m2 == -INFINITY) ? 0.f : exp2f(m2 - mm);
          ll = fmaf(ms[s2 * PART_W + 1], f, ll);
          aa = fmaf(ms[s2 * PART_W + 2 + dd], f, aa);
        }
        float* ps = a.part + (((size_t)r * splits + sp) * H + head2) * PART_W;
        if (dd == 0) { ps[0] = mm; ps[1] = ll; }
        ps[2 + dd] = aa;
      }
    }
    __syncthreads();
  }
}

// ---- phase C prologue: merge the slices (all their states requested in ONE round trip) -------------------------------
__device__ __noinline__ void merge_slices(const Args& a, const Ctx& cx) {
  const int H = a.H, HD = a.H * DH, splits = cx.splits;
  for (int i = threadIdx.x; i < a.b * HD; i += NT) {
    const int r = i / HD, hd = i - r * HD, head = hd / DH, dd = hd - head * DH;
    const float* ps = a.part + ((size_t)r * splits * H + head) * PART_W;
    const size_t sstride = (size_t)H * PART_W;
    float ms[MAX_SPLITS], ls[MAX_SPLITS], as[MAX_SPLITS];
#pragma unroll
    for (int s2 = 0; s2 < MAX_SPLITS; ++s2) {
      const bool on = s2 < splits;
      ms[s2] = on ? __ldcg(ps + s2 * sstride) : -INFINITY;
      ls[s2] = on ? __ldcg(ps + s2 * sstride + 1) : 0.f;
      as[s2] = on ? __ldcg(ps + s2 * sstride + 2 + dd) : 0.f;
    }
    float mm = -INFINITY;
#pragma unroll
    for (int s2 = 0; s2 < MAX_SPLITS; ++s2) mm = fmaxf(mm, ms[s2]);
    float ll = 0.f, aa = 0.f;
#pragma unroll
    for (int s2 = 0; s2 < MAX_SPLITS; ++s2) {
      const float f = (ms[s2] == -INFINITY) ? 0.f : exp2f(ms[s2] - mm);
      ll = fmaf(ls[s2], f, ll);
      aa = fmaf(as[s2], f, aa);
    }
    cx.sO[i] = __float2bfloat16(ll > 0.f ? __fdividef(aa, ll) : 0.f);   // fully masked row -> zeros (as alm_mqa_attn_fwd)
  }
  __syncthreads();
}

// ---- phase E prologue: GEGLU + LayerNorm(inner) of every row (geglu_ln_fwd_kernel) -------------------------------------
__device__ __noinline__ void geglu_rows(const Args& a, const Ctx& cx, const float* ln2, int& which) {
  const int ip = a.ip, inner = a.inner;
#pragma unroll 1
  for (int r = 0; r < a.b; ++r) {
    const __nv_bfloat16* hr = a.h + (size_t)r * 2 * ip;
    float v[MAXG][8], gm[MAXG][8];
    float s1 = 0.f, s2 = 0.f, dummy = 0.f;
#pragma unroll
    for (int k = 0; k < MAXG; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) { v[k][e] = 0.f; gm[k][e] = 0.f; }
      if (c0 < ip) {
        const uint4 ua = __ldcg(reinterpret_cast<const uint4*>(hr + c0));
        const uint4 ug = __ldcg(reinterpret_cast<const uint4*>(hr + ip + c0));
        if (c0 + 8 <= inner) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(ln2 + c0));
          const float4 g1 = __ldg(reinterpret_cast<const float4*>(ln2 + c0 + 4));
          gm[k][0] = g0.x; gm[k][1] = g0.y; gm[k][2] = g0.z; gm[k][3] = g0.w;
          gm[k][4] = g1.x; gm[k][5] = g1.y; gm[k][6] = g1.z; gm[k][7] = g1.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (c0 + e < inner) gm[k][e] = __ldg(ln2 + c0 + e);
        }
        const float av[8] = {bf16_lo(ua.x), bf16_hi(ua.x), bf16_lo(ua.y), bf16_hi(ua.y),
                             bf16_lo(ua.z), bf16_hi(ua.z), bf16_lo(ua.w), bf16_hi(ua.w)};
        const float gt[8] = {bf16_lo(ug.x), bf16_hi(ug.x), bf16_lo(ug.y), bf16_hi(ug.y),
                             bf16_lo(ug.z), bf16_hi(ug.z), bf16_lo(ug.w), bf16_hi(ug.w)};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float cdf, xpdf;
          gelu_parts(gt[e], cdf, xpdf);
          const float val = c0 + e < inner ? gt[e] * cdf * av[e] : 0.f;
          v[k][e] = val;
          s1 += val;
        }
      }
    }
    block_sum2(s1, dummy, cx.sRed2, which);
    const float mean = s1 * a.inv_inner;
    // the variance in a second pass over the registers (as geglu_ln_fwd_kernel)
#pragma unroll
    for (int k = 0; k < MAXG; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (c0 + e < inner) s2 = fmaf(v[k][e] - mean, v[k][e] - mean, s2);
    }
    dummy = 0.f;
    block_sum2(s2, dummy, cx.sRed2, which);
    const float rstd = rsqrtf(s2 * a.inv_inner + 1e-5f);
#pragma unroll
    for (int k = 0; k < MAXG; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
      if (c0 < ip) {
        __nv_bfloat162 o[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float lo = c0 + 2 * e < inner ? (v[k][2 * e] - mean) * rstd * gm[k][2 * e] : 0.f;
          const float hi = c0 + 2 * e + 1 < inner ? (v[k][2 * e + 1] - mean) * rstd * gm[k][2 * e + 1] : 0.f;
          o[e] = __floats2bfloat162_rn(lo, hi);
        }
        *reinterpret_cast<uint4*>(cx.sGn + (size_t)r * ip + c0) = *reinterpret_cast<const uint4*>(o);
      }
    }
  }
  __syncthreads();
}

// ---- end: depth of the last branch, stream sum, final LayerNorm (hc_post_fwd_kernel), CTA 0 only -----------------------
__device__ __noinline__ void final_post(const Args& a, const Ctx& cx, int& which) {
  const int d = a.d;
#pragma unroll 1
  for (int r = 0; r < a.b; ++r) {
    const float bsum = cx.sBeta[r * HS] + cx.sBeta[r * HS + 1] + cx.sBeta[r * HS + 2] + cx.sBeta[r * HS + 3];
    constexpr int MAXC = 2 * MAXP;
    float xs[MAXC];
    float s1 = 0.f, dummy = 0.f;
#pragma unroll
    for (int k = 0; k < MAXC; ++k) {
      const int c = threadIdx.x + k * NT;
      xs[k] = 0.f;
      if (c < d) {
        float v = 0.f;
#pragma unroll
        for (int s = 0; s < HS; ++s) v += __bfloat162float(cx.sR[((size_t)r * HS + s) * d + c]);
        v += bsum * ld_bf16_cg(a.Y2 + (size_t)r * d + c);
        xs[k] = v;
        s1 += v;
      }
    }
    block_sum2(s1, dummy, cx.sRed2, which);
    const float mean = s1 * a.inv_d;
    float s2 = 0.f;
    dummy = 0.f;
#pragma unroll
    for (int k = 0; k < MAXC; ++k) {
      const int c = threadIdx.x + k * NT;
      if (c < d) s2 += (xs[k] - mean) * (xs[k] - mean);
    }
    block_sum2(s2, dummy, cx.sRed2, which);
    const float rstd = rsqrtf(s2 * a.inv_d + 1e-5f);
#pragma unroll
    for (int k = 0; k < MAXC; ++k) {
      const int c = threadIdx.x + k * NT;
      if (c < d) a.out[(size_t)r * d + c] = __float2bfloat16((xs[k] - mean) * rstd * __ldg(a.final_gamma + c));
    }
  }
  if (threadIdx.x == 0) *a.len = cx.pos + 1;
}

__device__ __noinline__ void jobs_of(const Args& a, const Ctx& cx, int layer, Job* J /*[4]: q|kv, out, W1, W2*/) {
  const unsigned long long* lp = cx.sTbl + (size_t)layer * NPTR;
  const int d = a.d, HD = a.H * DH, ip = a.ip, G = gridDim.x;
  // (k / v come from the UN-normalised branch input)
  J[0] = Job{tptr<const __nv_bfloat16>(lp, P_WA), HD + 2 * DH, d, ceil_div(HD + 2 * DH, G), HD, cx.sXn, cx.sBin, a.q, a.kvn, HD, 2 * DH};
  J[1] = Job{tptr<const __nv_bfloat16>(lp, P_WC), d, HD, ceil_div(d, G), d, cx.sO, cx.sO, a.Y, a.Y, d, d};
  J[2] = Job{tptr<const __nv_bfloat16>(lp, P_WD), 2 * ip, d, ceil_div(2 * ip, G), 2 * ip, cx.sXn, cx.sXn, a.h, a.h, 2 * ip, 2 * ip};
  J[3] = Job{tptr<const __nv_bfloat16>(lp, P_WE), d, ip, ceil_div(d, G), d, cx.sGn, cx.sGn, a.Y2, a.Y2, d, d};
}

// ---- the kernel ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT, 1) decode_stack_step_kernel(const __grid_constant__ Args a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  const int b = a.b, d = a.d, H = a.H, ip = a.ip, HD = a.H * DH;
  // shared-memory carve-up (all offsets 16-byte aligned: d, ip, HD are multiples of 8)
  Ctx cx;
  cx.sR = reinterpret_cast<__nv_bfloat16*>(smem_raw);                         // [b][HS][d]
  cx.sBin = cx.sR + (size_t)b * HS * d;                                       // [b][d]
  cx.sXn = cx.sBin + (size_t)b * d;                                           // [b][d]
  cx.sGn = cx.sXn + (size_t)b * d;                                            // [b][ip]
  cx.sO = cx.sGn + (size_t)b * ip;                                            // [b][HD]
  cx.sKV = cx.sO + (size_t)b * HD;                                            // [b][128] new k | v (after the value residual)
  cx.sVfirst = reinterpret_cast<float*>(cx.sKV + (size_t)b * 128);            // [b][64]
  cx.sBeta = cx.sVfirst + b * DH;                                             // [MAXB][HS]
  cx.sRed32 = cx.sBeta + MAXB * HS;                                           // [NW][32]
  cx.sRed2 = cx.sRed32 + NW * 32;                                             // [2][NW][2]
  cx.sStat = cx.sRed2 + 4 * NW;                                               // [32]
  cx.sGacc = cx.sStat + 32;                                                   // [MAX_SLOTS][MAXB]
  cx.sMerge = cx.sGacc + MAX_SLOTS * MAXB;                                    // [max(NW, H)][PART_W]
  unsigned long long* sTblW = reinterpret_cast<unsigned long long*>(cx.sMerge + (size_t)(H > NW ? H : NW) * PART_W);
  cx.sTbl = sTblW;                                                            // [L][NPTR]
  cx.sBar = reinterpret_cast<uint64_t*>(sTblW + (size_t)a.L * NPTR);          // [4] one per weight slot
#pragma unroll
  for (int i = 0; i < 4; ++i) cx.slot[i] = a.st_off[i] >= 0 ? reinterpret_cast<__nv_bfloat16*>(smem_raw + a.st_off[i]) : nullptr;

  for (int i = threadIdx.x; i < a.L * NPTR; i += NT) sTblW[i] = __ldg(a.table + i);
  if (threadIdx.x == 0) {
    for (int i = 0; i < 4; ++i) mbar_init(&cx.sBar[i], 1);
    fence_mbar_init();
  }
#ifdef ALM_DSTEP_TRACE
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    g_sub_trace = a.trace + 32 * 16;
    g_sub_count = 0;
  }
#endif
  unsigned epoch = 0;
  int which = 0;
  cx.pos = *a.len;                              // position of the new token
  cx.has_new = cx.pos >= 0 && cx.pos < a.max_len;
  cx.n_all = min(cx.pos + 1, a.max_len);
  cx.splits = min(a.splits, max(1, (cx.n_all + KEYS_PER_SPLIT - 1) / KEYS_PER_SPLIT));
  __syncthreads();

  Job J[4], N[4];
  jobs_of(a, cx, 0, J);
  for (int i = 0; i < 4; ++i) stage_rows(J[i], cx.slot[i], &cx.sBar[i]);   // weights of layer 0

#pragma unroll 1
  for (int layer = 0; layer < a.L; ++layer) {
    const unsigned long long* lp = cx.sTbl + (size_t)layer * NPTR;
    const bool has_next = layer + 1 < a.L;
    if (has_next) jobs_of(a, cx, layer + 1, N);
    const uint32_t parity = layer & 1;

    // ---------------- A: hyper-connection (attention branch) + q / kv projections ----------------
    DSTEP_STAMP(0);
#pragma unroll 1
    for (int r = 0; r < b; ++r)
      hc_pre_row(cx, layer == 0, lp, A_GAMMA, d, a.inv_d, r, a.x + (size_t)r * d, a.Y2 + (size_t)r * d, which);
    DSTEP_STAMP(1);
    gemv_phase(J[0], N[0], has_next, b, cx.sGacc, cx.slot[0], &cx.sBar[0], parity);
    DSTEP_STAMP(2);
    grid_barrier(a.counter, epoch, a.err);
    DSTEP_STAMP(3);

    // ---------------- B: attention over the cache ----------------
    attn_slices(a, cx, layer, tptr<__nv_bfloat16>(lp, P_KC), tptr<__nv_bfloat16>(lp, P_VC));
    DSTEP_STAMP(4);
    grid_barrier(a.counter, epoch, a.err);
    DSTEP_STAMP(5);

    // ---------------- C: merge the slices, out projection ----------------
    merge_slices(a, cx);
    DSTEP_STAMP(6);
    gemv_phase(J[1], N[1], has_next, b, cx.sGacc, cx.slot[1], &cx.sBar[1], parity);
    DSTEP_STAMP(7);
    grid_barrier(a.counter, epoch, a.err);
    DSTEP_STAMP(8);

    // ---------------- D: hyper-connection (feed-forward branch) + W1 ----------------
#pragma unroll 1
    for (int r = 0; r < b; ++r)
      hc_pre_row(cx, false, lp, F_GAMMA, d, a.inv_d, r, nullptr, a.Y + (size_t)r * d, which);
    DSTEP_STAMP(9);
    gemv_phase(J[2], N[2], has_next, b, cx.sGacc, cx.slot[2], &cx.sBar[2], parity);
    DSTEP_STAMP(10);
    grid_barrier(a.counter, epoch, a.err);
    DSTEP_STAMP(11);

    // ---------------- E: GEGLU + LayerNorm(inner), W2 ----------------
    geglu_rows(a, cx, tptr<const float>(lp, P_LN2), which);
    DSTEP_STAMP(12);
    gemv_phase(J[3], N[3], has_next, b, cx.sGacc, cx.slot[3], &cx.sBar[3], parity);
    DSTEP_STAMP(13);
    grid_barrier(a.counter, epoch, a.err);
    DSTEP_STAMP(14);
#pragma unroll
    for (int i = 0; i < 4; ++i) J[i] = N[i];
  }
  if (blockIdx.x == 0) final_post(a, cx, which);
}

// shared memory: fixed part, then the weight slots that fit (A, C, E first: they are small; D = the W1 rows last)
struct SmemPlan {
  size_t total;
  int st_off[4];
};
inline SmemPlan smem_plan(int L, int b, int d, int H, int ip, int grid) {
  size_t n = 0;
  n += (size_t)b * HS * d * 2 + (size_t)b * d * 2 * 2 + (size_t)b * ip * 2 + (size_t)b * H * DH * 2 + (size_t)b * 128 * 2;
  n += ((size_t)b * DH + MAXB * HS + NW * 32 + 4 * NW + 32 + MAX_SLOTS * MAXB + (size_t)(H > NW ? H : NW) * PART_W) * 4;
  n += (size_t)L * NPTR * 8 + 4 * 8;  // pointer table, mbarriers
  n = (n + 15) & ~size_t(15);
  const int HD = H * DH;
  const size_t need[4] = {(size_t)ceil_div(HD + 2 * DH, grid) * d * 2, (size_t)ceil_div(d, grid) * HD * 2,
                          (size_t)ceil_div(2 * ip, grid) * d * 2, (size_t)ceil_div(d, grid) * ip * 2};
  const size_t budget = 220 * 1024;
  SmemPlan p;
  const int order[4] = {0, 1, 3, 2};
  for (int i = 0; i < 4; ++i) p.st_off[i] = -1;
  for (int oi = 0; oi < 4; ++oi) {
    const int i = order[oi];
    if (n + need[i] <= budget) {
      p.st_off[i] = (int)n;
      n += (need[i] + 15) & ~size_t(15);
    }
  }
  p.total = n;
  return p;
}

constexpr size_t SMEM_LIMIT = 224 * 1024;   // dynamic shared memory the kernel is allowed

// Every shape limit of the kernel, in one place: alm_decode_stack_plan reports it to the host (which falls back to the
// multi-kernel step for a refused shape) and alm_decode_stack_step refuses exactly these shapes.  Fills *plan.
inline bool shape_supported(int L, int b, int d, int H, int inner, int grid, SmemPlan* plan) {
  if (b < 1 || b > MAXB || H < 1 || H > 64 || L < 1 || L > MAXL) return false;
  if (d % 8 != 0 || d < 8 || d > 2 * MAXP * NT || inner < 1 || inner > 8 * MAXG * NT - 8) return false;
  const int ip = (inner + 7) & ~7, HD = H * DH;
  // a thread owns one 8-channel chunk of K; per-warp partial sums of a phase must fit the shared-memory table
  const int Ns[4] = {HD + 2 * DH, d, 2 * ip, d}, Ks[4] = {d, HD, d, ip};
  for (int i = 0; i < 4; ++i)
    if (Ks[i] / 8 > NT || ceil_div(Ns[i], grid) * ceil_div(Ks[i] / 8, 32) > MAX_SLOTS) return false;
  *plan = smem_plan(L, b, d, H, ip, grid);
  return plan->total <= SMEM_LIMIT;
}

struct Scratch {
  size_t counter, err, q, kvn, part, Y, Y2, h, trace, total;
};
inline Scratch scratch_layout(int b, int d, int H, int ip, int splits) {
  Scratch s;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    const size_t at = o;
    o += (bytes + 255) & ~size_t(255);
    return at;
  };
  s.counter = take(4);
  s.err = take(4);
  s.q = take((size_t)b * H * DH * 2);
  s.kvn = take((size_t)b * 128 * 2);
  s.part = take((size_t)b * splits * H * PART_W * 4);
  s.Y = take((size_t)b * d * 2);
  s.Y2 = take((size_t)b * d * 2);
  s.h = take((size_t)b * 2 * ip * 2);
  s.trace = take((size_t)MAXL * 16 * 8);
  s.total = o;
  return s;
}
inline int pick_splits(int b) { return max(1, min(MAX_SPLITS, num_sms() / max(b, 1))); }

}  // namespace dstep
}  // namespace alm

using namespace alm;

// byte offset of the [64][16] int64 phase-stamp area inside the scratch (filled only by -DALM_DSTEP_TRACE builds)
extern "C" int64_t alm_decode_stack_trace_offset(int b, int d, int heads, int inner) {
  if (b < 1 || b > dstep::MAXB || d < 8 || heads < 1 || inner < 1) return -1;
  return (int64_t)dstep::scratch_layout(b, d, heads, (inner + 7) & ~7, dstep::pick_splits(b)).trace;
}

// CTAs of the step kernel = SMs of the current device (the row regrouping of the operands depends on it)
extern "C" int alm_decode_stack_grid() { return num_sms(); }

extern "C" int64_t alm_decode_stack_scratch_bytes(int b, int d, int heads, int inner) {
  if (b < 1 || b > dstep::MAXB || d < 8 || heads < 1 || inner < 1) return -1;
  const int ip = (inner + 7) & ~7;
  return (int64_t)dstep::scratch_layout(b, d, heads, ip, dstep::pick_splits(b)).total;
}

extern "C" int alm_decode_stack_plan(int b, int d, int heads, int inner, int n_layers, int32_t* staged) {
  dstep::SmemPlan plan;
  if (!dstep::shape_supported(n_layers, b, d, heads, inner, num_sms(), &plan)) return ALM_ERR_UNSUPPORTED;
  if (staged != nullptr)
    for (int i = 0; i < 4; ++i) staged[i] = plan.st_off[i] >= 0;
  return ALM_OK;
}

extern "C" int alm_decode_stack_plan_dh(int b, int d, int heads, int inner, int n_layers, int dim_head, int32_t* staged) {
  if (dim_head != dstep::DH) return ALM_ERR_UNSUPPORTED;   // the one-kernel step is built for one head width
  return alm_decode_stack_plan(b, d, heads, inner, n_layers, staged);
}

extern "C" int alm_decode_stack_step(const void* layer_table, int n_layers, const float* x, void* out,
                                     const float* final_gamma, int32_t* len, int max_len, int64_t cache_bstride,
                                     const void* key_mask, int64_t mask_bstride, void* scratch, int64_t scratch_bytes,
                                     int b, int d, int heads, int inner, int value_residual, float scale,
                                     int grid_ctas, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(layer_table && x && out && final_gamma && len && scratch && n_layers > 0, ALM_ERR_ARG);
  ALM_REQUIRE(max_len > 0, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(cache_bstride % 8 == 0 && (reinterpret_cast<uintptr_t>(scratch) & 255u) == 0, ALM_ERR_ALIGN);
  const int grid = num_sms();
  ALM_REQUIRE(grid_ctas == grid, ALM_ERR_ARG);   // the operands were regrouped for this many CTAs
  dstep::SmemPlan plan;
  ALM_REQUIRE(dstep::shape_supported(n_layers, b, d, heads, inner, grid, &plan), ALM_ERR_UNSUPPORTED);
  const int ip = (inner + 7) & ~7;
  const int splits = dstep::pick_splits(b);
  const dstep::Scratch lay = dstep::scratch_layout(b, d, heads, ip, splits);
  ALM_REQUIRE(scratch_bytes >= (int64_t)lay.total, ALM_ERR_ARG);
  static bool attr = false;
  if (!attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(dstep::decode_stack_step_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)dstep::SMEM_LIMIT));
    attr = true;
  }
  uint8_t* sc = reinterpret_cast<uint8_t*>(scratch);
  dstep::Args a;
  a.table = reinterpret_cast<const unsigned long long*>(layer_table);
  a.x = x;
  a.out = reinterpret_cast<__nv_bfloat16*>(out);
  a.final_gamma = final_gamma;
  a.len = len;
  a.key_mask = reinterpret_cast<const uint8_t*>(key_mask);
  a.mask_bstride = mask_bstride;
  a.cache_bstride = cache_bstride;
  a.counter = reinterpret_cast<unsigned*>(sc + lay.counter);
  a.err = reinterpret_cast<int*>(sc + lay.err);
  a.q = reinterpret_cast<__nv_bfloat16*>(sc + lay.q);
  a.kvn = reinterpret_cast<__nv_bfloat16*>(sc + lay.kvn);
  a.part = reinterpret_cast<float*>(sc + lay.part);
  a.Y = reinterpret_cast<__nv_bfloat16*>(sc + lay.Y);
  a.Y2 = reinterpret_cast<__nv_bfloat16*>(sc + lay.Y2);
  a.h = reinterpret_cast<__nv_bfloat16*>(sc + lay.h);
  a.trace = reinterpret_cast<long long*>(sc + lay.trace);
  a.L = n_layers; a.b = b; a.d = d; a.H = heads; a.inner = inner; a.ip = ip; a.max_len = max_len;
  a.splits = splits; a.value_residual = value_residual;
  a.scale_log2 = scale * 1.4426950408889634f;
  a.inv_d = 1.f / (float)d;
  a.inv_inner = 1.f / (float)inner;
  for (int i = 0; i < 4; ++i) a.st_off[i] = plan.st_off[i];
  // the barrier counter restarts at 0 every launch (the error flag is sticky: the host reads it in tests)
  ALM_CUDA_OK(cudaMemsetAsync(a.counter, 0, 4, stream));
  // co-residency of all CTAs is what the device-wide barrier relies on: one CTA per SM, cooperative launch
  void* kargs[] = {(void*)&a};
  ALM_CUDA_OK(cudaLaunchCooperativeKernel((const void*)dstep::decode_stack_step_kernel, dim3(grid), dim3(dstep::NT),
                                          kargs, plan.total, stream));
  ALM_LAUNCHED(1);
  return ALM_OK;
}
