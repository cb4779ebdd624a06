// SoundStream gate-loop layer (use_gate_loop_layers=True; the reference wraps gateloop-transformer's
// SimpleGateLoopLayer as Residual(ChannelTranspose(.)), soundstream.py:314-330, 524-525, 620-621):
//   r_t = 1 / max(||u_t||_2, 1e-12),   [q; kv; a]_t = r_t W' u_t,   W' = W diag(sqrt(C) gamma)  (ops.gate_loop_fold_weight)
//   h_t = sigmoid(a_t) * h_{t-1} + kv_t,  h_{-1} = 0                (per batch and channel, forward in time)
//   y_t = 2 u_t + q_t * h_t
//
// Both paths use a fixed-order two-pass scan over time tiles, so every output is the same bits on every run:
//   pass 1: per tile and channel, the tile's aggregate (A, H) = (prod sigmoid(a), end state from 0);
//   carry (carry_kernel): per batch and channel, in tile order, the state entering each tile;
//   pass 2: per tile, the recurrence from its carry-in, and the output.
// No CTA waits on another.  Inside a tile each channel's steps are cut into sub-chunks scanned by separate threads,
// whose aggregates are combined in sub-chunk order.
//
// Tensor-core path (proj_scan_tc_kernel, C8S in and out): a CTA owns 64 time steps and a slice of NS channels and
// computes q, kv and a of that slice on wgmma (split bf16: x_hi w_hi + x_lo w_hi + x_hi w_lo), so the projection never
// leaves the CTA; pass 1 computes only kv and a, pass 2 recomputes all three.  The epilogue applies r_t (from per-chunk
// sums of squares gathered while x streams through shared memory), the sigmoid and the scan.
// CUDA-core path (fp32 [B][C][T]): the projection fp32 [B][3C][T] comes from alm_causal_conv1d_fwd (K = 1); the
// tile_agg / apply kernels here do the norm, the gates and the scan.
#include <cuda_bf16.h>

#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace gl {

constexpr int THREADS = 128;
constexpr int TILE_FLOATS = 8192;  // fp32 path: x tile [TT][C + 1] fp32 in shared memory: TT = clamp(8192 / C, 8, 128) steps

struct Params {
  const float* x;     // fp32 [B][C][T]
  const float* proj;  // fp32 [B][3C][T]; rows q [0, C), kv [C, 2C), a [2C, 3C)
  float* y;           // fp32 [B][C][T]
  float* agg_a;       // [B][ntiles][C] tile aggregates (pass 1)
  float* agg_h;
  float* carry;       // [B][ntiles][C] state entering each tile; null when ntiles == 1
  int B, C, T, tt, ntiles, nsub;
};

static int tile_steps(int C) { return max(8, min(128, TILE_FLOATS / C)); }

__device__ __forceinline__ void load_tile(const Params& p, int b, int t0, int n, float* xs) {
  const int ld = p.C + 1;
  for (int i = threadIdx.x; i < p.C * n; i += THREADS) {
    const int c = i / n, t = i - c * n;
    xs[t * ld + c] = __ldg(p.x + ((size_t)b * p.C + c) * p.T + t0 + t);
  }
}

__device__ __forceinline__ void store_tile(const Params& p, int b, int t0, int n, const float* xs) {
  const int ld = p.C + 1;
  for (int i = threadIdx.x; i < p.C * n; i += THREADS) {
    const int c = i / n, t = i - c * n;
    p.y[((size_t)b * p.C + c) * p.T + t0 + t] = xs[t * ld + c];
  }
}

// rn[t] = 1 / max(||x_t||_2, 1e-12) for the n staged steps: one warp per step, lanes over channels, fixed shuffle tree
__device__ __forceinline__ void tile_norms(const Params& p, int n, const float* xs, float* rn) {
  const int ld = p.C + 1, lane = threadIdx.x & 31;
  for (int t = threadIdx.x >> 5; t < n; t += THREADS / 32) {
    float s = 0.f;
    for (int c = lane; c < p.C; c += 32) s = fmaf(xs[t * ld + c], xs[t * ld + c], s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) rn[t] = rsqrtf(fmaxf(s, 1e-24f));
  }
}

__device__ __forceinline__ float proj_at(const Params& p, int b, int row, int t) {
  return __ldg(p.proj + ((size_t)b * 3 * p.C + row) * p.T + t);
}

// fast-math intrinsics (MUFU, about 2 ulp): IEEE division, expf and sqrtf would bring slow-path subroutine calls
__device__ __forceinline__ float sigmoidf_(float v) { return __fdividef(1.f, 1.f + __expf(-v)); }

// (A, H) of each channel's sub-chunk s of the tile: steps [s * len, (s + 1) * len), len = ceil(n / nsub), from a zero state
__device__ __forceinline__ void sub_aggregates(const Params& p, int b, int t0, int n, const float* rn, float* sub_a,
                                               float* sub_h) {
  const int len = (n + p.nsub - 1) / p.nsub;
  for (int w = threadIdx.x; w < p.C * p.nsub; w += THREADS) {
    const int c = w % p.C, s = w / p.C;
    float A = 1.f, H = 0.f;
    const int e = min(n, (s + 1) * len);
    for (int t = s * len; t < e; ++t) {
      const float g = sigmoidf_(proj_at(p, b, 2 * p.C + c, t0 + t) * rn[t]);
      H = fmaf(g, H, proj_at(p, b, p.C + c, t0 + t) * rn[t]);
      A *= g;
    }
    sub_a[s * p.C + c] = A;
    sub_h[s * p.C + c] = H;
  }
}

// pass 1: per tile and channel, (A, H) of the tile's steps from a zero state
__global__ void __launch_bounds__(THREADS) tile_agg_kernel(const Params p) {
  extern __shared__ float smem[];
  const int tile = blockIdx.x, b = blockIdx.y;
  const int t0 = tile * p.tt, n = min(p.tt, p.T - t0);
  float* xs = smem;                              // [tt][C + 1]
  float* rn = xs + p.tt * (p.C + 1);            // [tt]
  float* sub_a = rn + p.tt;                     // [nsub][C]
  float* sub_h = sub_a + p.nsub * p.C;
  load_tile(p, b, t0, n, xs);
  __syncthreads();
  tile_norms(p, n, xs, rn);
  __syncthreads();
  sub_aggregates(p, b, t0, n, rn, sub_a, sub_h);
  __syncthreads();
  for (int c = threadIdx.x; c < p.C; c += THREADS) {
    float A = 1.f, H = 0.f;
    for (int s = 0; s < p.nsub; ++s) {
      const float a_ = sub_a[s * p.C + c];
      H = fmaf(a_, H, sub_h[s * p.C + c]);
      A *= a_;
    }
    const size_t o = ((size_t)b * p.ntiles + tile) * p.C + c;
    p.agg_a[o] = A;
    p.agg_h[o] = H;
  }
}

// per batch and channel, in tile order: carry[b][i][c] = state after tiles 0 .. i-1 (both paths)
__global__ void __launch_bounds__(THREADS) carry_kernel(const float* __restrict__ agg_a, const float* __restrict__ agg_h,
                                                        float* __restrict__ carry, int B, int C, int ntiles) {
  const int i = blockIdx.x * THREADS + threadIdx.x;
  if (i >= B * C) return;
  const int b = i / C, c = i - b * C;
  float h = 0.f;
  for (int tile = 0; tile < ntiles; ++tile) {
    const size_t o = ((size_t)b * ntiles + tile) * C + c;
    carry[o] = h;
    h = fmaf(__ldg(agg_a + o), h, __ldg(agg_h + o));
  }
}

// pass 2: each sub-chunk's carry-in from the tile's carry-in and the preceding sub-chunks, then y = 2u + q * h
__global__ void __launch_bounds__(THREADS) apply_kernel(const Params p) {
  extern __shared__ float smem[];
  const int tile = blockIdx.x, b = blockIdx.y;
  const int t0 = tile * p.tt, n = min(p.tt, p.T - t0);
  float* xs = smem;
  float* rn = xs + p.tt * (p.C + 1);
  float* sub_a = rn + p.tt;
  float* sub_h = sub_a + p.nsub * p.C;
  const int ld = p.C + 1;
  load_tile(p, b, t0, n, xs);
  __syncthreads();
  tile_norms(p, n, xs, rn);
  __syncthreads();
  if (p.nsub > 1) {
    sub_aggregates(p, b, t0, n, rn, sub_a, sub_h);
    __syncthreads();
  }
  const int len = (n + p.nsub - 1) / p.nsub;
  for (int w = threadIdx.x; w < p.C * p.nsub; w += THREADS) {
    const int c = w % p.C, s = w / p.C;
    float h = p.carry ? __ldg(p.carry + ((size_t)b * p.ntiles + tile) * p.C + c) : 0.f;
    for (int s2 = 0; s2 < s; ++s2) h = fmaf(sub_a[s2 * p.C + c], h, sub_h[s2 * p.C + c]);
    const int e = min(n, (s + 1) * len);
    for (int t = s * len; t < e; ++t) {
      const float q = proj_at(p, b, c, t0 + t) * rn[t];
      const float g = sigmoidf_(proj_at(p, b, 2 * p.C + c, t0 + t) * rn[t]);
      h = fmaf(g, h, proj_at(p, b, p.C + c, t0 + t) * rn[t]);
      const float u = xs[t * ld + c];
      xs[t * ld + c] = fmaf(q, h, 2.f * u);  // each (t, c) is read and written by this thread only
    }
  }
  __syncthreads();
  store_tile(p, b, t0, n, xs);
}

static int run_fp32(Params p, cudaStream_t stream) {
  const size_t smem = (size_t)(p.tt * (p.C + 1) + p.tt + 2 * p.nsub * p.C) * sizeof(float);
  if (smem > 48 * 1024) return ALM_ERR_UNSUPPORTED;
  const dim3 grid(p.ntiles, p.B);
  if (p.ntiles > 1) {
    tile_agg_kernel<<<grid, THREADS, smem, stream>>>(p);
    ALM_CHECK_LAUNCH();
    carry_kernel<<<ceil_div(p.B * p.C, THREADS), THREADS, 0, stream>>>(p.agg_a, p.agg_h, p.carry, p.B, p.C, p.ntiles);
    ALM_CHECK_LAUNCH();
    ALM_LAUNCHED(2);
  } else {
    p.carry = nullptr;
  }
  apply_kernel<<<grid, THREADS, smem, stream>>>(p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// ---------------------------------------------------------------------------------------------
// Tensor-core path: fused projection + scan on C8S activations.
// CTA = (channel slice of NS, 64-step time tile, batch); one warpgroup.  x streams through shared memory in blocks of
// KB = min(C, 64) channels: A hi / lo [KB/8 chunks][64 rows][8] bf16 is the no-swizzle K-major layout (a core matrix is
// 8 consecutive time steps of one 8-channel chunk, contiguous in C8S too), W' [KB/16 k-steps][hi, lo][2][3 NS][8] the
// slice's rows q | kv | a as ops.pack_gate_loop_weights lays them out.  Three m64nNSk16 accumulators (two in pass 1).
// ---------------------------------------------------------------------------------------------
constexpr int TC_M = 64;

struct TcParams {
  const __nv_bfloat16* x;   // C8S [B][2C/8][T][8]
  const __nv_bfloat16* w;   // [C/NS][C/16][2][2][3 NS][8]
  __nv_bfloat16* y;         // C8S
  float* agg_a;             // [B][ntiles][C]
  float* agg_h;
  const float* carry;       // [B][ntiles][C] or null (ntiles == 1)
  int C, T, ntiles;
};

template <int NS>
struct TcCfg {
  static constexpr int NSUB = 128 / NS;                       // sub-chunks of a channel's 64 steps
  static constexpr int KB_MAX = 64;
  static constexpr int A_BYTES = 2 * KB_MAX * TC_M * 2;       // hi + lo, 16 KB
  static constexpr int W_BYTES = (KB_MAX / 16) * 2 * 2 * 3 * NS * 16;
  static constexpr int P_BYTES = 3 * TC_M * (NS + 1) * 4;     // epilogue: q | kv | a fp32, aliases A + W
  static constexpr int MAIN_BYTES = (A_BYTES + W_BYTES) > P_BYTES ? (A_BYTES + W_BYTES) : P_BYTES;
  static constexpr int U_BYTES = TC_M * (NS + 1) * 4;         // x of the slice, then y
  static constexpr int SMALL_BYTES = (TC_M + 2 * NSUB * NS) * 4;
  static int smem(int C) { return MAIN_BYTES + U_BYTES + (C / 8) * TC_M * 4 + SMALL_BYTES + 128; }
};

template <int NS, bool PASS2>
__global__ void __launch_bounds__(128, 1) proj_scan_tc_kernel(const TcParams p) {
  using Cfg = TcCfg<NS>;
  constexpr int NSUB = Cfg::NSUB, LEN = TC_M / NSUB, ACC = NS / 2;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  uint8_t* sA = smem;
  uint8_t* sW = smem + Cfg::A_BYTES;
  float* sP = reinterpret_cast<float*>(smem);                        // after the K loop
  float* sU = reinterpret_cast<float*>(smem + Cfg::MAIN_BYTES);      // [64][NS + 1]
  float* sSq = sU + TC_M * (NS + 1);                                 // [C/8][64] sums of squares per chunk and step
  float* sRn = sSq + (p.C / 8) * TC_M;                               // [64]
  float* sSubA = sRn + TC_M;                                         // [NSUB][NS]
  float* sSubH = sSubA + NSUB * NS;

  const int slice = blockIdx.x, tile = blockIdx.y, b = blockIdx.z;
  const int c0 = slice * NS, t0 = tile * TC_M, n = min(TC_M, p.T - t0);
  const int tid = threadIdx.x, nch = p.C / 8;
  const int KB = p.C < Cfg::KB_MAX ? p.C : Cfg::KB_MAX;
  const __nv_bfloat16* xb = p.x + (size_t)b * 2 * nch * p.T * 8;
  const uint4* wslice = reinterpret_cast<const uint4*>(p.w + (size_t)slice * (p.C / 16) * 2 * 2 * 3 * NS * 8);

  float dq[ACC], dk[ACC], da[ACC];
#pragma unroll
  for (int i = 0; i < ACC; ++i) { dq[i] = 0.f; dk[i] = 0.f; da[i] = 0.f; }

  for (int kb = 0; kb < p.C; kb += KB) {
    const int kch = KB / 8;
    // A block: hi / lo of chunks [kb/8, kb/8 + kch) for the tile's 64 rows (zero past T); sums of squares on the way
    for (int i = tid; i < kch * TC_M; i += 128) {
      const int g = i / TC_M, t = i - g * TC_M;
      uint4 hv = make_uint4(0, 0, 0, 0), lv = hv;
      if (t < n) {
        hv = __ldg(reinterpret_cast<const uint4*>(xb + ((size_t)(kb / 8 + g) * p.T + t0 + t) * 8));
        lv = __ldg(reinterpret_cast<const uint4*>(xb + ((size_t)(nch + kb / 8 + g) * p.T + t0 + t) * 8));
      }
      reinterpret_cast<uint4*>(sA)[g * TC_M + t] = hv;
      reinterpret_cast<uint4*>(sA)[(kch + g) * TC_M + t] = lv;
      const __nv_bfloat162* h2 = reinterpret_cast<const __nv_bfloat162*>(&hv);
      const __nv_bfloat162* l2 = reinterpret_cast<const __nv_bfloat162*>(&lv);
      float sq = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 hf = __bfloat1622float2(h2[j]), lf = __bfloat1622float2(l2[j]);
        const float v0 = hf.x + lf.x, v1 = hf.y + lf.y;
        sq = fmaf(v0, v0, sq);
        sq = fmaf(v1, v1, sq);
      }
      sSq[(kb / 8 + g) * TC_M + t] = sq;
      const int cl = 8 * (kb / 8 + g) - c0;   // this chunk's x also feeds the output's skip term
      if (PASS2 && cl >= 0 && cl < NS && t < n) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 hf = __bfloat1622float2(h2[j]), lf = __bfloat1622float2(l2[j]);
          sU[t * (NS + 1) + cl + 2 * j] = hf.x + lf.x;
          sU[t * (NS + 1) + cl + 2 * j + 1] = hf.y + lf.y;
        }
      }
    }
    // W block: k-steps [kb/16, kb/16 + KB/16) of the slice, contiguous in the packed units
    const int wvec = (KB / 16) * 2 * 2 * 3 * NS;
    const uint4* wsrc = wslice + (size_t)(kb / 16) * 2 * 2 * 3 * NS;
    for (int i = tid; i < wvec; i += 128) reinterpret_cast<uint4*>(sW)[i] = __ldg(wsrc + i);
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
    const uint32_t a_addr = smem_u32(sA), w_addr = smem_u32(sW);
#pragma unroll 1
    for (int kk = 0; kk < KB / 16; ++kk) {
      const uint64_t a_hi = wgmma_desc_nosw(a_addr + 2 * kk * TC_M * 16, 128, TC_M * 16);
      const uint64_t a_lo = wgmma_desc_nosw(a_addr + (kch + 2 * kk) * TC_M * 16, 128, TC_M * 16);
      const uint32_t wk = w_addr + kk * 2 * 2 * 3 * NS * 16;           // [hi, lo][2][3 NS][8]
      const uint32_t acc = (kb > 0 || kk > 0) ? 1u : 0u;
      // group g: rows [g NS, (g + 1) NS) of the slice's units (0 q, 1 kv, 2 a); hi part, then lo part 3 NS rows on
      const uint64_t b_hi = wgmma_desc_nosw(wk, 128, 3 * NS * 16);
      const uint64_t b_lo = wgmma_desc_nosw(wk + 2 * 3 * NS * 16, 128, 3 * NS * 16);
      constexpr uint64_t G = (uint64_t)(NS * 16) >> 4;   // descriptor start-address step of one group
      if constexpr (PASS2) {
        wgmma_ss<NS>(dq, a_hi, b_hi, acc);
        wgmma_ss<NS>(dq, a_lo, b_hi, 1u);
        wgmma_ss<NS>(dq, a_hi, b_lo, 1u);
      }
      wgmma_ss<NS>(dk, a_hi, b_hi + G, acc);
      wgmma_ss<NS>(dk, a_lo, b_hi + G, 1u);
      wgmma_ss<NS>(dk, a_hi, b_lo + G, 1u);
      wgmma_ss<NS>(da, a_hi, b_hi + 2 * G, acc);
      wgmma_ss<NS>(da, a_lo, b_hi + 2 * G, 1u);
      wgmma_ss<NS>(da, a_hi, b_lo + 2 * G, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dq);
    wgmma_fence_acc(dk);
    wgmma_fence_acc(da);
    __syncthreads();   // every wgmma of this block has read sA / sW
  }

  // epilogue: accumulators -> sP [3][64][NS + 1]; d[4 j + 2 h + c] = D[16 w + l / 4 + 8 h][8 j + 2 (l % 4) + c]
  {
    const int w = tid >> 5, l = tid & 31;
#pragma unroll
    for (int j = 0; j < NS / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int row = 16 * w + l / 4 + 8 * h, col = 8 * j + 2 * (l % 4) + c;
          if (PASS2) sP[row * (NS + 1) + col] = dq[4 * j + 2 * h + c];
          sP[(TC_M + row) * (NS + 1) + col] = dk[4 * j + 2 * h + c];
          sP[(2 * TC_M + row) * (NS + 1) + col] = da[4 * j + 2 * h + c];
        }
  }
  if (tid < TC_M) {
    float s = 0.f;
    for (int g = 0; g < nch; ++g) s += sSq[g * TC_M + tid];
    sRn[tid] = rsqrtf(fmaxf(s, 1e-24f));
  }
  __syncthreads();

  const float* sK = sP + TC_M * (NS + 1);
  const float* sAg = sP + 2 * TC_M * (NS + 1);
  const int c = tid % NS, sub = tid / NS;
  {  // (A, H) of this thread's sub-chunk from a zero state
    float A = 1.f, H = 0.f;
    const int e = min(n, (sub + 1) * LEN);
    for (int t = sub * LEN; t < e; ++t) {
      const float g = sigmoidf_(sAg[t * (NS + 1) + c] * sRn[t]);
      H = fmaf(g, H, sK[t * (NS + 1) + c] * sRn[t]);
      A *= g;
    }
    sSubA[sub * NS + c] = A;
    sSubH[sub * NS + c] = H;
  }
  __syncthreads();
  if (!PASS2) {
    if (sub == 0) {
      float A = 1.f, H = 0.f;
      for (int s2 = 0; s2 < NSUB; ++s2) {
        H = fmaf(sSubA[s2 * NS + c], H, sSubH[s2 * NS + c]);
        A *= sSubA[s2 * NS + c];
      }
      const size_t o = ((size_t)b * p.ntiles + tile) * p.C + c0 + c;
      p.agg_a[o] = A;
      p.agg_h[o] = H;
    }
    return;
  }
  float h = p.carry ? __ldg(p.carry + ((size_t)b * p.ntiles + tile) * p.C + c0 + c) : 0.f;
  for (int s2 = 0; s2 < sub; ++s2) h = fmaf(sSubA[s2 * NS + c], h, sSubH[s2 * NS + c]);
  const int e = min(n, (sub + 1) * LEN);
  for (int t = sub * LEN; t < e; ++t) {
    const float g = sigmoidf_(sAg[t * (NS + 1) + c] * sRn[t]);
    h = fmaf(g, h, sK[t * (NS + 1) + c] * sRn[t]);
    const float q = sP[t * (NS + 1) + c] * sRn[t];
    sU[t * (NS + 1) + c] = fmaf(q, h, 2.f * sU[t * (NS + 1) + c]);   // each (t, c) is this thread's alone
  }
  __syncthreads();
  // y of the slice -> C8S: chunk (c0 / 8 + g) hi and lo, rows [t0, t0 + n)
  __nv_bfloat16* yb = p.y + (size_t)b * 2 * nch * p.T * 8;
  for (int i = tid; i < (NS / 8) * n; i += 128) {
    const int g = i / n, t = i - g * n;
    uint4 hv, lv;
    __nv_bfloat162* h2 = reinterpret_cast<__nv_bfloat162*>(&hv);
    __nv_bfloat162* l2 = reinterpret_cast<__nv_bfloat162*>(&lv);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float v0 = sU[t * (NS + 1) + 8 * g + 2 * j], v1 = sU[t * (NS + 1) + 8 * g + 2 * j + 1];
      const __nv_bfloat16 a0 = __float2bfloat16_rn(v0), a1 = __float2bfloat16_rn(v1);
      h2[j] = __halves2bfloat162(a0, a1);
      l2[j] = __halves2bfloat162(__float2bfloat16_rn(v0 - __bfloat162float(a0)),
                                 __float2bfloat16_rn(v1 - __bfloat162float(a1)));
    }
    *reinterpret_cast<uint4*>(yb + ((size_t)(c0 / 8 + g) * p.T + t0 + t) * 8) = hv;
    *reinterpret_cast<uint4*>(yb + ((size_t)(nch + c0 / 8 + g) * p.T + t0 + t) * 8) = lv;
  }
}

template <int NS>
static int run_tc(TcParams p, int B, cudaStream_t stream) {
  auto k1 = proj_scan_tc_kernel<NS, false>;
  auto k2 = proj_scan_tc_kernel<NS, true>;
  const int smem = TcCfg<NS>::smem(p.C);
  static int attr = 0;
  if (smem > attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ALM_CUDA_OK(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = smem;
  }
  const dim3 grid(p.C / NS, p.ntiles, B);
  if (p.ntiles > 1) {
    k1<<<grid, 128, smem, stream>>>(p);
    ALM_CHECK_LAUNCH();
    carry_kernel<<<ceil_div(B * p.C, THREADS), THREADS, 0, stream>>>(p.agg_a, p.agg_h, const_cast<float*>(p.carry),
                                                                   B, p.C, p.ntiles);
    ALM_CHECK_LAUNCH();
    ALM_LAUNCHED(2);
  } else {
    p.carry = nullptr;
  }
  k2<<<grid, 128, smem, stream>>>(p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

}  // namespace gl

extern "C" long long alm_codec_gate_loop_workspace(int B, int C, int T, int tc) {
  if (B <= 0 || C <= 0 || T <= 0) return 0;
  const int tt = tc ? gl::TC_M : gl::tile_steps(C);
  const long long ntiles = (T + tt - 1) / tt;
  return ntiles > 1 ? 3LL * B * ntiles * C : 0;
}

extern "C" int alm_codec_gate_loop_fp32(const float* x, const float* proj, float* y, float* workspace, int B, int C,
                                        int T, alm_stream_t stream_) {
  ALM_REQUIRE(x && proj && y && B > 0 && C > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(C <= 1024, ALM_ERR_UNSUPPORTED);
  gl::Params p;
  p.x = x; p.proj = proj; p.y = y;
  p.B = B; p.C = C; p.T = T;
  p.tt = gl::tile_steps(C);
  p.ntiles = ceil_div(T, p.tt);
  p.nsub = C >= gl::THREADS ? 1 : gl::THREADS / C;
  if (p.nsub > p.tt) p.nsub = p.tt;
  const size_t per = (size_t)B * p.ntiles * C;
  p.agg_a = workspace; p.agg_h = workspace + per; p.carry = workspace + 2 * per;
  ALM_REQUIRE(p.ntiles == 1 || workspace, ALM_ERR_ARG);
  return gl::run_fp32(p, reinterpret_cast<cudaStream_t>(stream_));
}

extern "C" int alm_codec_gate_loop_tc(const void* x, const void* w_units, void* y, float* workspace, int B, int C,
                                      int T, alm_stream_t stream_) {
  ALM_REQUIRE(x && w_units && y && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(C == 32 || C == 64 || C == 128 || C == 256 || C == 512, ALM_ERR_UNSUPPORTED);
  gl::TcParams p;
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.w = reinterpret_cast<const __nv_bfloat16*>(w_units);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.C = C; p.T = T;
  p.ntiles = ceil_div(T, gl::TC_M);
  const size_t per = (size_t)B * p.ntiles * C;
  p.agg_a = workspace; p.agg_h = workspace + per; p.carry = workspace + 2 * per;
  ALM_REQUIRE(p.ntiles == 1 || workspace, ALM_ERR_ARG);
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  return C == 32 ? gl::run_tc<32>(p, B, stream) : gl::run_tc<64>(p, B, stream);
}

}  // namespace alm
