// Hyper-Connections forward, second generation (d <= 1024): 2 warps per token and 4 tokens per CTA for S <= 4, 4
// warps per token and 2 tokens per CTA for S = 5..8; no CTA-wide barrier.  (The first generation in hyper_conn.cuh
// uses one CTA per token with 5-6 __syncthreads per token and runs far off the HBM roofline.)  The backward is
// hyper_conn_ring.cuh (S <= 4) and hyper_conn_ring_wide.cuh (S >= 5).
//
//  - a token's TPT threads each own NCH chunks of 8 channels (16-B vector loads, fully coalesced);
//  - reductions: warp shuffle + one 64-thread named barrier (bar.sync id, 64) through a tiny smem mailbox;
//  - per-channel parameters live in shared memory (fp32).
#pragma once
#include "alm_common.cuh"

namespace alm {
namespace hc2 {

constexpr int THREADS = 256;      // a CTA holds THREADS / TPT token slots; TPT = threads per token (64 or 128)
// floats per warp row of the reduction mailbox: the largest reduction has S * (S + 3) values (32 at S = 4)
__host__ __device__ constexpr int mailw(int S) { return S * (S + 3) <= 32 ? 32 : (S * (S + 3) + 3) / 4 * 4; }
// Per-token aux row for S streams (T = S + 1 map columns):
//   ta[S*T] tb[S] inv[S] z[S*T + S] (pre-tanh) pad mean rstd
// rounded up to 4 floats so that the backward stages a row with one bulk copy (S = 4: 56 floats, 224-B rows)
__host__ __device__ constexpr int aux_floats(int S) { return (2 * S * (S + 1) + 3 * S + 4 + 3) / 4 * 4; }
__host__ __device__ constexpr int z_offset(int S) { return S * (S + 1) + 2 * S; }
__host__ __device__ constexpr int z_end(int S) { return 2 * S * (S + 1) + 3 * S; }
static_assert(aux_floats(4) == 56, "the 4-stream aux row is 56 floats");

template <int TPT>
__device__ __forceinline__ void bar_slot(int id) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(TPT) : "memory");
}

// sum N values over the TPT threads of a token slot; all of them get the result.
template <int N, int TPT, int MAILW>
__device__ __forceinline__ void slot_sum(float (&v)[N], float* mail /*[2][TPT/32][MAILW]*/, int& which, int w2, int lane,
                                         int bar_id) {
  constexpr int WPT = TPT / 32;
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
  float* b = mail + which * (WPT * MAILW);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) b[w2 * MAILW + i] = v[i];
  }
  bar_slot<TPT>(bar_id);
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float a = b[i];
#pragma unroll
    for (int w = 1; w < WPT; ++w) a += b[w * MAILW + i];
    v[i] = a;
  }
  which ^= 1;
}

__device__ __forceinline__ void unpack8(const uint4& u, float* f) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint32_t pk(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  return make_uint4(pk(f[0], f[1]), pk(f[2], f[3]), pk(f[4], f[5]), pk(f[6], f[7]));
}

__device__ __forceinline__ void prefetch_l2(const void* p) {
  asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
}

__device__ __forceinline__ void lds4(const float* p, float* f) {
  const float4 v = *reinterpret_cast<const float4*>(p);
  f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
}
__device__ __forceinline__ float tanh_fast(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));  // MUFU.TANH, rel. err ~2^-11: far below the bf16 noise floor
  return y;
}

struct Params {
  const float* gamma_hc;      // [d]      RMSNorm gain (applied as gamma + 1)
  const float* dyn_alpha;     // [d, S+1]
  const float* dyn_beta;      // [d]
  const float* static_alpha;  // [S, S+1]
  const float* static_beta;   // [S]
  const float* alpha_scale;   // scalar
  const float* beta_scale;    // scalar
  const float* ln_gamma;      // [d] LayerNorm gain of the branch's pre-norm
};
struct Grads {  // fp32 accumulators (atomicAdd), same shapes as Params
  float* gamma_hc; float* dyn_alpha; float* dyn_beta; float* static_alpha; float* static_beta;
  float* alpha_scale; float* beta_scale; float* ln_gamma;
};

// smem: [0,d) g1 = (gamma+1)*sqrt(d); [d,2d) dyn_beta; [2d,3d) ln_gamma; [3d, (3+T)d) dyn_alpha transposed [T][d]
template <int T>
__device__ __forceinline__ void stage_params(float* sm, const Params& p, int d) {
  const float sqrt_d = sqrtf((float)d);
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    sm[i] = (p.gamma_hc[i] + 1.f) * sqrt_d;
    sm[d + i] = p.dyn_beta[i];
    sm[2 * d + i] = p.ln_gamma[i];
#pragma unroll
    for (int t = 0; t < T; ++t) sm[(3 + t) * d + i] = p.dyn_alpha[(size_t)i * T + t];
  }
}

// ------------------------------------------------------------------------------------------------
template <int S, int NCH, int TPT>
__global__ void __launch_bounds__(THREADS, S <= 4 ? 2 : 1)
pre_fwd_kernel(const __nv_bfloat16* __restrict__ R_in, const __nv_bfloat16* __restrict__ Y,
               const float* __restrict__ beta_prev, const float* __restrict__ x_expand, Params prm,
               __nv_bfloat16* __restrict__ R_out, __nv_bfloat16* __restrict__ bin, __nv_bfloat16* __restrict__ xn,
               float* __restrict__ beta_out, float* __restrict__ aux, int M, int d) {
  extern __shared__ float sm[];
  constexpr int T = S + 1, AUX = aux_floats(S), MAILW = mailw(S);
  constexpr int TOK = THREADS / TPT, WPT = TPT / 32;
  float* mailbox = sm + (3 + T) * d;  // [TOK][2][WPT][MAILW]
  stage_params<T>(sm, prm, d);
  __syncthreads();
  const float* sG1 = sm;
  const float* sBf = sm + d;
  const float* sLn = sm + 2 * d;
  const float* sA = sm + 3 * d;
  const int slot = threadIdx.x / TPT, lt = threadIdx.x % TPT, w2 = lt >> 5, lane = lt & 31;
  float* mail = mailbox + slot * (2 * WPT * MAILW);
  int which = 0;
  const int bar_id = 1 + slot;
  const float a_scale = *prm.alpha_scale, b_scale = *prm.beta_scale;
  float Astat[S][T], Bstat[S];
#pragma unroll
  for (int s = 0; s < S; ++s) {
    Bstat[s] = prm.static_beta[s];
#pragma unroll
    for (int t = 0; t < T; ++t) Astat[s][t] = prm.static_alpha[s * T + t];
  }
  int ch[NCH];
  bool act[NCH];
#pragma unroll
  for (int k = 0; k < NCH; ++k) { ch[k] = (lt + TPT * k) * 8; act[k] = ch[k] < d; }

  for (int m = blockIdx.x * TOK + slot; m < M; m += gridDim.x * TOK) {
    {  // pull the next token of this slot towards L2 while this one is processed (one lane per 128-B line)
      const int mn = m + gridDim.x * TOK;
      if (mn < M && (lt & 7) == 0) {
#pragma unroll
        for (int k = 0; k < NCH; ++k)
          if (act[k]) {
            if (x_expand != nullptr) {
              prefetch_l2(x_expand + (size_t)mn * d + ch[k]);
              prefetch_l2(x_expand + (size_t)mn * d + ch[k] + 32);
            } else {
              prefetch_l2(Y + (size_t)mn * d + ch[k]);
#pragma unroll
              for (int s = 0; s < S; ++s) prefetch_l2(R_in + ((size_t)mn * S + s) * d + ch[k]);
            }
          }
      }
    }
    float R[S][NCH][8];
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      if (act[k]) {
        if (x_expand != nullptr) {
          const float4 a = *reinterpret_cast<const float4*>(x_expand + (size_t)m * d + ch[k]);
          const float4 b = *reinterpret_cast<const float4*>(x_expand + (size_t)m * d + ch[k] + 4);
          const float xv[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
          for (int s = 0; s < S; ++s)
#pragma unroll
            for (int e = 0; e < 8; ++e) R[s][k][e] = xv[e];
        } else {
          float yv[8];
          unpack8(*reinterpret_cast<const uint4*>(Y + (size_t)m * d + ch[k]), yv);
#pragma unroll
          for (int s = 0; s < S; ++s) {
            float rv[8];
            unpack8(*reinterpret_cast<const uint4*>(R_in + ((size_t)m * S + s) * d + ch[k]), rv);
            const float bp = beta_prev[(size_t)m * S + s];
#pragma unroll
            for (int e = 0; e < 8; ++e) R[s][k][e] = fmaf(bp, yv[e], rv[e]);
          }
        }
      } else {
#pragma unroll
        for (int s = 0; s < S; ++s)
#pragma unroll
          for (int e = 0; e < 8; ++e) R[s][k][e] = 0.f;
      }
    }
    // ONE reduction for the stream norms and every dynamic-map dot product: the dots are taken on the raw residual
    // (z[s][c] = inv_s * sum_d R_s[d] g1[d] P_c[d]) so they do not have to wait for inv_s
    float w[S * T + S + S];  // [0, S*T+S): raw dots, then S sums of squares
#pragma unroll
    for (int i = 0; i < S * T + S + S; ++i) w[i] = 0.f;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      if (act[k]) {
#pragma unroll
        for (int h4 = 0; h4 < 2; ++h4) {  // 4 channels at a time: 16-B shared loads, no bank-conflict replays
          const int c = ch[k] + h4 * 4;
          float g1[4], bf[4], av[T][4];
          lds4(sG1 + c, g1);
          lds4(sBf + c, bf);
#pragma unroll
          for (int t = 0; t < T; ++t) lds4(sA + t * d + c, av[t]);
#pragma unroll
          for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int s = 0; s < S; ++s) {
              const float rv = R[s][k][h4 * 4 + e];
              const float nv = rv * g1[e];
              w[S * T + S + s] = fmaf(rv, rv, w[S * T + S + s]);
#pragma unroll
              for (int t = 0; t < T; ++t) w[s * T + t] = fmaf(nv, av[t][e], w[s * T + t]);
              w[S * T + s] = fmaf(nv, bf[e], w[S * T + s]);
            }
        }
      }
    }
    slot_sum<S * T + S + S, TPT, MAILW>(w, mail, which, w2, lane, bar_id);
    float inv[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
      inv[s] = 1.f / fmaxf(sqrtf(w[S * T + S + s]), 1e-12f);
#pragma unroll
      for (int t = 0; t < T; ++t) w[s * T + t] *= inv[s];
      w[S * T + s] *= inv[s];
    }
    if (lt == 0) {  // pre-activations: the ring backward's RMS-norm term needs them (hyper_conn_ring.cuh)
      float* az = aux + (size_t)m * AUX + z_offset(S);
#pragma unroll
      for (int i = 0; i < S * T + S; ++i) az[i] = w[i];
    }
    float alpha[S][T], beta[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
#pragma unroll
      for (int t = 0; t < T; ++t) {
        w[s * T + t] = tanh_fast(w[s * T + t]);
        alpha[s][t] = fmaf(w[s * T + t], a_scale, Astat[s][t]);
      }
      w[S * T + s] = tanh_fast(w[S * T + s]);
      beta[s] = fmaf(w[S * T + s], b_scale, Bstat[s]);
    }
    // mixed residual streams out; branch input kept for the LayerNorm
    float bi[NCH][8];
    float st[2] = {0.f, 0.f};  // sum, sum of squares of the branch input (LayerNorm statistics in one reduction)
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float a = 0.f;
#pragma unroll
        for (int s = 0; s < S; ++s) a = fmaf(alpha[s][0], R[s][k][e], a);
        bi[k][e] = a;
        st[0] += a;
        st[1] = fmaf(a, a, st[1]);
      }
      if (act[k]) {
#pragma unroll
        for (int t = 1; t < T; ++t) {
          float o[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            float a = 0.f;
#pragma unroll
            for (int s = 0; s < S; ++s) a = fmaf(alpha[s][t], R[s][k][e], a);
            o[e] = a;
          }
          *reinterpret_cast<uint4*>(R_out + ((size_t)m * S + (t - 1)) * d + ch[k]) = pack8(o);
        }
        if (bin != nullptr) *reinterpret_cast<uint4*>(bin + (size_t)m * d + ch[k]) = pack8(bi[k]);
      }
    }
    slot_sum<2, TPT, MAILW>(st, mail, which, w2, lane, bar_id);
    const float mean = st[0] / d;
    const float rstd = rsqrtf(fmaxf(st[1] / d - mean * mean, 0.f) + 1e-5f);
#pragma unroll
    for (int k = 0; k < NCH; ++k)
      if (act[k]) {
        float o[8], lg[8];
        lds4(sLn + ch[k], lg);
        lds4(sLn + ch[k] + 4, lg + 4);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = (bi[k][e] - mean) * rstd * lg[e];
        *reinterpret_cast<uint4*>(xn + (size_t)m * d + ch[k]) = pack8(o);
      }
    if (lt == 0) {
      float* a = aux + (size_t)m * AUX;
#pragma unroll
      for (int i = 0; i < S * T + S; ++i) a[i] = w[i];
#pragma unroll
      for (int s = 0; s < S; ++s) {
        a[S * T + S + s] = inv[s];
        beta_out[(size_t)m * S + s] = beta[s];
      }
#pragma unroll
      for (int i = z_end(S); i < AUX - 2; ++i) a[i] = 0.f;  // pad: the row is copied whole, so it is written
      a[AUX - 2] = mean;
      a[AUX - 1] = rstd;
    }
  }
}

inline size_t fwd_smem(int S, int d, int tpt) {
  return (size_t)((4 + S) * d + (THREADS / tpt) * 2 * (tpt / 32) * mailw(S)) * sizeof(float);
}

}  // namespace hc2
}  // namespace alm
