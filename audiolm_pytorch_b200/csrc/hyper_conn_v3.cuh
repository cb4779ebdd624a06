// Hyper-Connections backward, third generation (depth(prev) + width + pre-LayerNorm backward of one branch).
//
// hc2::pre_bwd_kernel held a token's 16 channels x 10 arrays in registers (255 regs) and the per-channel
// parameter-gradient accumulators in 128 KB of shared memory: 8 warps per SM, too few to hide global-load latency.
// This version
//   * streams the token twice in 4-channel pieces (pass 1: every per-token dot product in ONE reduction,
//     pass 2: gradients; the second read hits L1/L2), so it fits 128 registers -> 2 CTAs (16 warps) per SM;
//   * uses the forward's pre-activations z (kept in aux) so that the RMS-norm backward needs no reduction:
//       sum_d u_s[d] R_s[d] = (1/inv_s) * sum_c dz[s][c] z[s][c];
//   * moves the per-channel parameter gradients (dyn_alpha, dyn_beta, gamma) out of the kernel: it emits
//     W[t,s,c] = inv_s * dz[s][c] and the caller forms G[d,c] = sum_{t,s} R[t,s,d] W[t,s,c] with two skinny
//     wgmma GEMMs (R = R_in + beta_prev (x) Y), finished by hc_param_finish_kernel.
// Reference semantics: hyper_connections.HyperConnections width/depth connections as called from
// audiolm_pytorch.py:446-454, 524-551 (third-party dependency, restated in oracle/third_party.py).
#pragma once
#include "hyper_conn_v2.cuh"

namespace alm {
namespace hc3 {

using hc2::AUX;
using hc2::S;
using hc2::T;
constexpr int THREADS = 256, TPT = 64, TOK = THREADS / TPT, WPT = TPT / 32;
constexpr int NRED = 34;    // pass-1 per-token sums
constexpr int MAILW = 40;   // floats per warp row of the reduction mailbox
constexpr int COEF = 16;    // per-stream coefficient row: alpha[5], C[6], kk, beta_prev, pad[3]
constexpr int NSMALL = 32;  // static_alpha[20], static_beta[4], alpha_scale, beta_scale partial sums per slot
constexpr int Z_OFF = S * T + S + S;  // aux: ta[20] tb[4] inv[4] z[24] mean rstd

template <int N>
__device__ __forceinline__ void slot_sum(float (&v)[N], float* mail /*[2][WPT][MAILW]*/, int& which, int w2, int lane,
                                         int bar_id) {
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
  float* b = mail + which * (WPT * MAILW);
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) b[w2 * MAILW + i] = v[i];
  }
  hc2::bar_slot<TPT>(bar_id);
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = b[i] + b[MAILW + i];
  which ^= 1;
}

// fp32 channel pairs (two IEEE fp32 operations each; sm_90 has no packed f32x2 arithmetic)
__device__ __forceinline__ float2 dup2(float a) { return make_float2(a, a); }
__device__ __forceinline__ float2 fma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 add2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 mul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ void unpack4p(const uint2& u, float2* f) {  // 4 bf16 -> two (even, odd) channel pairs
  f[0] = make_float2(bf16_lo(u.x), bf16_hi(u.x));
  f[1] = make_float2(bf16_lo(u.y), bf16_hi(u.y));
}
__device__ __forceinline__ uint2 pack4p(const float2* f) {
  return make_uint2(hc2::pk(f[0].x, f[0].y), hc2::pk(f[1].x, f[1].y));
}

__device__ __forceinline__ void unpack4(const uint2& u, float* f) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
}
__device__ __forceinline__ uint2 pack4(const float* f) { return make_uint2(hc2::pk(f[0], f[1]), hc2::pk(f[2], f[3])); }
__device__ __forceinline__ uint2 ldg8(const __nv_bfloat16* p) { return __ldg(reinterpret_cast<const uint2*>(p)); }

inline size_t bwd_smem(int d) {
  return (size_t)(11 * d + TOK * 2 * WPT * MAILW + TOK * S * COEF + TOK * NSMALL) * sizeof(float);
}

// NCH = ceil(d / 256): a token's 64 threads each own NCH pieces of 4 channels (8-B loads, 256 B per warp).
template <int NCH>
__global__ void __launch_bounds__(THREADS, 2)
pre_bwd_kernel(const __nv_bfloat16* __restrict__ R_in, const __nv_bfloat16* __restrict__ Y,
               const float* __restrict__ beta_prev, hc2::Params prm, const float* __restrict__ aux,
               const __nv_bfloat16* __restrict__ dR_out, const __nv_bfloat16* __restrict__ dxn,
               const __nv_bfloat16* __restrict__ dbin_extra, const float* __restrict__ dbeta,
               __nv_bfloat16* __restrict__ dR_in, __nv_bfloat16* __restrict__ dY, float* __restrict__ dbeta_prev,
               __nv_bfloat16* __restrict__ Wout /*[M*S, 8]*/, __nv_bfloat16* __restrict__ WYout /*[M, 8]*/,
               hc2::Grads gr, int M, int d) {
  extern __shared__ float sm[];
  float* sLn = sm;                    // [d]     ln_gamma
  float* sPg = sm + d;                // [6][d]  g1 * (dyn_alpha[:,0..4], dyn_beta),  g1 = (gamma + 1) * sqrt(d)
  float* sGlnAll = sm + 7 * d;        // [TOK][d] private d(ln_gamma) accumulators
  float* mailbox = sm + 11 * d;       // [TOK][2][WPT][MAILW]
  float* sCoefAll = mailbox + TOK * 2 * WPT * MAILW;  // [TOK][S][COEF]
  float* sSmallAll = sCoefAll + TOK * S * COEF;       // [TOK][NSMALL]
  {
    const float sqrt_d = sqrtf((float)d);
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
      const float g1 = (prm.gamma_hc[i] + 1.f) * sqrt_d;
      sLn[i] = prm.ln_gamma[i];
#pragma unroll
      for (int t = 0; t < T; ++t) sPg[t * d + i] = g1 * prm.dyn_alpha[(size_t)i * T + t];
      sPg[T * d + i] = g1 * prm.dyn_beta[i];
    }
    for (int i = threadIdx.x; i < TOK * d; i += blockDim.x) sGlnAll[i] = 0.f;
    for (int i = threadIdx.x; i < TOK * NSMALL; i += blockDim.x) sSmallAll[i] = 0.f;
  }
  __syncthreads();
  const int slot = threadIdx.x / TPT, lt = threadIdx.x % TPT, w2 = lt >> 5, lane = lt & 31;
  float* mail = mailbox + slot * (2 * WPT * MAILW);
  float* sCoef = sCoefAll + slot * (S * COEF);
  float* sSmall = sSmallAll + slot * NSMALL;
  float* sGln = sGlnAll + (size_t)slot * d;
  int which = 0;
  const int bar_id = 1 + slot;
  const float a_scale = *prm.alpha_scale, b_scale = *prm.beta_scale;
  const float inv_d = 1.f / (float)d;
  int ch[NCH];
  bool act[NCH];
#pragma unroll
  for (int k = 0; k < NCH; ++k) { ch[k] = (lt + TPT * k) * 4; act[k] = ch[k] < d; }

  for (int m = blockIdx.x * TOK + slot; m < M; m += gridDim.x * TOK) {
    {  // pull the next token of this slot towards L2 (one lane per 128-B line: 16 lanes x 8 B x 4 = 128 B)
      const int mn = m + gridDim.x * TOK;
      if (mn < M && (lt & 15) == 0) {
#pragma unroll
        for (int k = 0; k < NCH; ++k)
          if (act[k]) {
            hc2::prefetch_l2(Y + (size_t)mn * d + ch[k]);
            hc2::prefetch_l2(dxn + (size_t)mn * d + ch[k]);
            if (dbin_extra != nullptr) hc2::prefetch_l2(dbin_extra + (size_t)mn * d + ch[k]);
#pragma unroll
            for (int s = 0; s < S; ++s) {
              hc2::prefetch_l2(R_in + ((size_t)mn * S + s) * d + ch[k]);
              hc2::prefetch_l2(dR_out + ((size_t)mn * S + s) * d + ch[k]);
            }
          }
      }
    }
    const float* a = aux + (size_t)m * AUX;
    const float mean = a[AUX - 2], rstd = a[AUX - 1];
    float bp[S], alpha0[S];
#pragma unroll
    for (int s = 0; s < S; ++s) {
      bp[s] = beta_prev[(size_t)m * S + s];
      alpha0[s] = fmaf(a[s * T], a_scale, prm.static_alpha[s * T]);
    }
    // ---------------- pass 1: every per-token sum in one reduction ----------------
    // red: 0 sum gl | 1 sum gl*xhat | 2+s sum gl*R_s | 6+s sum R_s | 10+s sum xhat*R_s | 14+s sum ex*R_s |
    //      18+4s+(t-1) sum dR_out[t-1]*R_s      (gl = dxn * ln_gamma, xhat = normalised branch input, ex = dbin_extra)
    float2 red2[NRED];  // .x / .y: partial sums over even / odd channels (added before the reduction)
#pragma unroll
    for (int i = 0; i < NRED; ++i) red2[i] = make_float2(0.f, 0.f);
    const float2 rstd2 = dup2(rstd), nmr2 = dup2(-mean * rstd);
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      if (act[k]) {
        const size_t o1 = (size_t)m * d + ch[k];
        float2 y[2], dx[2], ex[2], r[S][2];
        unpack4p(ldg8(Y + o1), y);
        unpack4p(ldg8(dxn + o1), dx);
        if (dbin_extra != nullptr) {
          unpack4p(ldg8(dbin_extra + o1), ex);
        } else {
          ex[0] = ex[1] = make_float2(0.f, 0.f);
        }
        const float4 lg4 = *reinterpret_cast<const float4*>(sLn + ch[k]);
        const float4 ga4 = *reinterpret_cast<const float4*>(sGln + ch[k]);
        const float2 lg[2] = {make_float2(lg4.x, lg4.y), make_float2(lg4.z, lg4.w)};
        float2 gacc[2] = {make_float2(ga4.x, ga4.y), make_float2(ga4.z, ga4.w)};
#pragma unroll
        for (int s = 0; s < S; ++s) {
          float2 rv[2];
          unpack4p(ldg8(R_in + ((size_t)m * S + s) * d + ch[k]), rv);
          const float2 b2 = dup2(bp[s]);
          r[s][0] = fma2(b2, y[0], rv[0]);
          r[s][1] = fma2(b2, y[1], rv[1]);
        }
        float2 gl[2], xh[2];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          float2 bsum = make_float2(0.f, 0.f);
#pragma unroll
          for (int s = 0; s < S; ++s) bsum = fma2(dup2(alpha0[s]), r[s][h2], bsum);
          xh[h2] = fma2(bsum, rstd2, nmr2);
          gl[h2] = mul2(dx[h2], lg[h2]);
          gacc[h2] = fma2(dx[h2], xh[h2], gacc[h2]);
          red2[0] = add2(red2[0], gl[h2]);
          red2[1] = fma2(gl[h2], xh[h2], red2[1]);
        }
        *reinterpret_cast<float4*>(sGln + ch[k]) = make_float4(gacc[0].x, gacc[0].y, gacc[1].x, gacc[1].y);
#pragma unroll
        for (int s = 0; s < S; ++s)
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
            red2[2 + s] = fma2(gl[h2], r[s][h2], red2[2 + s]);
            red2[6 + s] = add2(red2[6 + s], r[s][h2]);
            red2[10 + s] = fma2(xh[h2], r[s][h2], red2[10 + s]);
            red2[14 + s] = fma2(ex[h2], r[s][h2], red2[14 + s]);
          }
#pragma unroll
        for (int t = 1; t < T; ++t) {
          float2 dm[2];
          unpack4p(ldg8(dR_out + ((size_t)m * S + (t - 1)) * d + ch[k]), dm);
#pragma unroll
          for (int s = 0; s < S; ++s)
#pragma unroll
            for (int h2 = 0; h2 < 2; ++h2)
              red2[18 + 4 * s + (t - 1)] = fma2(dm[h2], r[s][h2], red2[18 + 4 * s + (t - 1)]);
        }
      }
    }
    float red[NRED];
#pragma unroll
    for (int i = 0; i < NRED; ++i) red[i] = red2[i].x + red2[i].y;
    slot_sum<NRED>(red, mail, which, w2, lane, bar_id);
    const float m1 = red[0] * inv_d, m2 = red[1] * inv_d;
    // ---------------- per-token scalars: thread s < 4 owns stream s ----------------
    if (lt < S) {
      const int s = lt;
      // pick stream s's sums with predicated moves (a runtime index would push red[] to local memory)
      float dal[T], bps = 0.f;
#pragma unroll
      for (int t = 0; t < T; ++t) dal[t] = 0.f;
#pragma unroll
      for (int ss = 0; ss < S; ++ss)
        if (ss == s) {
          dal[0] = fmaf(rstd, red[2 + ss] - m1 * red[6 + ss] - m2 * red[10 + ss], red[14 + ss]);
#pragma unroll
          for (int t = 1; t < T; ++t) dal[t] = red[18 + 4 * ss + (t - 1)];
          bps = bp[ss];
        }
      const float inv = a[S * T + S + s];
      const float tb = a[S * T + s], zb = a[Z_OFF + S * T + s], dbe = dbeta[(size_t)m * S + s];
      const float dwb = dbe * b_scale * (1.f - tb * tb);
      float zsum = dwb * zb, ascale_acc = 0.f;
      float* c = sCoef + s * COEF;
#pragma unroll
      for (int t = 0; t < T; ++t) {
        const float ta = a[s * T + t];
        const float dw = dal[t] * a_scale * (1.f - ta * ta);
        zsum = fmaf(dw, a[Z_OFF + s * T + t], zsum);
        ascale_acc = fmaf(dal[t], ta, ascale_acc);
        c[t] = fmaf(ta, a_scale, prm.static_alpha[s * T + t]);  // alpha[s][t]
        c[T + t] = inv * dw;                                     // C[s][t]
        sSmall[s * T + t] += dal[t];                             // d static_alpha
      }
      c[2 * T] = inv * dwb;                                      // C[s][5]
      c[2 * T + 1] = inv * inv * zsum;                           // kk[s]: RMS-norm backward coefficient
      c[2 * T + 2] = bps;
      sSmall[S * T + s] += dbe;                                  // d static_beta
      sSmall[S * T + S + s] += ascale_acc;                       // d alpha_scale (per-stream partial)
      sSmall[S * T + 2 * S + s] = fmaf(dbe, tb, sSmall[S * T + 2 * S + s]);  // d beta_scale partial
      // W row of this (token, stream): the skinny GEMM's B operand
      float wrow[8];
#pragma unroll
      for (int t = 0; t < T; ++t) wrow[t] = c[T + t];
      wrow[5] = c[2 * T]; wrow[6] = 0.f; wrow[7] = 0.f;
      *reinterpret_cast<uint4*>(Wout + ((size_t)m * S + s) * 8) = hc2::pack8(wrow);
    }
    hc2::bar_slot<TPT>(bar_id);
    if (lt == 0) {
      float wy[8];
#pragma unroll
      for (int c6 = 0; c6 < 8; ++c6) wy[c6] = 0.f;
#pragma unroll
      for (int s = 0; s < S; ++s)
#pragma unroll
        for (int c6 = 0; c6 < 6; ++c6) wy[c6] = fmaf(bp[s], sCoef[s * COEF + T + c6], wy[c6]);
      *reinterpret_cast<uint4*>(WYout + (size_t)m * 8) = hc2::pack8(wy);
    }
    // ---------------- pass 2: gradients ----------------
    float2 dbp2[S];
#pragma unroll
    for (int s = 0; s < S; ++s) dbp2[s] = make_float2(0.f, 0.f);
    const float2 nm1 = dup2(-m1), nm2 = dup2(-m2);
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      if (act[k]) {
        const size_t o1 = (size_t)m * d + ch[k];
        float2 y[2], r[S][2], dm[T][2], dy[2];
        unpack4p(ldg8(Y + o1), y);
#pragma unroll
        for (int s = 0; s < S; ++s) {
          float2 rv[2];
          unpack4p(ldg8(R_in + ((size_t)m * S + s) * d + ch[k]), rv);
          const float2 b2 = dup2(bp[s]);
          r[s][0] = fma2(b2, y[0], rv[0]);
          r[s][1] = fma2(b2, y[1], rv[1]);
        }
        {
          float2 dx[2], ex[2];
          unpack4p(ldg8(dxn + o1), dx);
          if (dbin_extra != nullptr) {
            unpack4p(ldg8(dbin_extra + o1), ex);
          } else {
            ex[0] = ex[1] = make_float2(0.f, 0.f);
          }
          const float4 lg4 = *reinterpret_cast<const float4*>(sLn + ch[k]);
          const float2 lg[2] = {make_float2(lg4.x, lg4.y), make_float2(lg4.z, lg4.w)};
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
            float2 bsum = make_float2(0.f, 0.f);
#pragma unroll
            for (int s = 0; s < S; ++s) bsum = fma2(dup2(alpha0[s]), r[s][h2], bsum);
            const float2 xhat = fma2(bsum, rstd2, nmr2);
            // d(branch input) = rstd * (dxn*ln_gamma - m1 - xhat*m2) + dbin_extra
            const float2 inner = fma2(xhat, nm2, fma2(dx[h2], lg[h2], nm1));
            dm[0][h2] = fma2(rstd2, inner, ex[h2]);
            dy[h2] = make_float2(0.f, 0.f);
          }
        }
#pragma unroll
        for (int t = 1; t < T; ++t) unpack4p(ldg8(dR_out + ((size_t)m * S + (t - 1)) * d + ch[k]), dm[t]);
        float2 pg[6][2];
#pragma unroll
        for (int c6 = 0; c6 < 6; ++c6) {
          const float4 p4 = *reinterpret_cast<const float4*>(sPg + c6 * d + ch[k]);
          pg[c6][0] = make_float2(p4.x, p4.y);
          pg[c6][1] = make_float2(p4.z, p4.w);
        }
#pragma unroll
        for (int s = 0; s < S; ++s) {
          float cf[COEF];
#pragma unroll
          for (int q = 0; q < 3; ++q) hc2::lds4(sCoef + s * COEF + q * 4, cf + q * 4);
          const float2 nkk = dup2(-cf[2 * T + 1]), bps2 = dup2(bp[s]);
          float2 dr[2];
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
            float2 acc = mul2(r[s][h2], nkk);
#pragma unroll
            for (int t = 0; t < T; ++t) acc = fma2(dup2(cf[t]), dm[t][h2], acc);
#pragma unroll
            for (int c6 = 0; c6 < 6; ++c6) acc = fma2(dup2(cf[T + c6]), pg[c6][h2], acc);
            dr[h2] = acc;
            dbp2[s] = fma2(acc, y[h2], dbp2[s]);
            dy[h2] = fma2(bps2, acc, dy[h2]);
          }
          *reinterpret_cast<uint2*>(dR_in + ((size_t)m * S + s) * d + ch[k]) = pack4p(dr);
        }
        *reinterpret_cast<uint2*>(dY + o1) = pack4p(dy);
      }
    }
    float dbp[S];
#pragma unroll
    for (int s = 0; s < S; ++s) dbp[s] = dbp2[s].x + dbp2[s].y;
    slot_sum<S>(dbp, mail, which, w2, lane, bar_id);
    if (lt == 0) {
#pragma unroll
      for (int s = 0; s < S; ++s) dbeta_prev[(size_t)m * S + s] = dbp[s];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float acc = 0.f;
#pragma unroll
    for (int sl = 0; sl < TOK; ++sl) acc += sGlnAll[(size_t)sl * d + i];
    atomicAdd(gr.ln_gamma + i, acc);
  }
  if (threadIdx.x < S * T + S + 2) {
    const int i = threadIdx.x;
    float acc = 0.f;
    if (i < S * T + S) {
#pragma unroll
      for (int sl = 0; sl < TOK; ++sl) acc += sSmallAll[sl * NSMALL + i];
      atomicAdd((i < S * T ? gr.static_alpha + i : gr.static_beta + (i - S * T)), acc);
    } else {
      const int base = (i == S * T + S) ? S * T + S : S * T + 2 * S;
#pragma unroll
      for (int sl = 0; sl < TOK; ++sl)
#pragma unroll
        for (int s = 0; s < S; ++s) acc += sSmallAll[sl * NSMALL + base + s];
      atomicAdd(i == S * T + S ? gr.alpha_scale : gr.beta_scale, acc);
    }
  }
}

// G [d, 8] fp32 = sum_{t,s} R[t,s,:] (x) W[t,s,:]  ->  gradients of the per-channel hyper-connection parameters
__global__ void hc_param_finish_kernel(const float* __restrict__ G, hc2::Params prm, hc2::Grads gr, int d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= d) return;
  const float sqrt_d = sqrtf((float)d);
  const float g1 = (prm.gamma_hc[i] + 1.f) * sqrt_d;
  float acc = G[(size_t)i * 8 + T] * prm.dyn_beta[i];
  gr.dyn_beta[i] += g1 * G[(size_t)i * 8 + T];
#pragma unroll
  for (int t = 0; t < T; ++t) {
    const float g = G[(size_t)i * 8 + t];
    acc = fmaf(g, prm.dyn_alpha[(size_t)i * T + t], acc);
    gr.dyn_alpha[(size_t)i * T + t] += g1 * g;
  }
  gr.gamma_hc[i] += sqrt_d * acc;
}

}  // namespace hc3
}  // namespace alm
