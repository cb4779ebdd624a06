// Hyper-Connections backward for d <= 1024 (depth(prev) + width + pre-LayerNorm backward of one branch), with every
// parameter gradient formed in the kernel.
//
// One persistent CTA per SM with NC warpgroups; warpgroup c takes every NC-th token of the CTA.  Each warpgroup owns a
// ring of NSC shared-memory stages, one token each, filled with 1-D bulk copies (cp.async.bulk completing on a full
// mbarrier): the token's aux / dbeta / beta_prev scalars, R_in and dR_out [S, d], Y, dxn and dbin_extra [d] (x [d]
// fp32 instead of R_in and Y when the op expanded the streams).  While it computes one token, the next NSC - 1 are in
// flight; a stage is refilled by the warpgroup itself once its reduction barrier shows that every thread is done with
// the stage.  (There is no producer warp: a ninth warp per SM would cap every thread at 168 registers, 3 warps x 168
// x 32 per quarter-SM register file, and the consumers need ~220.)  Thread l owns channels [8l, 8l + 8) of every
// row, so the per-channel parameter gradients (gamma, dyn_alpha, dyn_beta, ln_gamma) stay in its registers for the
// whole launch and are flushed once.  Per token:
//   pass 1   every per-token dot product (2 + 4S + S^2 sums, 34 at S = 4) from the stage, one warpgroup reduction;
//   scalars  warp 0, one lane per (stream s, map column c): the tanh and RMS-norm backward coefficients;
//   pass 2   dR_in, dY (or dx) and the parameter-gradient accumulators, again from the stage.
// The RMS-norm backward needs no second reduction: with the forward's pre-activations z (kept in aux),
//   sum_d u_s[d] R_s[d] = (1 / inv_s) * sum_c dz[s][c] z[s][c],
// and with C[s][c] = inv_s * dz[s][c] the per-channel map gradient is G[d][c] = sum_tokens sum_s R_s[d] C[s][c].
// Reference semantics: hyper_connections.HyperConnections width/depth connections as called from
// audiolm_pytorch.py:446-454, 524-551 (third-party dependency, restated in oracle/third_party.py).
#pragma once
#include "hyper_conn_v2.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace hcr {

constexpr int NC = 2;                   // warpgroups
constexpr int NSC = 3;                  // ring stages per warpgroup (one token each)
constexpr int NST = NC * NSC;
constexpr int THREADS = NC * 128;
constexpr int NRED = 34;                // pass-1 per-token sums, zero-padded: 2 + 4S + S*S <= 34 for S <= 4
constexpr int MAILW = 36;               // floats per warp row of the reduction mailbox
constexpr int COEF = 16;                // per-stream coefficient row: alpha[T], C[S + 2], kk, pad
// The ring is built for S <= 4 streams: pass 1 then fits one reduce_scatter32 and warp 0's scalar phase one lane per
// (stream, column) pair.
__host__ __device__ constexpr bool ring_ok(int S) { return S >= 2 && S <= 4; }
// Stage head: aux[AUX] then dbeta[S] and beta_prev[S] (fp32), 16-B aligned.  A bulk copy needs 16-B sizes and
// addresses, so the [M, S] rows are staged only when S % 4 == 0; otherwise the kernel reads them from global memory.
__host__ __device__ constexpr bool head_bulk(int S) { return S % 4 == 0; }
__host__ __device__ constexpr int scal_bytes(int S) { return hc2::aux_floats(S) * 4 + (head_bulk(S) ? 8 * S : 0); }
static_assert(scal_bytes(4) == 256, "the 4-stream stage head is 256 B");
static_assert(scal_bytes(2) % 16 == 0 && scal_bytes(3) % 16 == 0 && scal_bytes(4) % 16 == 0,
              "aux rows and the stage head must be 16-B multiples so that one bulk copy stages a row");

// stage: scalars | R_in [S][d] bf16 (or x [d] fp32) | dR_out [S][d] | Y [d] | dxn [d] | dbin_extra [d]
template <int S> __host__ __device__ inline int off_dr(int d) { return scal_bytes(S) + 2 * S * d; }
template <int S> __host__ __device__ inline int off_y(int d) { return scal_bytes(S) + 4 * S * d; }
template <int S> __host__ __device__ inline int off_dxn(int d) { return off_y<S>(d) + 2 * d; }
template <int S> __host__ __device__ inline int off_dbin(int d) { return off_y<S>(d) + 4 * d; }
template <int S> __host__ __device__ inline int stage_bytes(int d) {
  return (scal_bytes(S) + (4 * S + 6) * d + 127) / 128 * 128;
}
// shared memory: params [S+3][d] fp32 | mailboxes [NC][4][MAILW] | dbeta_prev partials [NC][4][S] | coefficients
// [NC][S][COEF] | full[NST] mbarriers | ring [NC][NSC] stages (128-B aligned)
template <int S> __host__ __device__ inline int ring_offset(int d) {
  return (4 * ((S + 3) * d + NC * (4 * MAILW + 4 * S + S * COEF)) + 8 * NST + 127) / 128 * 128;
}
template <int S> inline size_t smem_bytes(int d) { return (size_t)ring_offset<S>(d) + (size_t)NST * stage_bytes<S>(d); }

// the per-channel parameters are stored so that thread l's channels 8l..8l+3 and 8l+4..8l+7 are two float4 at
// [4l] and [d/2 + 4l]: a warp's 16-B loads are then contiguous (no bank-conflict replays)
__host__ __device__ inline int par_index(int c, int d) { return ((c >> 2) & 1) * (d >> 1) + (c >> 3) * 4 + (c & 3); }

// one halving step of reduce_scatter32: a lane keeps the half of v[0, 2 OFF) its lane bit OFF selects, adds the
// partner's copy of that half, and sends the other
template <int OFF>
__device__ __forceinline__ void scatter_step(float (&v)[32], int lane) {
  const bool up = (lane & OFF) != 0;
#pragma unroll
  for (int i = 0; i < OFF; ++i) {
    const float send = up ? v[i] : v[i + OFF];
    const float keep = up ? v[i + OFF] : v[i];
    v[i] = keep + __shfl_xor_sync(0xffffffffu, send, OFF);
  }
}
// sum v[i] over the warp's 32 lanes for all i < 32; lane i returns the total of v[i] (31 shuffles instead of 160)
__device__ __forceinline__ float reduce_scatter32(float (&v)[32], int lane) {
  scatter_step<16>(v, lane);
  scatter_step<8>(v, lane);
  scatter_step<4>(v, lane);
  scatter_step<2>(v, lane);
  scatter_step<1>(v, lane);
  return v[0];
}

__device__ __forceinline__ void lds8(const float* p, int half, float* f) {  // 8 parameters of a thread's channels
  hc2::lds4(p, f);
  hc2::lds4(p + half, f + 4);
}

template <int S, bool EXPAND>
__global__ void __launch_bounds__(THREADS, 1)
pre_bwd_kernel(const __nv_bfloat16* __restrict__ R_in, const __nv_bfloat16* __restrict__ Y,
               const float* __restrict__ beta_prev, const float* __restrict__ x_expand, hc2::Params prm,
               const float* __restrict__ aux, const __nv_bfloat16* __restrict__ dR_out,
               const __nv_bfloat16* __restrict__ dxn, const __nv_bfloat16* __restrict__ dbin_extra,
               const float* __restrict__ dbeta, __nv_bfloat16* __restrict__ dR_in, __nv_bfloat16* __restrict__ dY,
               float* __restrict__ dbeta_prev, float* __restrict__ dx_expand, float dx_scale, hc2::Grads gr, int M,
               int d) {
  static_assert(ring_ok(S), "the ring backward is built for 2 to 4 streams");
  constexpr int T = S + 1, AUX = hc2::aux_floats(S), Z_OFF = hc2::z_offset(S), SCAL_B = scal_bytes(S);
  constexpr int NP = S + 3;  // per-channel parameter rows: ln_gamma, g1 * dyn_alpha[:, t] (T), g1 * dyn_beta
  constexpr int NG = S + 2;  // map columns: T alpha columns and beta
  extern __shared__ __align__(128) unsigned char smem[];
  float* sPar = reinterpret_cast<float*>(smem);  // [NP][d]: ln_gamma, g1 * dyn_alpha[:, t], g1 * dyn_beta
  float* sMail = sPar + NP * d;                  // [NC][4][MAILW]
  float* sDbp = sMail + NC * 4 * MAILW;          // [NC][4][S]
  float* sCoef = sDbp + NC * 4 * S;              // [NC][S][COEF]
  uint64_t* full = reinterpret_cast<uint64_t*>(sCoef + NC * S * COEF);
  unsigned char* ring = smem + ring_offset<S>(d);
  const int stage_b = stage_bytes<S>(d), half = d >> 1;
  const float sqrt_d = sqrtf((float)d);
  for (int c = threadIdx.x; c < d; c += blockDim.x) {
    const int p = par_index(c, d);
    const float g1 = (prm.gamma_hc[c] + 1.f) * sqrt_d;
    sPar[p] = prm.ln_gamma[c];
#pragma unroll
    for (int t = 0; t < T; ++t) sPar[(1 + t) * d + p] = g1 * prm.dyn_alpha[(size_t)c * T + t];
    sPar[(1 + T) * d + p] = g1 * prm.dyn_beta[c];
  }
  if (threadIdx.x == 0) {
    for (int i = 0; i < NST; ++i) mbar_init(&full[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, lt = threadIdx.x & 127;
  const int cw = warp >> 2, w = lt >> 5;
  const bool act = lt * 8 < d;  // this thread owns channels
  const bool has_dbin = dbin_extra != nullptr;
  uint64_t* my_full = full + cw * NSC;
  unsigned char* my_ring = ring + (size_t)cw * NSC * stage_b;
  // stage the k-th token of this warpgroup into its stage k % NSC (warp 3: lane 0 arms the barrier, lanes 0-7 copy)
  auto fill = [&](int k) {
    const int m = blockIdx.x + (cw + k * NC) * gridDim.x;
    if (m >= M) return;
    const int ls = k % NSC;
    uint64_t* bar = my_full + ls;
    unsigned char* st = my_ring + (size_t)ls * stage_b;
    constexpr int head = AUX * 4 + (head_bulk(S) ? (EXPAND ? 4 * S : 8 * S) : 0);
    const uint32_t bytes = head + (EXPAND ? 4 * d : (2 * S + 2) * d) + (2 * S + 2) * d + (has_dbin ? 2 * d : 0);
    if (lane == 0) mbar_arrive_expect_tx(bar, bytes);
    __syncwarp();
    const size_t md = (size_t)m * d;
    switch (lane) {
      case 0: bulk_copy_g2s(st, aux + (size_t)m * AUX, AUX * 4, bar); break;
      case 1:
        if (head_bulk(S)) bulk_copy_g2s(st + AUX * 4, dbeta + (size_t)m * S, 4 * S, bar);
        break;
      case 2:
        if (head_bulk(S) && !EXPAND) bulk_copy_g2s(st + AUX * 4 + 4 * S, beta_prev + (size_t)m * S, 4 * S, bar);
        break;
      case 3:
        if (EXPAND) bulk_copy_g2s(st + SCAL_B, x_expand + md, 4 * d, bar);
        else bulk_copy_g2s(st + SCAL_B, R_in + md * S, 2 * S * d, bar);
        break;
      case 4: bulk_copy_g2s(st + off_dr<S>(d), dR_out + md * S, 2 * S * d, bar); break;
      case 5:
        if (!EXPAND) bulk_copy_g2s(st + off_y<S>(d), Y + md, 2 * d, bar);
        break;
      case 6: bulk_copy_g2s(st + off_dxn<S>(d), dxn + md, 2 * d, bar); break;
      case 7:
        if (has_dbin) bulk_copy_g2s(st + off_dbin<S>(d), dbin_extra + md, 2 * d, bar);
        break;
      default: break;
    }
  };
  if (w == 3) {
    for (int k = 0; k < NSC; ++k) fill(k);
  }
  {
    float G[NG][8], gLn[8];  // this thread's channels: G[c][e] = sum over its tokens of sum_s R_s C[s][c]; d ln_gamma
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      gLn[e] = 0.f;
#pragma unroll
      for (int c6 = 0; c6 < NG; ++c6) G[c6][e] = 0.f;
    }
    const int bar_id = 1 + cw;
    float* mail = sMail + cw * 4 * MAILW;
    float* dbpm = sDbp + cw * 4 * S;
    float* coef = sCoef + cw * S * COEF;
    const float a_scale = *prm.alpha_scale, b_scale = *prm.beta_scale;
    const float inv_d = 1.f / (float)d;
    float sa0[S];
#pragma unroll
    for (int s = 0; s < S; ++s) sa0[s] = prm.static_alpha[s * T];
    // scalar-phase role of warp 0's lanes: stream ss, column q (q < T: alpha column, q == T: beta, q == T + 1: kk)
    const int ss = lane >> 3, q = lane & 7;
    const bool sv = ss < S;  // (S < 4: the lanes of the missing streams stay idle)
    const float stat = sv && q < T ? prm.static_alpha[ss * T + q] : 0.f;
    float small0 = 0.f, small1 = 0.f;  // q < T: d static_alpha, d alpha_scale part; q == T: d static_beta, d beta_scale part
    const float* pLn = sPar + lt * 4;
    int ls = 0;
    uint32_t phase = 0;
    int pend = -1;  // token whose dbeta_prev partials wait in dbpm
    for (int k = 0, m = blockIdx.x + cw * gridDim.x; m < M; ++k, m += NC * gridDim.x) {
      mbar_wait(&my_full[ls], phase);
      const unsigned char* st = my_ring + (size_t)ls * stage_b;
      const float* a = reinterpret_cast<const float*>(st);
      const float mean = a[AUX - 2], rstd = a[AUX - 1], nmr = -mean * rstd;
      float alpha0[S], bp[S];
#pragma unroll
      for (int s = 0; s < S; ++s) {
        alpha0[s] = fmaf(a[s * T], a_scale, sa0[s]);
        bp[s] = EXPAND ? 0.f : head_bulk(S) ? a[AUX + S + s] : beta_prev[(size_t)m * S + s];
      }
      const int c8 = lt * 8;
      // r[s][e] = R_in + beta_prev (x) Y  (or x)
      auto load_r = [&](float (&r)[S][8], float (&y)[8]) {
        if (EXPAND) {
          float xv[8];
          hc2::lds4(reinterpret_cast<const float*>(st + SCAL_B) + c8, xv);
          hc2::lds4(reinterpret_cast<const float*>(st + SCAL_B) + c8 + 4, xv + 4);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            y[e] = 0.f;
#pragma unroll
            for (int s = 0; s < S; ++s) r[s][e] = xv[e];
          }
        } else {
          hc2::unpack8(*reinterpret_cast<const uint4*>(st + off_y<S>(d) + 2 * c8), y);
#pragma unroll
          for (int s = 0; s < S; ++s) {
            float rv[8];
            hc2::unpack8(*reinterpret_cast<const uint4*>(st + SCAL_B + 2 * (s * d + c8)), rv);
#pragma unroll
            for (int e = 0; e < 8; ++e) r[s][e] = fmaf(bp[s], y[e], rv[e]);
          }
        }
      };
      // ---------------- pass 1 ----------------
      // red: 0 sum gl | 1 sum gl*xhat | 2+s sum gl*R_s | 2+S+s sum R_s | 2+2S+s sum xhat*R_s | 2+3S+s sum ex*R_s |
      //      2+4S+S*s+(t-1) sum dR_out[t-1]*R_s  (gl = dxn * ln_gamma, xhat = normalised branch input, ex = dbin_extra;
      //      S = 4: 2+s, 6+s, 10+s, 14+s, 18+4s+(t-1))
      float red[NRED];
#pragma unroll
      for (int i = 0; i < NRED; ++i) red[i] = 0.f;
      if (act) {
        float r[S][8], y[8], dx[8], ex[8], lg[8];
        load_r(r, y);
        hc2::unpack8(*reinterpret_cast<const uint4*>(st + off_dxn<S>(d) + 2 * c8), dx);
        if (has_dbin) {
          hc2::unpack8(*reinterpret_cast<const uint4*>(st + off_dbin<S>(d) + 2 * c8), ex);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) ex[e] = 0.f;
        }
        lds8(pLn, half, lg);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float bsum = 0.f;
#pragma unroll
          for (int s = 0; s < S; ++s) bsum = fmaf(alpha0[s], r[s][e], bsum);
          const float xh = fmaf(bsum, rstd, nmr);
          const float gl = dx[e] * lg[e];
          gLn[e] = fmaf(dx[e], xh, gLn[e]);
          red[0] += gl;
          red[1] = fmaf(gl, xh, red[1]);
#pragma unroll
          for (int s = 0; s < S; ++s) {
            red[2 + s] = fmaf(gl, r[s][e], red[2 + s]);
            red[2 + S + s] += r[s][e];
            red[2 + 2 * S + s] = fmaf(xh, r[s][e], red[2 + 2 * S + s]);
            red[2 + 3 * S + s] = fmaf(ex[e], r[s][e], red[2 + 3 * S + s]);
          }
        }
#pragma unroll
        for (int t = 1; t < T; ++t) {
          float dm[8];
          hc2::unpack8(*reinterpret_cast<const uint4*>(st + off_dr<S>(d) + 2 * ((t - 1) * d + c8)), dm);
#pragma unroll
          for (int e = 0; e < 8; ++e)
#pragma unroll
            for (int s = 0; s < S; ++s) {
              const int i = 2 + 4 * S + S * s + (t - 1);
              red[i] = fmaf(dm[e], r[s][e], red[i]);
            }
        }
      }
      {
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = red[2 + i];
        const float mine = reduce_scatter32(v, lane);
        const float r0 = warp_sum(red[0]), r1 = warp_sum(red[1]);
        mail[w * MAILW + 2 + lane] = mine;
        if (lane == 0) {
          mail[w * MAILW] = r0;
          mail[w * MAILW + 1] = r1;
        }
      }
      named_bar_sync(bar_id, 128);
      if (k > 0 && w == 3) {  // every thread is past token k - 1: its stage takes token k - 1 + NSC
        fence_proxy_async_smem();
        fill(k - 1 + NSC);
      }
      auto total = [&](int i) { return (mail[i] + mail[MAILW + i]) + (mail[2 * MAILW + i] + mail[3 * MAILW + i]); };
      const float m1 = total(0) * inv_d, m2 = total(1) * inv_d;
      // ---------------- per-token scalars (warp 0) ----------------
      if (w == 0) {
        if (pend >= 0 && lane < S)
          dbeta_prev[(size_t)pend * S + lane] = (dbpm[lane] + dbpm[S + lane]) + (dbpm[2 * S + lane] + dbpm[3 * S + lane]);
        const float inv = a[S * T + S + ss];
        float zpart = 0.f, cst = 0.f;
        if (sv && q < T) {
          const float dal = q == 0 ? fmaf(rstd, total(2 + ss) - m1 * total(2 + S + ss) - m2 * total(2 + 2 * S + ss),
                                          total(2 + 3 * S + ss))
                                   : total(2 + 4 * S + S * ss + q - 1);
          const float ta = a[ss * T + q];
          const float dw = dal * a_scale * (1.f - ta * ta);
          zpart = dw * a[Z_OFF + ss * T + q];
          cst = inv * dw;
          coef[ss * COEF + q] = fmaf(ta, a_scale, stat);  // alpha[s][q]
          small0 += dal;
          small1 = fmaf(dal, ta, small1);
        } else if (sv && q == T) {
          const float tb = a[S * T + ss], dbe = head_bulk(S) ? a[AUX + ss] : dbeta[(size_t)m * S + ss];
          const float dwb = dbe * b_scale * (1.f - tb * tb);
          zpart = dwb * a[Z_OFF + S * T + ss];
          cst = inv * dwb;
          small0 += dbe;
          small1 = fmaf(dbe, tb, small1);
        }
        float zsum = zpart;
#pragma unroll
        for (int o = 1; o < 8; o <<= 1) zsum += __shfl_xor_sync(0xffffffffu, zsum, o);
        if (sv && q <= T) coef[ss * COEF + T + q] = cst;                 // C[s][q]
        else if (sv && q == T + 1) coef[ss * COEF + 2 * T + 1] = inv * inv * zsum;  // kk[s]: RMS-norm backward coefficient
      }
      named_bar_sync(bar_id, 128);
      // ---------------- pass 2 ----------------
      float al[S][T], C[S][NG], kk[S];
#pragma unroll
      for (int s = 0; s < S; ++s) {
        float cf[12];  // T + NG + 1 <= 12
#pragma unroll
        for (int i = 0; i < 3; ++i) hc2::lds4(coef + s * COEF + 4 * i, cf + 4 * i);
#pragma unroll
        for (int t = 0; t < T; ++t) al[s][t] = cf[t];
#pragma unroll
        for (int c6 = 0; c6 < NG; ++c6) C[s][c6] = cf[T + c6];
        kk[s] = cf[2 * T + 1];
      }
      float dbp[S];
#pragma unroll
      for (int s = 0; s < S; ++s) dbp[s] = 0.f;
      if (act) {
        float r[S][8], y[8], dr[S][8], dy[8];
        load_r(r, y);
        uint4 dmp[S], dxp, exp_ = make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int t = 0; t < S; ++t) dmp[t] = *reinterpret_cast<const uint4*>(st + off_dr<S>(d) + 2 * (t * d + c8));
        dxp = *reinterpret_cast<const uint4*>(st + off_dxn<S>(d) + 2 * c8);
        if (has_dbin) exp_ = *reinterpret_cast<const uint4*>(st + off_dbin<S>(d) + 2 * c8);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float pg[NG][4], lg[4];
          hc2::lds4(pLn + h * half, lg);
#pragma unroll
          for (int c6 = 0; c6 < NG; ++c6) hc2::lds4(pLn + (1 + c6) * d + h * half, pg[c6]);
#pragma unroll
          for (int e4 = 0; e4 < 4; ++e4) {
            const int e = 4 * h + e4;
            auto bf = [&](const uint4& u) {  // channel e of a packed row of 8
              const uint32_t x = (e >> 1) == 0 ? u.x : (e >> 1) == 1 ? u.y : (e >> 1) == 2 ? u.z : u.w;
              return (e & 1) ? bf16_hi(x) : bf16_lo(x);
            };
            float bsum = 0.f;
#pragma unroll
            for (int s = 0; s < S; ++s) bsum = fmaf(alpha0[s], r[s][e], bsum);
            const float xh = fmaf(bsum, rstd, nmr);
            // d(branch input) = rstd * (dxn*ln_gamma - m1 - xhat*m2) + dbin_extra
            float dm[T];
            dm[0] = fmaf(rstd, fmaf(xh, -m2, fmaf(bf(dxp), lg[e4], -m1)), bf(exp_));
#pragma unroll
            for (int t = 1; t < T; ++t) dm[t] = bf(dmp[t - 1]);
            dy[e] = 0.f;
#pragma unroll
            for (int s = 0; s < S; ++s) {
              float acc = -r[s][e] * kk[s];
#pragma unroll
              for (int t = 0; t < T; ++t) acc = fmaf(al[s][t], dm[t], acc);
#pragma unroll
              for (int c6 = 0; c6 < NG; ++c6) acc = fmaf(C[s][c6], pg[c6][e4], acc);
              dr[s][e] = acc;
              dbp[s] = fmaf(acc, y[e], dbp[s]);
              dy[e] = fmaf(bp[s], acc, dy[e]);
#pragma unroll
              for (int c6 = 0; c6 < NG; ++c6) G[c6][e] = fmaf(r[s][e], C[s][c6], G[c6][e]);
            }
          }
        }
        const size_t md = (size_t)m * d;
        if (EXPAND) {
          float o[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            float sum;
            if constexpr (S == 4) {
              sum = (dr[0][e] + dr[1][e]) + (dr[2][e] + dr[3][e]);
            } else {
              sum = dr[0][e];
#pragma unroll
              for (int s = 1; s < S; ++s) sum += dr[s][e];
            }
            o[e] = sum * dx_scale;
          }
          float* dst = dx_expand + md + c8;
          *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
          *reinterpret_cast<float4*>(dst + 4) = make_float4(o[4], o[5], o[6], o[7]);
        } else {
#pragma unroll
          for (int s = 0; s < S; ++s)
            *reinterpret_cast<uint4*>(dR_in + (md * S + (size_t)s * d) + c8) = hc2::pack8(dr[s]);
          *reinterpret_cast<uint4*>(dY + md + c8) = hc2::pack8(dy);
        }
      }
      if (!EXPAND) {
#pragma unroll
        for (int s = 0; s < S; ++s) dbp[s] = warp_sum(dbp[s]);
        if (lane == 0) {
#pragma unroll
          for (int s = 0; s < S; ++s) dbpm[w * S + s] = dbp[s];
        }
        pend = m;
      }
      if (++ls == NSC) {
        ls = 0;
        phase ^= 1;
      }
    }
    named_bar_sync(bar_id, 128);
    if (w == 0) {
      if (pend >= 0 && lane < S)
        dbeta_prev[(size_t)pend * S + lane] = (dbpm[lane] + dbpm[S + lane]) + (dbpm[2 * S + lane] + dbpm[3 * S + lane]);
      if (sv && q < T) atomicAdd(gr.static_alpha + ss * T + q, small0);
      else if (sv && q == T) atomicAdd(gr.static_beta + ss, small0);
      const float as = warp_sum(sv && q < T ? small1 : 0.f), bs = warp_sum(sv && q == T ? small1 : 0.f);
      if (lane == 0) {
        atomicAdd(gr.alpha_scale, as);
        atomicAdd(gr.beta_scale, bs);
      }
    }
    // per-channel partials of each warpgroup -> the ring, idle once every stage has been consumed: [NC][NP][d]
    __syncthreads();
    if (act) {
      float* buf = reinterpret_cast<float*>(ring) + (size_t)cw * NP * d + lt * 8;
#pragma unroll
      for (int c6 = 0; c6 < NG; ++c6) {
        *reinterpret_cast<float4*>(buf + c6 * d) = make_float4(G[c6][0], G[c6][1], G[c6][2], G[c6][3]);
        *reinterpret_cast<float4*>(buf + c6 * d + 4) = make_float4(G[c6][4], G[c6][5], G[c6][6], G[c6][7]);
      }
      *reinterpret_cast<float4*>(buf + NG * d) = make_float4(gLn[0], gLn[1], gLn[2], gLn[3]);
      *reinterpret_cast<float4*>(buf + NG * d + 4) = make_float4(gLn[4], gLn[5], gLn[6], gLn[7]);
    }
  }
  __syncthreads();
  // CTA sum of the per-channel partials, folded into the parameter gradients:
  //   d dyn_alpha[:, t] += g1 G_t,  d dyn_beta += g1 G_5,  d gamma += sqrt(d) sum_c P_c G_c,  g1 = (gamma + 1) sqrt(d)
  const float* buf = reinterpret_cast<const float*>(ring);
  for (int i = threadIdx.x; i < d; i += blockDim.x) {
    float g[NP];
#pragma unroll
    for (int k = 0; k < NP; ++k) {
      g[k] = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) g[k] += buf[(size_t)(c * NP + k) * d + i];
    }
    const float g1 = (prm.gamma_hc[i] + 1.f) * sqrt_d;
    float acc = g[T] * prm.dyn_beta[i];
    atomicAdd(gr.dyn_beta + i, g1 * g[T]);
#pragma unroll
    for (int t = 0; t < T; ++t) {
      acc = fmaf(g[t], prm.dyn_alpha[(size_t)i * T + t], acc);
      atomicAdd(gr.dyn_alpha + (size_t)i * T + t, g1 * g[t]);
    }
    atomicAdd(gr.gamma_hc + i, sqrt_d * acc);
    atomicAdd(gr.ln_gamma + i, g[NG]);
  }
}

}  // namespace hcr
}  // namespace alm
