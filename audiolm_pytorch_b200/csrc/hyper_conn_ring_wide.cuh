// Hyper-Connections backward for d <= 1024 and S = 5..8 streams: the ring of hyper_conn_ring.cuh, reorganised so that
// the per-thread state stays in the register file as S grows.  Same work per token, same stage contents:
//   pass 1   the 2 + 4S + S^2 per-token sums in rounds of 32 (one reduce_scatter32 per round), each round walking the
//            thread's 8 channels as two halves of 4, so that only R[S][4] is live;
//   scalars  warp 0 loops over the S (S + 2) (stream, column) pairs; the RMS-norm coefficient kk[s] sums its stream's
//            pairs through a small shared-memory row instead of an 8-lane shuffle;
//   pass 2   a runtime loop over the streams, each half of the thread's channels inside, one dR_out row and one map
//            column at a time: the coefficients, the map columns and dR_out come from shared memory where they are
//            used, and dR_in is written 4 channels (8 B) at a time.  What stays in registers is mainly the G[S + 2][8]
//            map-gradient accumulators.
// Two ring stages per warpgroup (a stage is (4S + 6) d bytes plus the head: 39 KB at S = 8, d = 1024).
#pragma once
#include "hyper_conn_ring.cuh"

namespace alm {
namespace hcr {

constexpr int NSC_W = 2;
constexpr int NST_W = NC * NSC_W;
__host__ __device__ constexpr bool ring_wide_ok(int S) { return S >= 5 && S <= 8; }
__host__ __device__ constexpr int nv_w(int S) { return 4 * S + S * S; }             // sums after the two LN sums
__host__ __device__ constexpr int rounds_w(int S) { return (nv_w(S) + 31) / 32; }
__host__ __device__ constexpr int mailw_w(int S) { return 4 + 32 * rounds_w(S); }
__host__ __device__ constexpr int coef_w(int S) { return (2 * S + 4 + 3) / 4 * 4; }  // alpha[T] C[S+2] kk, pad
static_assert(scal_bytes(8) % 16 == 0 && hc2::aux_floats(5) % 4 == 0 && hc2::aux_floats(7) % 4 == 0,
              "aux rows and the stage head must be 16-B multiples so that one bulk copy stages a row");

// shared memory: params [S+3][d] | mailboxes [NC][4][MAILW] | dbeta_prev partials [NC][4][S] | coefficients
// [NC][S][COEF] | z-partials [NC][S][S+2] | full[NST_W] mbarriers | ring [NC][NSC_W] stages (128-B aligned)
template <int S> __host__ __device__ inline int ring_offset_w(int d) {
  return (4 * ((S + 3) * d + NC * (4 * mailw_w(S) + 4 * S + S * coef_w(S) + S * (S + 2))) + 8 * NST_W + 127) / 128 *
         128;
}
template <int S> inline size_t smem_bytes_w(int d) {
  return (size_t)ring_offset_w<S>(d) + (size_t)NST_W * stage_bytes<S>(d);
}

__device__ __forceinline__ void unpack4(const uint2& u, float* f) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
}

template <int S, bool EXPAND>
__global__ void __launch_bounds__(THREADS, 1)
pre_bwd_wide_kernel(const __nv_bfloat16* __restrict__ R_in, const __nv_bfloat16* __restrict__ Y,
                    const float* __restrict__ beta_prev, const float* __restrict__ x_expand, hc2::Params prm,
                    const float* __restrict__ aux, const __nv_bfloat16* __restrict__ dR_out,
                    const __nv_bfloat16* __restrict__ dxn, const __nv_bfloat16* __restrict__ dbin_extra,
                    const float* __restrict__ dbeta, __nv_bfloat16* __restrict__ dR_in,
                    __nv_bfloat16* __restrict__ dY, float* __restrict__ dbeta_prev, float* __restrict__ dx_expand,
                    float dx_scale, hc2::Grads gr, int M, int d) {
  static_assert(ring_wide_ok(S), "the wide ring backward is built for 5 to 8 streams");
  constexpr int T = S + 1, AUX = hc2::aux_floats(S), Z_OFF = hc2::z_offset(S), SCAL_B = scal_bytes(S);
  constexpr int NP = S + 3, NG = S + 2, NV = nv_w(S), ROUNDS = rounds_w(S), MW = mailw_w(S), CW = coef_w(S);
  constexpr int NPAIR = S * NG, JP = (NPAIR + 31) / 32;  // scalar phase: (stream, column) pairs, per lane
  extern __shared__ __align__(128) unsigned char smem[];
  float* sPar = reinterpret_cast<float*>(smem);  // [NP][d]: ln_gamma, g1 * dyn_alpha[:, t], g1 * dyn_beta
  float* sMail = sPar + NP * d;                  // [NC][4][MW]
  float* sDbp = sMail + NC * 4 * MW;             // [NC][4][S]
  float* sCoef = sDbp + NC * 4 * S;              // [NC][S][CW]
  float* sZ = sCoef + NC * S * CW;               // [NC][S][NG]
  uint64_t* full = reinterpret_cast<uint64_t*>(sZ + NC * S * NG);
  unsigned char* ring = smem + ring_offset_w<S>(d);
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
    for (int i = 0; i < NST_W; ++i) mbar_init(&full[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, lt = threadIdx.x & 127;
  const int cw = warp >> 2, w = lt >> 5;
  const bool act = lt * 8 < d;
  const bool has_dbin = dbin_extra != nullptr;
  uint64_t* my_full = full + cw * NSC_W;
  unsigned char* my_ring = ring + (size_t)cw * NSC_W * stage_b;
  auto fill = [&](int k) {
    const int m = blockIdx.x + (cw + k * NC) * gridDim.x;
    if (m >= M) return;
    const int ls = k % NSC_W;
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
    for (int k = 0; k < NSC_W; ++k) fill(k);
  }
  {
    float G[NG][8], gLn[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      gLn[e] = 0.f;
#pragma unroll
      for (int c = 0; c < NG; ++c) G[c][e] = 0.f;
    }
    const int bar_id = 1 + cw;
    float* mail = sMail + cw * 4 * MW;
    float* dbpm = sDbp + cw * 4 * S;
    float* coef = sCoef + cw * S * CW;
    float* zrow = sZ + cw * S * NG;
    const float a_scale = *prm.alpha_scale, b_scale = *prm.beta_scale;
    const float inv_d = 1.f / (float)d;
    // (static_alpha is read through the read-only cache where it is used: registers go to G)
    float small0[JP], small1[JP];  // scalar phase, pair p = lane + 32 j: d static_alpha/beta, scale parts
#pragma unroll
    for (int j = 0; j < JP; ++j) small0[j] = small1[j] = 0.f;
    const float* pLn = sPar + lt * 4;
    int ls = 0;
    uint32_t phase = 0;
    int pend = -1;
    for (int k = 0, m = blockIdx.x + cw * gridDim.x; m < M; ++k, m += NC * gridDim.x) {
      mbar_wait(&my_full[ls], phase);
      const unsigned char* st = my_ring + (size_t)ls * stage_b;
      const float* a = reinterpret_cast<const float*>(st);
      const float mean = a[AUX - 2], rstd = a[AUX - 1], nmr = -mean * rstd;
      float alpha0[S];
#pragma unroll
      for (int s = 0; s < S; ++s) alpha0[s] = fmaf(a[s * T], a_scale, __ldg(prm.static_alpha + s * T));
      // beta_prev of stream s, from the stage head (or global memory) where it is used
      auto bp_of = [&](int s) {
        return EXPAND ? 0.f : head_bulk(S) ? a[AUX + S + s] : __ldg(beta_prev + (size_t)m * S + s);
      };
      const int c8 = lt * 8;
      // channels c8 + 4h .. c8 + 4h + 3 of the residual R_s = R_in + beta_prev (x) Y (or x), and Y
      auto load_y4 = [&](int h, float (&y)[4]) {
        if (EXPAND) {
#pragma unroll
          for (int e = 0; e < 4; ++e) y[e] = 0.f;
        } else {
          unpack4(*reinterpret_cast<const uint2*>(st + off_y<S>(d) + 2 * (c8 + 4 * h)), y);
        }
      };
      auto load_r4 = [&](int s, int h, const float (&y)[4], float (&r)[4]) {
        if (EXPAND) {
          hc2::lds4(reinterpret_cast<const float*>(st + SCAL_B) + c8 + 4 * h, r);
        } else {
          float rv[4];
          unpack4(*reinterpret_cast<const uint2*>(st + SCAL_B + 2 * (s * d + c8 + 4 * h)), rv);
#pragma unroll
          for (int e = 0; e < 4; ++e) r[e] = fmaf(bp_of(s), y[e], rv[e]);
        }
      };
      auto load_row4 = [&](int off, int h, float (&f)[4]) {  // a bf16 [d] row of the stage, the half's 4 channels
        unpack4(*reinterpret_cast<const uint2*>(st + off + 2 * (c8 + 4 * h)), f);
      };
      // ---------------- pass 1 ----------------
      // sums (as in hyper_conn_ring.cuh): 0 gl | 1 gl*xhat | 2+s gl*R_s | 2+S+s R_s | 2+2S+s xhat*R_s |
      //   2+3S+s ex*R_s | 2+4S+S*s+(t-1) dR_out[t-1]*R_s; round q reduces sums 2+32q .. 2+32q+31
      float r01[2] = {0.f, 0.f};
#pragma unroll
      for (int q = 0; q < ROUNDS; ++q) {
        float v[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = 0.f;
        if (act) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float y[4], r[S][4], dx[4], ex[4], lg[4], gl[4], xh[4];
            load_y4(h, y);
#pragma unroll
            for (int s = 0; s < S; ++s) load_r4(s, h, y, r[s]);
            load_row4(off_dxn<S>(d), h, dx);
            if (has_dbin) {
              load_row4(off_dbin<S>(d), h, ex);
            } else {
#pragma unroll
              for (int e = 0; e < 4; ++e) ex[e] = 0.f;
            }
            hc2::lds4(pLn + h * half, lg);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              float bsum = 0.f;
#pragma unroll
              for (int s = 0; s < S; ++s) bsum = fmaf(alpha0[s], r[s][e], bsum);
              xh[e] = fmaf(bsum, rstd, nmr);
              gl[e] = dx[e] * lg[e];
              if (q == 0) {
                gLn[4 * h + e] = fmaf(dx[e], xh[e], gLn[4 * h + e]);
                r01[0] += gl[e];
                r01[1] = fmaf(gl[e], xh[e], r01[1]);
              }
            }
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const int idx = 32 * q + i;
              if (idx < 4 * S) {
                const int kind = idx / S, s = idx % S;
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float f = kind == 0 ? gl[e] : kind == 1 ? 1.f : kind == 2 ? xh[e] : ex[e];
                  v[i] = fmaf(f, r[s][e], v[i]);
                }
              } else if (idx < NV) {
                const int j = idx - 4 * S, s = j / S, tm1 = j % S;
                float dm[4];
                load_row4(off_dr<S>(d) + 2 * tm1 * d, h, dm);
#pragma unroll
                for (int e = 0; e < 4; ++e) v[i] = fmaf(dm[e], r[s][e], v[i]);
              }
            }
          }
        }
        const float mine = reduce_scatter32(v, lane);
        mail[w * MW + 2 + 32 * q + lane] = mine;
      }
      {
        const float r0 = warp_sum(r01[0]), r1 = warp_sum(r01[1]);
        if (lane == 0) {
          mail[w * MW] = r0;
          mail[w * MW + 1] = r1;
        }
      }
      named_bar_sync(bar_id, 128);
      if (k > 0 && w == 3) {  // every thread is past token k - 1: its stage takes token k - 1 + NSC_W
        fence_proxy_async_smem();
        fill(k - 1 + NSC_W);
      }
      auto total = [&](int i) { return (mail[i] + mail[MW + i]) + (mail[2 * MW + i] + mail[3 * MW + i]); };
      const float m1 = total(0) * inv_d, m2 = total(1) * inv_d;
      // ---------------- per-token scalars (warp 0) ----------------
      if (w == 0) {
        if (pend >= 0 && lane < S)
          dbeta_prev[(size_t)pend * S + lane] = (dbpm[lane] + dbpm[S + lane]) + (dbpm[2 * S + lane] + dbpm[3 * S + lane]);
#pragma unroll
        for (int j = 0; j < JP; ++j) {
          const int p = lane + 32 * j, ps = p / NG, pq = p % NG;
          if (p < NPAIR) {
            const float inv = a[S * T + S + ps];
            float zpart, cst;
            if (pq < T) {
              const float dal = pq == 0 ? fmaf(rstd, total(2 + ps) - m1 * total(2 + S + ps) - m2 * total(2 + 2 * S + ps),
                                               total(2 + 3 * S + ps))
                                        : total(2 + 4 * S + S * ps + pq - 1);
              const float ta = a[ps * T + pq];
              const float dw = dal * a_scale * (1.f - ta * ta);
              zpart = dw * a[Z_OFF + ps * T + pq];
              cst = inv * dw;
              coef[ps * CW + pq] = fmaf(ta, a_scale, __ldg(prm.static_alpha + ps * T + pq));  // alpha[s][q]
              small0[j] += dal;
              small1[j] = fmaf(dal, ta, small1[j]);
            } else {
              const float tb = a[S * T + ps], dbe = head_bulk(S) ? a[AUX + ps] : dbeta[(size_t)m * S + ps];
              const float dwb = dbe * b_scale * (1.f - tb * tb);
              zpart = dwb * a[Z_OFF + S * T + ps];
              cst = inv * dwb;
              small0[j] += dbe;
              small1[j] = fmaf(dbe, tb, small1[j]);
            }
            coef[ps * CW + T + pq] = cst;  // C[s][q]
            zrow[p] = zpart;
          }
        }
        __syncwarp();
        if (lane < S) {
          float zsum = 0.f;
#pragma unroll
          for (int q = 0; q < NG; ++q) zsum += zrow[lane * NG + q];
          const float inv = a[S * T + S + lane];
          coef[lane * CW + 2 * T + 1] = inv * inv * zsum;  // kk[s]: RMS-norm backward coefficient
        }
      }
      named_bar_sync(bar_id, 128);
      // ---------------- pass 2 ----------------
      // stream-outer (a runtime loop: one stream's values live at a time), the thread's two halves inside
      const size_t md = (size_t)m * d;
      float y[2][4], dm0[2][4], out[2][4];
      if (act) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float lg[4], bsum[4] = {0.f, 0.f, 0.f, 0.f}, dx[4], ex[4];
          load_y4(h, y[h]);
          hc2::lds4(pLn + h * half, lg);
#pragma unroll
          for (int s = 0; s < S; ++s) {
            float r[4];
            load_r4(s, h, y[h], r);
#pragma unroll
            for (int e = 0; e < 4; ++e) bsum[e] = fmaf(alpha0[s], r[e], bsum[e]);
          }
          load_row4(off_dxn<S>(d), h, dx);
          if (has_dbin) {
            load_row4(off_dbin<S>(d), h, ex);
          } else {
#pragma unroll
            for (int e = 0; e < 4; ++e) ex[e] = 0.f;
          }
          // d(branch input) = rstd * (dxn*ln_gamma - m1 - xhat*m2) + dbin_extra
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float xh = fmaf(bsum[e], rstd, nmr);
            dm0[h][e] = fmaf(rstd, fmaf(xh, -m2, fmaf(dx[e], lg[e], -m1)), ex[e]);
            out[h][e] = 0.f;
          }
        }
      }
      // per stream: dR_s = sum_t alpha[s][t] dmix_t + sum_c C[s][c] P_c - kk[s] R_s, one dR_out row and one map column
      // at a time (the coefficients are read where they are used)
#pragma unroll 1
      for (int s = 0; s < S; ++s) {
        const float bps = bp_of(s);
        float dbps = 0.f;
        if (act) {
          const float* cf = coef + s * CW;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float r[4], acc[4];
            if (EXPAND) {
              hc2::lds4(reinterpret_cast<const float*>(st + SCAL_B) + c8 + 4 * h, r);
            } else {
              float rv[4];
              unpack4(*reinterpret_cast<const uint2*>(st + SCAL_B + 2 * (s * d + c8 + 4 * h)), rv);
#pragma unroll
              for (int e = 0; e < 4; ++e) r[e] = fmaf(bps, y[h][e], rv[e]);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[e] = fmaf(cf[0], dm0[h][e], -r[e] * cf[2 * T + 1]);
#pragma unroll
            for (int t = 1; t < T; ++t) {
              float dmt[4];
              load_row4(off_dr<S>(d) + 2 * (t - 1) * d, h, dmt);
              const float al = cf[t];
#pragma unroll
              for (int e = 0; e < 4; ++e) acc[e] = fmaf(al, dmt[e], acc[e]);
            }
#pragma unroll
            for (int c = 0; c < NG; ++c) {
              float pg[4];
              hc2::lds4(pLn + (1 + c) * d + h * half, pg);
              const float C = cf[T + c];
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                acc[e] = fmaf(C, pg[e], acc[e]);
                G[c][4 * h + e] = fmaf(r[e], C, G[c][4 * h + e]);
              }
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              dbps = fmaf(acc[e], y[h][e], dbps);
              out[h][e] = EXPAND ? out[h][e] + acc[e] : fmaf(bps, acc[e], out[h][e]);
            }
            if (!EXPAND)
              *reinterpret_cast<uint2*>(dR_in + (md * S + (size_t)s * d) + c8 + 4 * h) =
                  make_uint2(hc2::pk(acc[0], acc[1]), hc2::pk(acc[2], acc[3]));
          }
        }
        if (!EXPAND) {
          dbps = warp_sum(dbps);
          if (lane == 0) dbpm[w * S + s] = dbps;
        }
      }
      if (act) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (EXPAND) {
            *reinterpret_cast<float4*>(dx_expand + md + c8 + 4 * h) = make_float4(
                out[h][0] * dx_scale, out[h][1] * dx_scale, out[h][2] * dx_scale, out[h][3] * dx_scale);
          } else {
            *reinterpret_cast<uint2*>(dY + md + c8 + 4 * h) =
                make_uint2(hc2::pk(out[h][0], out[h][1]), hc2::pk(out[h][2], out[h][3]));
          }
        }
      }
      if (!EXPAND) pend = m;
      if (++ls == NSC_W) {
        ls = 0;
        phase ^= 1;
      }
    }
    named_bar_sync(bar_id, 128);
    if (w == 0) {
      if (pend >= 0 && lane < S)
        dbeta_prev[(size_t)pend * S + lane] = (dbpm[lane] + dbpm[S + lane]) + (dbpm[2 * S + lane] + dbpm[3 * S + lane]);
      float as = 0.f, bs = 0.f;
#pragma unroll
      for (int j = 0; j < JP; ++j) {
        const int p = lane + 32 * j, ps = p / NG, pq = p % NG;
        if (p < NPAIR) {
          if (pq < T) {
            atomicAdd(gr.static_alpha + ps * T + pq, small0[j]);
            as += small1[j];
          } else {
            atomicAdd(gr.static_beta + ps, small0[j]);
            bs += small1[j];
          }
        }
      }
      as = warp_sum(as);
      bs = warp_sum(bs);
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
      for (int c = 0; c < NG; ++c) {
        *reinterpret_cast<float4*>(buf + c * d) = make_float4(G[c][0], G[c][1], G[c][2], G[c][3]);
        *reinterpret_cast<float4*>(buf + c * d + 4) = make_float4(G[c][4], G[c][5], G[c][6], G[c][7]);
      }
      *reinterpret_cast<float4*>(buf + NG * d) = make_float4(gLn[0], gLn[1], gLn[2], gLn[3]);
      *reinterpret_cast<float4*>(buf + NG * d + 4) = make_float4(gLn[4], gLn[5], gLn[6], gLn[7]);
    }
  }
  __syncthreads();
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
