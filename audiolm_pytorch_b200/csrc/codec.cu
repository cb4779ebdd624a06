// SoundStream codec kernels (fp32): causal strided / dilated Conv1d with in-kernel reflect halo,
// polyphase causal ConvTranspose1d, residual-VQ nearest-code search (8 stages in one launch) and
// RVQ decode.  References: soundstream.py:332-369 (CausalConv1d / CausalConvTranspose1d /
// ResidualUnit), :691-709, :840 and vector-quantize-pytorch's ResidualVQ eval path (oracle/third_party.py).
//
// These are CUDA-core kernels: the convs and the code search are FMA-bound in fp32 (arithmetic
// intensity 64-512 FLOP/B, see DESIGN.md); data movement is coalesced along time and staged through
// shared memory so each input sample / codebook row is read from HBM once per output tile.
#include <stdlib.h>

#include "alm_common.cuh"
#include "conv_tiled.cuh"

namespace alm {

__device__ __forceinline__ float elu1(float x) { return x > 0.f ? x : expm1f(x); }

// index into the causally padded signal: position i of xp (pad = left padding) -> source sample or -1 (zero)
__device__ __forceinline__ int padded_src(int i, int pad, int T, int mode) {
  if (i >= pad) return i - pad;
  if (mode == 0) return pad - i;      // reflect (edge sample excluded): xp[i] = x[pad - i]
  if (mode == 1) return -1;           // constant zero
  return 0;                           // replicate
}

// ------------------------------------------------------------------------------------------------
// y[b, o, t] = act( bias[o] + sum_c sum_j W[o, c, j] * xp[b, c, t*stride + j*dil] ) (+ residual[b, o, t])
// tile: 32 output channels x 128 output samples per CTA, input channels in chunks of 8.
// ------------------------------------------------------------------------------------------------
constexpr int CV_CO = 32, CV_T = 128, CV_CI = 8, CV_THREADS = 256;

__global__ void __launch_bounds__(CV_THREADS)
causal_conv1d_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                     const float* __restrict__ residual, float* __restrict__ y, int B, int Cin, int Cout, int T,
                     int Tout, int K, int stride, int dil, int pad, int pad_mode, int act) {
  extern __shared__ float smem[];
  const int span = (CV_T - 1) * stride + (K - 1) * dil + 1;  // input samples needed per tile
  float* xs = smem;                    // [CV_CI][span]
  float* ws = smem + CV_CI * span;     // [CV_CI][K][CV_CO]
  const int t0 = blockIdx.x * CV_T, o0 = blockIdx.y * CV_CO, b = blockIdx.z;
  const int to = threadIdx.x & 31;     // 32 time lanes, each 4 samples strided by 32
  const int oc = threadIdx.x >> 5;     // 8 groups of 4 output channels
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int in0 = t0 * stride;  // first padded-signal index of this tile
  for (int c0 = 0; c0 < Cin; c0 += CV_CI) {
    __syncthreads();
    for (int i = threadIdx.x; i < CV_CI * span; i += CV_THREADS) {
      const int c = i / span, p = i - c * span;
      float v = 0.f;
      if (c0 + c < Cin) {
        const int src = padded_src(in0 + p, pad, T, pad_mode);
        if (src >= 0 && src < T) v = x[((size_t)b * Cin + c0 + c) * T + src];
      }
      xs[i] = v;
    }
    for (int i = threadIdx.x; i < CV_CI * K * CV_CO; i += CV_THREADS) {
      const int o = i % CV_CO, r = i / CV_CO, j = r % K, c = r / K;
      float v = 0.f;
      if (c0 + c < Cin && o0 + o < Cout) v = w[((size_t)(o0 + o) * Cin + c0 + c) * K + j];
      ws[i] = v;
    }
    __syncthreads();
    for (int c = 0; c < CV_CI; ++c) {
      const float* xc = xs + c * span;
      const float* wc = ws + c * K * CV_CO + oc * 4;
      for (int j = 0; j < K; ++j) {
        const float4 wv = *reinterpret_cast<const float4*>(wc + j * CV_CO);
        float xv[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) xv[q] = xc[(to + q * 32) * stride + j * dil];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          acc[0][q] = fmaf(wv.x, xv[q], acc[0][q]);
          acc[1][q] = fmaf(wv.y, xv[q], acc[1][q]);
          acc[2][q] = fmaf(wv.z, xv[q], acc[2][q]);
          acc[3][q] = fmaf(wv.w, xv[q], acc[3][q]);
        }
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int o = o0 + oc * 4 + i;
    if (o >= Cout) continue;
    const float bv = bias ? bias[o] : 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int t = t0 + to + q * 32;
      if (t >= Tout) continue;
      float v = acc[i][q] + bv;
      if (act) v = elu1(v);
      const size_t idx = ((size_t)b * Cout + o) * Tout + t;
      if (residual) v += residual[idx];
      y[idx] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// causal ConvTranspose1d, kernel 2s, stride s, output trimmed to n*s (soundstream.py:347-360):
//   y[b, o, i*s + r] = bias[o] + sum_c W[c, o, r] x[b, c, i] + W[c, o, r + s] x[b, c, i - 1]
// tile: 32 output channels x 64 input positions (x s phases) per CTA.
// ------------------------------------------------------------------------------------------------
constexpr int CT_CO = 32, CT_TI = 64, CT_CI = 8, CT_MAXS = 8;

__global__ void __launch_bounds__(256)
causal_convT1d_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                      float* __restrict__ y, int B, int Cin, int Cout, int n, int s) {
  __shared__ float xs[CT_CI][CT_TI + 1];
  __shared__ float ws[CT_CI][2 * CT_MAXS][CT_CO];
  const int i0 = blockIdx.x * CT_TI, o0 = blockIdx.y * CT_CO, b = blockIdx.z;
  const int o = threadIdx.x & 31, ig = threadIdx.x >> 5;  // 8 groups x 8 input positions
  float acc[8][CT_MAXS];
#pragma unroll
  for (int p = 0; p < 8; ++p)
#pragma unroll
    for (int r = 0; r < CT_MAXS; ++r) acc[p][r] = 0.f;
  for (int c0 = 0; c0 < Cin; c0 += CT_CI) {
    __syncthreads();
    for (int i = threadIdx.x; i < CT_CI * (CT_TI + 1); i += 256) {
      const int c = i / (CT_TI + 1), p = i - c * (CT_TI + 1);
      const int src = i0 + p - 1;  // xs[c][p] = x[i0 + p - 1]
      xs[c][p] = (c0 + c < Cin && src >= 0 && src < n) ? x[((size_t)b * Cin + c0 + c) * n + src] : 0.f;
    }
    for (int i = threadIdx.x; i < CT_CI * 2 * s * CT_CO; i += 256) {
      const int oo = i % CT_CO, r2 = (i / CT_CO) % (2 * s), c = i / (CT_CO * 2 * s);
      ws[c][r2][oo] = (c0 + c < Cin && o0 + oo < Cout) ? w[((size_t)(c0 + c) * Cout + o0 + oo) * (2 * s) + r2] : 0.f;
    }
    __syncthreads();
    for (int c = 0; c < CT_CI; ++c) {
      float xv[9];
#pragma unroll
      for (int p = 0; p < 9; ++p) xv[p] = xs[c][ig * 8 + p];
#pragma unroll
      for (int r = 0; r < CT_MAXS; ++r) {
        if (r < s) {
          const float w0 = ws[c][r][o], w1 = ws[c][r + s][o];
#pragma unroll
          for (int p = 0; p < 8; ++p) acc[p][r] = fmaf(w0, xv[p + 1], fmaf(w1, xv[p], acc[p][r]));
        }
      }
    }
  }
  if (o0 + o >= Cout) return;
  const float bv = bias ? bias[o0 + o] : 0.f;
#pragma unroll
  for (int p = 0; p < 8; ++p) {
    const int i = i0 + ig * 8 + p;
    if (i >= n) continue;
#pragma unroll
    for (int r = 0; r < CT_MAXS; ++r)
      if (r < s) y[((size_t)b * Cout + o0 + o) * ((size_t)n * s) + (size_t)i * s + r] = acc[p][r] + bv;
  }
}

// ------------------------------------------------------------------------------------------------
// residual VQ, eval path.  One CTA owns RV_ROWS rows for ALL stages: the residual tile lives in smem,
// codebook tiles stream through smem, distances follow the reference's expansion
//     d = sqrt(max((|r|^2 + |e|^2) - 2 r.e, 0)),  argmin with lowest index on ties.
// ------------------------------------------------------------------------------------------------
constexpr int RV_ROWS = 32, RV_CODES = 32, RV_THREADS = 256;

__global__ void code_norms_kernel(const float* __restrict__ cb, float* __restrict__ e2, int total, int D) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (gw >= total) return;
  float a = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = cb[(size_t)gw * D + d];
    a = fmaf(v, v, a);
  }
  a = warp_sum(a);
  if (lane == 0) e2[gw] = a;
}

__global__ void __launch_bounds__(RV_THREADS)
rvq_encode_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ cb,
                  const float* __restrict__ e2, float* __restrict__ quant, long long ldq,
                  long long* __restrict__ indices, long long ldi, int N, int D, int C, int Q) {
  extern __shared__ float smem[];
  const int DP = D + 4;                       // padded row stride (conflict-free float4 reads)
  float* R = smem;                            // [RV_ROWS][DP] residual
  float* E = R + RV_ROWS * DP;                // [RV_CODES][DP] code tile
  float* x2 = E + RV_CODES * DP;              // [RV_ROWS]
  int* best_idx = reinterpret_cast<int*>(x2 + RV_ROWS);  // [RV_ROWS]
  const int n0 = blockIdx.x * RV_ROWS;
  const int tid = threadIdx.x;
  const int tx = tid & 15;        // code lane: codes tx and tx+16 of the tile
  const int ty = tid >> 4;        // 16 row groups of 2 rows
  for (int i = tid; i < RV_ROWS * D; i += RV_THREADS) {
    const int r = i / D, d = i - r * D;
    R[r * DP + d] = (n0 + r < N) ? x[(size_t)(n0 + r) * ldx + d] : 0.f;
  }
  __syncthreads();
  for (int q = 0; q < Q; ++q) {
    // |r|^2 per row: 8 threads per row
    {
      const int r = tid >> 3, part = tid & 7;
      float a = 0.f;
      for (int d = part; d < D; d += 8) a = fmaf(R[r * DP + d], R[r * DP + d], a);
      a += __shfl_xor_sync(0xffffffffu, a, 1);
      a += __shfl_xor_sync(0xffffffffu, a, 2);
      a += __shfl_xor_sync(0xffffffffu, a, 4);
      if (part == 0) x2[r] = a;
    }
    float bd[2] = {INFINITY, INFINITY};
    int bi[2] = {0, 0};
    const float* cbq = cb + (size_t)q * C * D;
    for (int c0 = 0; c0 < C; c0 += RV_CODES) {
      __syncthreads();
      for (int i = tid; i < RV_CODES * D; i += RV_THREADS) {
        const int c = i / D, d = i - c * D;
        E[c * DP + d] = (c0 + c < C) ? cbq[(size_t)(c0 + c) * D + d] : 0.f;
      }
      __syncthreads();
      float dot[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
      const float* r0 = R + (ty * 2) * DP;
      const float* r1 = r0 + DP;
      const float* ea = E + tx * DP;
      const float* eb = E + (tx + 16) * DP;
      for (int d = 0; d < D; d += 4) {
        const float4 a0 = *reinterpret_cast<const float4*>(r0 + d), a1 = *reinterpret_cast<const float4*>(r1 + d);
        const float4 va = *reinterpret_cast<const float4*>(ea + d), vb = *reinterpret_cast<const float4*>(eb + d);
        dot[0][0] = fmaf(a0.x, va.x, dot[0][0]); dot[0][0] = fmaf(a0.y, va.y, dot[0][0]);
        dot[0][0] = fmaf(a0.z, va.z, dot[0][0]); dot[0][0] = fmaf(a0.w, va.w, dot[0][0]);
        dot[0][1] = fmaf(a0.x, vb.x, dot[0][1]); dot[0][1] = fmaf(a0.y, vb.y, dot[0][1]);
        dot[0][1] = fmaf(a0.z, vb.z, dot[0][1]); dot[0][1] = fmaf(a0.w, vb.w, dot[0][1]);
        dot[1][0] = fmaf(a1.x, va.x, dot[1][0]); dot[1][0] = fmaf(a1.y, va.y, dot[1][0]);
        dot[1][0] = fmaf(a1.z, va.z, dot[1][0]); dot[1][0] = fmaf(a1.w, va.w, dot[1][0]);
        dot[1][1] = fmaf(a1.x, vb.x, dot[1][1]); dot[1][1] = fmaf(a1.y, vb.y, dot[1][1]);
        dot[1][1] = fmaf(a1.z, vb.z, dot[1][1]); dot[1][1] = fmaf(a1.w, vb.w, dot[1][1]);
      }
#pragma unroll
      for (int rr = 0; rr < 2; ++rr)
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const int c = c0 + tx + cc * 16;
          if (c < C) {
            const float d2 = (x2[ty * 2 + rr] + e2[(size_t)q * C + c]) + (-2.f * dot[rr][cc]);
            const float dist = __fsqrt_rn(fmaxf(d2, 0.f));
            if (dist < bd[rr]) { bd[rr] = dist; bi[rr] = c; }  // codes visited in increasing order
          }
        }
    }
    // argmin across the 16 code lanes of each row (lowest index wins ties)
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, bd[rr], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[rr], o);
        if (od < bd[rr] || (od == bd[rr] && oi < bi[rr])) { bd[rr] = od; bi[rr] = oi; }
      }
      if (tx == 0) best_idx[ty * 2 + rr] = bi[rr];
    }
    __syncthreads();
    // residual -= code ; quantized += code ; emit index
    for (int i = tid; i < RV_ROWS * D; i += RV_THREADS) {
      const int r = i / D, d = i - r * D;
      if (n0 + r < N) {
        const float e = cbq[(size_t)best_idx[r] * D + d];
        R[r * DP + d] -= e;
        float* qp = quant + (size_t)(n0 + r) * ldq + d;
        *qp = (q == 0 ? 0.f : *qp) + e;
      }
    }
    if (tid < RV_ROWS && n0 + tid < N) indices[(size_t)(n0 + tid) * ldi + q] = best_idx[tid];
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// residual VQ, second generation: same arithmetic (dot products accumulate over d in ascending order with one fp32
// FMA chain, so every distance - and therefore every index - is bit-identical to rvq_encode_kernel above), but
//   * a thread owns 8 rows x 4 codes (32 accumulators): per 4 channels it issues 8 broadcast LDS.128 (rows) and
//     4 conflict-free LDS.128 (codes) for 128 FMAs - the first version issued 4 LDS.128 per 16 FMAs and stalled on
//     shared-memory bandwidth and on synchronous codebook loads;
//   * the codebook streams through shared memory in [256 codes x 32 channels] chunks with cp.async double buffering.
// CTA = 32 rows (4 row groups x 8) x 256 codes per tile (2 code groups x 32 lanes x 4), all Q stages.
// ------------------------------------------------------------------------------------------------
constexpr int RQ_ROWS = 32, RQ_CT = 256, RQ_KC = 32, RQ_ES = RQ_KC + 4, RQ_THREADS = 256;

__device__ __forceinline__ void cp_async16(void* dst_smem, const void* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  const int sz = valid ? 16 : 0;  // src-size 0 -> the 16 destination bytes are zero-filled
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

__global__ void __launch_bounds__(RQ_THREADS, 1)
rvq_encode_v2_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ cb,
                     const float* __restrict__ e2, float* __restrict__ quant, long long ldq,
                     long long* __restrict__ indices, long long ldi, int N, int D, int C, int Q) {
  extern __shared__ __align__(16) float smem[];
  const int DP = D + 4;
  float* R = smem;                                 // [RQ_ROWS][DP] residual
  float* E = R + RQ_ROWS * DP;                     // [2][RQ_CT][RQ_ES] codebook chunk (double buffered)
  float* x2 = E + 2 * RQ_CT * RQ_ES;               // [RQ_ROWS]
  float* sbd = x2 + RQ_ROWS;                       // [2][RQ_ROWS] best distance per code group
  int* sbi = reinterpret_cast<int*>(sbd + 2 * RQ_ROWS);  // [2][RQ_ROWS]
  int* best_idx = sbi + 2 * RQ_ROWS;               // [RQ_ROWS]
  const int n0 = blockIdx.x * RQ_ROWS;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rg = warp & 3, cg = warp >> 2;         // row group (8 rows), code group (128 codes of the tile)
  const int n_kc = D / RQ_KC;
  for (int i = tid; i < RQ_ROWS * D; i += RQ_THREADS) {
    const int r = i / D, d = i - r * D;
    R[r * DP + d] = (n0 + r < N) ? x[(size_t)(n0 + r) * ldx + d] : 0.f;
  }
  __syncthreads();
  for (int q = 0; q < Q; ++q) {
    {  // |r|^2 per row: 8 threads per row (same partial-sum order as the first-generation kernel)
      const int r = tid >> 3, part = tid & 7;
      float a = 0.f;
      for (int d = part; d < D; d += 8) a = fmaf(R[r * DP + d], R[r * DP + d], a);
      a += __shfl_xor_sync(0xffffffffu, a, 1);
      a += __shfl_xor_sync(0xffffffffu, a, 2);
      a += __shfl_xor_sync(0xffffffffu, a, 4);
      if (part == 0) x2[r] = a;
    }
    float bd[8];
    int bi[8];
#pragma unroll
    for (int rr = 0; rr < 8; ++rr) { bd[rr] = INFINITY; bi[rr] = 0; }
    const float* cbq = cb + (size_t)q * C * D;
    auto issue_chunk = [&](int c0, int kc, int buf) {
      // 256 codes x 32 channels = 2048 float4: 8 per thread; a warp copies 4 codes x 128 B per pass (coalesced)
      float* dst = E + buf * (RQ_CT * RQ_ES);
#pragma unroll
      for (int it = 0; it < (RQ_CT * RQ_KC / 4) / RQ_THREADS; ++it) {
        const int v = tid + it * RQ_THREADS;
        const int code = v >> 3, f4 = v & 7;
        const bool ok = c0 + code < C;
        cp_async16(dst + code * RQ_ES + f4 * 4, cbq + (size_t)(ok ? c0 + code : 0) * D + kc * RQ_KC + f4 * 4, ok);
      }
      cp_async_commit();
    };
    for (int c0 = 0; c0 < C; c0 += RQ_CT) {
      float acc[8][4];
#pragma unroll
      for (int rr = 0; rr < 8; ++rr)
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) acc[rr][cc] = 0.f;
      __syncthreads();  // every warp is done with both chunk buffers (and x2 / R are up to date)
      issue_chunk(c0, 0, 0);
      for (int kc = 0; kc < n_kc; ++kc) {
        if (kc + 1 < n_kc) {
          issue_chunk(c0, kc + 1, (kc + 1) & 1);
          cp_async_wait<1>();
        } else {
          cp_async_wait<0>();
        }
        __syncthreads();
        const float* rbase = R + (rg * 8) * DP + kc * RQ_KC;
        const float* ebase = E + (kc & 1) * (RQ_CT * RQ_ES) + (cg * 128 + lane) * RQ_ES;
#pragma unroll 2
        for (int d4 = 0; d4 < RQ_KC / 4; ++d4) {
          float4 ev[4];
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) ev[cc] = *reinterpret_cast<const float4*>(ebase + cc * 32 * RQ_ES + d4 * 4);
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) {
            const float4 rv = *reinterpret_cast<const float4*>(rbase + rr * DP + d4 * 4);
#pragma unroll
            for (int cc = 0; cc < 4; ++cc) {
              float a = acc[rr][cc];
              a = fmaf(rv.x, ev[cc].x, a);
              a = fmaf(rv.y, ev[cc].y, a);
              a = fmaf(rv.z, ev[cc].z, a);
              a = fmaf(rv.w, ev[cc].w, a);
              acc[rr][cc] = a;
            }
          }
        }
        __syncthreads();  // this chunk buffer may be refilled by the copy issued in the next iteration
      }
#pragma unroll
      for (int cc = 0; cc < 4; ++cc) {  // codes in increasing order per thread: strict '<' keeps the lowest index
        const int c = c0 + cg * 128 + lane + 32 * cc;
        if (c < C) {
          const float e2c = e2[(size_t)q * C + c];
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) {
            const float d2 = (x2[rg * 8 + rr] + e2c) + (-2.f * acc[rr][cc]);
            const float dist = __fsqrt_rn(fmaxf(d2, 0.f));
            if (dist < bd[rr]) { bd[rr] = dist; bi[rr] = c; }
          }
        }
      }
    }
    // argmin across the 32 lanes, then across the two code groups (lowest index wins ties)
#pragma unroll
    for (int rr = 0; rr < 8; ++rr) {
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float od = __shfl_xor_sync(0xffffffffu, bd[rr], o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi[rr], o);
        if (od < bd[rr] || (od == bd[rr] && oi < bi[rr])) { bd[rr] = od; bi[rr] = oi; }
      }
      if (lane == 0) { sbd[cg * RQ_ROWS + rg * 8 + rr] = bd[rr]; sbi[cg * RQ_ROWS + rg * 8 + rr] = bi[rr]; }
    }
    __syncthreads();
    if (tid < RQ_ROWS) {
      const float d0 = sbd[tid], d1 = sbd[RQ_ROWS + tid];
      const int i0 = sbi[tid], i1 = sbi[RQ_ROWS + tid];
      best_idx[tid] = (d1 < d0 || (d1 == d0 && i1 < i0)) ? i1 : i0;
    }
    __syncthreads();
    // residual -= code ; quantized += code ; emit index
    for (int i = tid; i < RQ_ROWS * D; i += RQ_THREADS) {
      const int r = i / D, d = i - r * D;
      if (n0 + r < N) {
        const float e = cbq[(size_t)best_idx[r] * D + d];
        R[r * DP + d] -= e;
        float* qp = quant + (size_t)(n0 + r) * ldq + d;
        *qp = (q == 0 ? 0.f : *qp) + e;
      }
    }
    if (tid < RQ_ROWS && n0 + tid < N) indices[(size_t)(n0 + tid) * ldi + q] = best_idx[tid];
    __syncthreads();
  }
}

// out[n, :] = sum_q cb[q][idx[n, q]]   (idx < 0 = dropped quantizer -> contributes 0)
__global__ void rvq_decode_kernel(const long long* __restrict__ indices, long long ldi, const float* __restrict__ cb,
                                  float* __restrict__ out, long long ldo, int N, int D, int C, int Q) {
  const int n = blockIdx.x;
  for (int d = threadIdx.x; d < D; d += blockDim.x) {
    float a = 0.f;
    for (int q = 0; q < Q; ++q) {
      const long long id = indices[(size_t)n * ldi + q];
      if (id >= 0) a += cb[((size_t)q * C + id) * D + d];
    }
    out[(size_t)n * ldo + d] = a;
  }
}

// ------------------------------------------------------------------------------------------------
// SqueezeExcite of a ResidualUnit (soundstream.py:145-169, 362-369), fp32 on CUDA cores:
//   out[b, c, t] = x[b, c, t] + y[b, c, t] * sigmoid(b2[c] + sum_i W2[c, i] silu(b1[i] + sum_c' W1'[i, c'] y[b, c', t]))
// y = the unit's ELU(conv1(...)) output, x its input; W1' is the first 1x1 conv with the reference's channel-wise
// cumulative mean folded in (ops.se_fold_weight), so every time step is independent.  One CTA = SE_T time steps of one
// clip; the y tile and the inner activations stay in shared memory, weights are warp-uniform loads.
// ------------------------------------------------------------------------------------------------
constexpr int SE_T = 64;

__global__ void __launch_bounds__(SE_T)
se_fp32_kernel(const float* __restrict__ y, const float* __restrict__ x, const float* __restrict__ w1,
               const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
               float* __restrict__ out, int C, int Ci, int T) {
  extern __shared__ float smem[];
  float* ys = smem;               // [C][SE_T]
  float* ss = smem + C * SE_T;    // [Ci][SE_T]
  const int b = blockIdx.y, tid = threadIdx.x;
  const int t = blockIdx.x * SE_T + tid;
  const bool ok = t < T;
  const size_t base = (size_t)b * C * T;
  for (int c = 0; c < C; ++c) ys[c * SE_T + tid] = ok ? y[base + (size_t)c * T + t] : 0.f;
  for (int i = 0; i < Ci; ++i) {
    float acc = __ldg(b1 + i);
    for (int c = 0; c < C; ++c) acc = fmaf(__ldg(w1 + (size_t)i * C + c), ys[c * SE_T + tid], acc);
    ss[i * SE_T + tid] = acc / (1.f + expf(-acc));
  }
  if (!ok) return;
  for (int c = 0; c < C; ++c) {
    float acc = __ldg(b2 + c);
    for (int i = 0; i < Ci; ++i) acc = fmaf(__ldg(w2 + (size_t)c * Ci + i), ss[i * SE_T + tid], acc);
    out[base + (size_t)c * T + t] = x[base + (size_t)c * T + t] + ys[c * SE_T + tid] / (1.f + expf(-acc));
  }
}

}  // namespace alm

using namespace alm;

extern "C" int alm_causal_conv1d_fwd(const float* x, const float* w, const float* bias, const float* residual,
                                     float* y, int B, int Cin, int Cout, int T, int K, int stride, int dilation,
                                     int pad_mode, int act_elu, int w_packed, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && w && y && B > 0 && Cin > 0 && Cout > 0 && T > 0 && K > 0 && stride > 0 && dilation > 0,
              ALM_ERR_ARG);
  ALM_REQUIRE(pad_mode >= 0 && pad_mode <= 2, ALM_ERR_ARG);
  const int pad = dilation * (K - 1) + 1 - stride;
  ALM_REQUIRE(pad >= 0, ALM_ERR_ARG);
  ALM_REQUIRE(pad_mode != 0 || pad < T, ALM_ERR_ARG);  // reflect needs pad < T (as F.pad does)
  const int Tout = (T + pad - dilation * (K - 1) - 1) / stride + 1;
  {
    if (w_packed) {  // register-tiled kernels read the packed [Cin][K][Cout] weight copy
      const int rc = cvt::dispatch(x, w, bias, residual, y, B, Cin, Cout, T, Tout, K, stride, dilation, pad, pad_mode,
                                   act_elu, stream);
      if (rc != -1) return rc;
    }
  }
  ALM_REQUIRE(!w_packed, ALM_ERR_UNSUPPORTED);  // the generic kernel reads the torch layout only
  const int span = (CV_T - 1) * stride + (K - 1) * dilation + 1;
  const size_t smem = (size_t)(CV_CI * span + CV_CI * K * CV_CO) * sizeof(float);
  ALM_REQUIRE(smem <= 200 * 1024, ALM_ERR_UNSUPPORTED);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(causal_conv1d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  dim3 grid(ceil_div(Tout, CV_T), ceil_div(Cout, CV_CO), B);
  causal_conv1d_kernel<<<grid, CV_THREADS, smem, stream>>>(x, w, bias, residual, y, B, Cin, Cout, T, Tout, K, stride,
                                                           dilation, pad, pad_mode, act_elu);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_residual_unit_fwd(const float* x, const float* w7_packed, const float* b7, const float* w1_packed,
                                     const float* b1, float* y, int B, int C, int T, int dilation, int pad_mode,
                                     alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && w7_packed && b7 && w1_packed && b1 && y && B > 0 && C > 0 && T > 0 && B <= 65535, ALM_ERR_ARG);
  ALM_REQUIRE(pad_mode >= 0 && pad_mode <= 2, ALM_ERR_ARG);
  ALM_REQUIRE(pad_mode != 0 || 6 * dilation < T, ALM_ERR_ARG);
  ALM_REQUIRE((reinterpret_cast<uintptr_t>(w7_packed) & 15u) == 0 && (reinterpret_cast<uintptr_t>(w1_packed) & 15u) == 0,
              ALM_ERR_ALIGN);
  const int rc = cvt::dispatch_ru(x, w7_packed, b7, w1_packed, b1, y, B, C, T, dilation, pad_mode, stream);
  return rc == -1 ? ALM_ERR_UNSUPPORTED : rc;
}

extern "C" int alm_codec_se_fp32(const float* y, const float* x, const float* w1_folded, const float* b1,
                                 const float* w2, const float* b2, float* out, int B, int C, int Ci, int T,
                                 alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(y && x && w1_folded && b1 && w2 && b2 && out && B > 0 && C > 0 && Ci > 0 && T > 0 && B <= 65535,
              ALM_ERR_ARG);
  const size_t smem = (size_t)(C + Ci) * SE_T * sizeof(float);
  ALM_REQUIRE(smem <= 200 * 1024, ALM_ERR_UNSUPPORTED);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(se_fp32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  dim3 grid(ceil_div(T, SE_T), B);
  se_fp32_kernel<<<grid, SE_T, smem, stream>>>(y, x, w1_folded, b1, w2, b2, out, C, Ci, T);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_causal_convT1d_fwd(const float* x, const float* w, const float* bias, float* y, int B, int Cin,
                                      int Cout, int n, int stride, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && w && y && B > 0 && Cin > 0 && Cout > 0 && n > 0, ALM_ERR_ARG);
  ALM_REQUIRE(stride >= 1 && stride <= CT_MAXS, ALM_ERR_UNSUPPORTED);
  dim3 grid(ceil_div(n, CT_TI), ceil_div(Cout, CT_CO), B);
  causal_convT1d_kernel<<<grid, 256, 0, stream>>>(x, w, bias, y, B, Cin, Cout, n, stride);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_rvq_encode(const float* x, int64_t ldx, const float* codebooks, float* e2_workspace, float* quantized,
                              int64_t ldq, int64_t* indices, int64_t ldi, int N, int D, int C, int Q,
                              alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && codebooks && e2_workspace && quantized && indices, ALM_ERR_ARG);
  ALM_REQUIRE(N > 0 && D > 0 && D % 4 == 0 && C > 0 && Q > 0, ALM_ERR_ARG);
  ALM_REQUIRE(ldx % 4 == 0 || true, ALM_ERR_ALIGN);
  code_norms_kernel<<<ceil_div(Q * C * 32, 256), 256, 0, stream>>>(codebooks, e2_workspace, Q * C, D);
  ALM_CHECK_LAUNCH();
  static const bool rvq_v1 = getenv("ALM_RVQ_V1") != nullptr;  // A/B switch
  if (!rvq_v1 && D % RQ_KC == 0 && ((reinterpret_cast<uintptr_t>(codebooks) & 15u) == 0)) {
    const size_t smem2 = (size_t)(RQ_ROWS * (D + 4) + 2 * RQ_CT * RQ_ES + RQ_ROWS + 2 * RQ_ROWS) * sizeof(float) +
                         (size_t)(2 * RQ_ROWS + RQ_ROWS) * sizeof(int);
    if (smem2 <= 200 * 1024) {
      static size_t attr2 = 0;
      if (smem2 > attr2) {
        ALM_CUDA_OK(cudaFuncSetAttribute(rvq_encode_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
        attr2 = smem2;
      }
      rvq_encode_v2_kernel<<<ceil_div(N, RQ_ROWS), RQ_THREADS, smem2, stream>>>(
          x, ldx, codebooks, e2_workspace, quantized, ldq, reinterpret_cast<long long*>(indices), ldi, N, D, C, Q);
      ALM_CHECK_LAUNCH();
      ALM_LAUNCHED(2);
      return ALM_OK;
    }
  }
  const size_t smem = (size_t)((RV_ROWS + RV_CODES) * (D + 4) + 2 * RV_ROWS) * sizeof(float);
  ALM_REQUIRE(smem <= 200 * 1024, ALM_ERR_UNSUPPORTED);
  static size_t attr = 0;
  if (smem > 48 * 1024 && smem > attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(rvq_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  rvq_encode_kernel<<<ceil_div(N, RV_ROWS), RV_THREADS, smem, stream>>>(
      x, ldx, codebooks, e2_workspace, quantized, ldq, reinterpret_cast<long long*>(indices), ldi, N, D, C, Q);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(2);
  return ALM_OK;
}

extern "C" int alm_rvq_decode(const int64_t* indices, int64_t ldi, const float* codebooks, float* out, int64_t ldo,
                              int N, int D, int C, int Q, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(indices && codebooks && out && N > 0 && D > 0 && C > 0 && Q > 0, ALM_ERR_ARG);
  rvq_decode_kernel<<<N, 128, 0, stream>>>(reinterpret_cast<const long long*>(indices), ldi, codebooks, out, ldo, N,
                                           D, C, Q);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
