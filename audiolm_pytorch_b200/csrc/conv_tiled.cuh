// Register-tiled causal Conv1d for the SoundStream stacks (soundstream.py:332-345, 362-395), fp32 CUDA cores.
//
// The first-generation kernel (causal_conv1d_kernel in codec.cu) gave each thread a 4 x 4 output tile and spent
// 5 shared-memory loads per 16 FMAs with run-time kernel size / stride / dilation, far below the fp32 FMA peak.
// Here
//   * (K, stride, dilation) are template parameters (the 10 shapes SoundStream uses; anything else falls back),
//     so the tap loop is fully unrolled and all smem offsets are immediates;
//   * a thread owns COT output channels x TQ output samples (8 x 8 = 64 accumulators): per (channel, tap) it
//     issues COT/4 broadcast LDS.128 for the weights + TQ conflict-free LDS.32 for the samples and COT*TQ FMAs;
//   * the staged input is split by phase (sample p -> xs[c][p % S][p / S]) so strided convs read consecutive
//     words across a warp as well;
//   * input-channel stages are double buffered with cp.async (zero-fill handles padding and ragged edges), so the
//     global-load latency of stage n+1 hides behind the FMAs of stage n;
//   * the accumulation order per output is unchanged (input channels ascending, taps ascending, one fp32 FMA
//     chain), so results are bit-identical to the first-generation kernel and the RVQ indices stay bit-exact.
// fp32 on CUDA cores is deliberate: the RVQ code search downstream is compared bit-exactly against the fp32
// oracle; a tf32 / bf16 tensor-core conv would flip near-tie codes.
#pragma once
#include "alm_common.cuh"

namespace alm {
namespace cvt {

// two IEEE fp32 FMAs on a pair of accumulators (sm_90 has no packed f32x2 FMA)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

constexpr int THREADS = 256;
// input channels per pipeline stage: more for short kernels so a stage carries enough FMAs to hide its copies
__host__ __device__ constexpr int ci_of(int K) { return K == 1 ? 32 : (K <= 4 ? 16 : (K <= 10 ? 8 : 4)); }

template <int K, int S, int D, int TQ>
struct Geo {
  static constexpr int CI = ci_of(K);
  static constexpr int T_TILE = 32 * TQ;
  static constexpr int SPAN = (T_TILE - 1) * S + (K - 1) * D + 1;  // padded-signal samples per tile and channel
  static constexpr int LI = (SPAN + S - 1) / S + 1;                 // row length of one phase (+1: bank skew)
  static constexpr int XS = CI * S * LI;                            // floats
};

template <int K, int S, int D, int COT, int TQ>
constexpr size_t smem_bytes() {  // two pipeline stages of (samples + weights)
  return 2 * (size_t)(Geo<K, S, D, TQ>::XS + Geo<K, S, D, TQ>::CI * K * 8 * COT) * sizeof(float);
}

__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  const int sz = valid ? 4 : 0;  // src-size 0: zero fill
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async16f(float* dst_smem, const float* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst_smem);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}

// w is the PACKED weight copy [Cin][K][Cout].  VEC: Cout % 4 == 0 (16-byte weight copies).
template <int K, int S, int D, int COT, int TQ, bool VEC>
__global__ void __launch_bounds__(THREADS, 2)
conv_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
            const float* __restrict__ residual, float* __restrict__ y, int Cin, int Cout, int T, int Tout, int pad,
            int pad_mode, int act) {
  using G = Geo<K, S, D, TQ>;
  constexpr int CI = G::CI;
  constexpr int CO_TILE = 8 * COT;
  constexpr int STAGE = G::XS + CI * K * CO_TILE;  // floats per pipeline stage
  extern __shared__ __align__(16) float smem[];
  const int t0 = blockIdx.x * G::T_TILE, o0 = blockIdx.y * CO_TILE, b = blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int in0 = t0 * S;
  // accumulators as float2 pairs along time (two time steps per weight load); each output sees a single FMA chain
  float2 acc[COT][TQ / 2];
#pragma unroll
  for (int i = 0; i < COT; ++i)
#pragma unroll
    for (int q = 0; q < TQ / 2; ++q) acc[i][q] = make_float2(0.f, 0.f);

  // asynchronous copy of one stage (CI input channels of samples + their weights) into buffer `buf`
  auto issue_stage = [&](int c0, int buf) {
    float* xs = smem + buf * STAGE;
    float* ws = xs + G::XS;
    // samples: warp <-> input channel(s), lanes along time (coalesced), phase-split on the way in
    for (int c = warp; c < CI; c += THREADS / 32) {
      const bool cok = c0 + c < Cin;
      const float* xrow = x + ((size_t)b * Cin + (cok ? c0 + c : 0)) * T;
      float* xrow_s = xs + c * (S * G::LI);
      for (int p = lane; p < G::SPAN; p += 32) {
        const int i = in0 + p;
        int src = i - pad;
        if (i < pad) src = pad_mode == 0 ? pad - i : (pad_mode == 1 ? -1 : 0);
        const bool ok = cok && src >= 0 && src < T;
        cp_async4(xrow_s + (p % S) * G::LI + p / S, xrow + (ok ? src : 0), ok);
      }
    }
    // weights -> ws[c][j][o] from the packed copy [Cin][K][Cout]
    if constexpr (VEC) {
      for (int i = threadIdx.x; i < CI * K * (CO_TILE / 4); i += THREADS) {
        const int o4 = i % (CO_TILE / 4), r = i / (CO_TILE / 4);  // r = c * K + j
        const bool ok = o0 + o4 * 4 < Cout && c0 + r / K < Cin;
        cp_async16f(ws + r * CO_TILE + o4 * 4, w + (ok ? ((size_t)c0 * K + r) * Cout + o0 + o4 * 4 : 0), ok);
      }
    } else {
      for (int i = threadIdx.x; i < CI * K * CO_TILE; i += THREADS) {
        const int o = i % CO_TILE, r = i / CO_TILE;
        const bool ok = o0 + o < Cout && c0 + r / K < Cin;
        cp_async4(ws + r * CO_TILE + o, w + (ok ? ((size_t)c0 * K + r) * Cout + o0 + o : 0), ok);
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  const int n_st = (Cin + CI - 1) / CI;
  issue_stage(0, 0);
  for (int st = 0; st < n_st; ++st) {
    if (st + 1 < n_st) {
      issue_stage((st + 1) * CI, (st + 1) & 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const float* xs = smem + (st & 1) * STAGE;
    const float* ws = xs + G::XS;
    const int c_lim = min(CI, Cin - st * CI);  // channels past Cin were zero-filled; skipping them saves time only
#pragma unroll 1
    for (int c = 0; c < c_lim; ++c) {
      const float* xc = xs + c * (S * G::LI) + lane;
      const float* wc = ws + c * (K * CO_TILE) + warp * COT;
#pragma unroll
      for (int j = 0; j < K; ++j) {
        float wv[COT];
        float2 xv[TQ / 2];
#pragma unroll
        for (int i4 = 0; i4 < COT / 4; ++i4) {
          const float4 t4 = *reinterpret_cast<const float4*>(wc + j * CO_TILE + i4 * 4);
          wv[i4 * 4 + 0] = t4.x; wv[i4 * 4 + 1] = t4.y; wv[i4 * 4 + 2] = t4.z; wv[i4 * 4 + 3] = t4.w;
        }
        const int off = ((j * D) % S) * G::LI + (j * D) / S;  // compile-time after unrolling
#pragma unroll
        for (int q = 0; q < TQ / 2; ++q) xv[q] = make_float2(xc[off + 32 * (2 * q)], xc[off + 32 * (2 * q + 1)]);
#pragma unroll
        for (int i = 0; i < COT; ++i) {
          const float2 w2 = make_float2(wv[i], wv[i]);
#pragma unroll
          for (int q = 0; q < TQ / 2; ++q) acc[i][q] = ffma2(w2, xv[q], acc[i][q]);
        }
      }
    }
    __syncthreads();  // the buffer just consumed is refilled by the copy issued at the top of the next iteration
  }
#pragma unroll
  for (int i = 0; i < COT; ++i) {
    const int o = o0 + warp * COT + i;
    if (o >= Cout) continue;
    const float bv = bias ? __ldg(bias + o) : 0.f;
#pragma unroll
    for (int q = 0; q < TQ; ++q) {
      const int t = t0 + lane + 32 * q;
      if (t >= Tout) continue;
      float v = ((q & 1) ? acc[i][q >> 1].y : acc[i][q >> 1].x) + bv;
      if (act) v = v > 0.f ? v : expm1f(v);
      const size_t idx = ((size_t)b * Cout + o) * Tout + t;
      if (residual) v += residual[idx];
      y[idx] = v;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Fused ResidualUnit (soundstream.py:362-369):  y = x + ELU(b1 + W1 . ELU(b7 + conv7_dil(x)))
// One CTA owns ALL C channels of a time tile, so the k=7 result never leaves the SM: it is written (after bias +
// ELU) to a [C][T_TILE] shared-memory tile and immediately contracted with the 1x1 weights.  Saves the HBM round
// trip of the intermediate and the standalone 1x1 launch (too little work per byte to hide its own latency).  Both contractions keep the channel-ascending single-FMA-chain order of the unfused
// kernels, so the result is bit-identical to conv7 -> conv1.
// Thread tile: COT = C/8 channels x TQ = 64/COT samples (64 accumulators); T_TILE = 32*TQ; C * T_TILE = 16384.
// ------------------------------------------------------------------------------------------------
template <int C, int D>
struct RuGeo {
  static constexpr int K = 7;
  static constexpr int COT = C / 8;
  static constexpr int TQ = 64 / COT;
  static constexpr int T_TILE = 32 * TQ;
  static constexpr int CI = C >= 256 ? 2 : 4;  // small stages: two CTAs (16 warps) per SM with the 64 KB tile
  static constexpr int SPAN = T_TILE - 1 + (K - 1) * D + 1;
  static constexpr int LI = SPAN + 1;
  static constexpr int XS = (CI * LI + 3) & ~3;      // staged samples of one stage (weights after it stay 16-B aligned)
  static constexpr int STAGE = XS + CI * K * C;      // + its k=7 weights
  static constexpr int CI2 = ((STAGE / C) & ~3) < 32 ? ((STAGE / C) & ~3) : 32;  // 1x1 weight rows per stage
  static constexpr int MID = C * T_TILE;
  static constexpr size_t SMEM = (size_t)(2 * STAGE + MID) * sizeof(float);
};

template <int C, int D>
__global__ void __launch_bounds__(THREADS, RuGeo<C, D>::SMEM <= 113 * 1024 ? 2 : 1)
residual_unit_kernel(const float* __restrict__ x, const float* __restrict__ w7 /*[C][7][C] packed*/,
                     const float* __restrict__ b7, const float* __restrict__ w1 /*[C][1][C] packed*/,
                     const float* __restrict__ b1, float* __restrict__ y, int T, int pad_mode) {
  using G = RuGeo<C, D>;
  constexpr int K = G::K, COT = G::COT, TQ = G::TQ, CI = G::CI, STAGE = G::STAGE;
  extern __shared__ __align__(16) float smem[];
  float* mid = smem + 2 * STAGE;  // [C][T_TILE]
  const int t0 = blockIdx.x * G::T_TILE, b = blockIdx.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int pad = D * (K - 1);
  float2 acc[COT][TQ / 2];
#pragma unroll
  for (int i = 0; i < COT; ++i)
#pragma unroll
    for (int q = 0; q < TQ / 2; ++q) acc[i][q] = make_float2(0.f, 0.f);

  auto issue7 = [&](int c0, int buf) {
    float* xs = smem + buf * STAGE;
    float* ws = xs + G::XS;
    for (int c = warp; c < CI; c += THREADS / 32) {
      const float* xrow = x + ((size_t)b * C + c0 + c) * T;
      float* xrow_s = xs + c * G::LI;
      for (int p = lane; p < G::SPAN; p += 32) {
        const int i = t0 + p;
        int src = i - pad;
        if (i < pad) src = pad_mode == 0 ? pad - i : (pad_mode == 1 ? -1 : 0);
        const bool ok = src >= 0 && src < T;
        cp_async4(xrow_s + p, xrow + (ok ? src : 0), ok);
      }
    }
    for (int i = threadIdx.x; i < CI * K * (C / 4); i += THREADS) {
      const int o4 = i % (C / 4), r = i / (C / 4);
      cp_async16f(ws + r * C + o4 * 4, w7 + ((size_t)c0 * K + r) * C + o4 * 4, true);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };

  // ---------------- phase A: dilated k=7 conv over all C input channels ----------------
  constexpr int n_st = C / CI;
  issue7(0, 0);
  for (int st = 0; st < n_st; ++st) {
    if (st + 1 < n_st) {
      issue7((st + 1) * CI, (st + 1) & 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    const float* xs = smem + (st & 1) * STAGE;
    const float* ws = xs + G::XS;
#pragma unroll 1
    for (int c = 0; c < CI; ++c) {
      const float* xc = xs + c * G::LI + lane;
      const float* wc = ws + c * (K * C) + warp * COT;
#pragma unroll
      for (int j = 0; j < K; ++j) {
        float2 xv[TQ / 2];
#pragma unroll
        for (int q = 0; q < TQ / 2; ++q) xv[q] = make_float2(xc[j * D + 32 * (2 * q)], xc[j * D + 32 * (2 * q + 1)]);
#pragma unroll
        for (int i4 = 0; i4 < COT / 4; ++i4) {
          const float4 t4 = *reinterpret_cast<const float4*>(wc + j * C + i4 * 4);
          const float wv[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const float2 w2 = make_float2(wv[u], wv[u]);
#pragma unroll
            for (int q = 0; q < TQ / 2; ++q) acc[i4 * 4 + u][q] = ffma2(w2, xv[q], acc[i4 * 4 + u][q]);
          }
        }
      }
    }
    __syncthreads();
  }
  // ---------------- phase B: bias + ELU -> shared-memory tile; start streaming the 1x1 weights ----------------
  auto issue1 = [&](int c0, int buf) {  // rows c0 .. c0+CI2 of the packed [C][C] matrix (row = input channel)
    float* ws = smem + buf * STAGE;
    for (int i = threadIdx.x; i < G::CI2 * (C / 4); i += THREADS) {
      const int o4 = i % (C / 4), r = i / (C / 4);
      const bool ok = c0 + r < C;
      cp_async16f(ws + r * C + o4 * 4, w1 + (size_t)(ok ? c0 + r : 0) * C + o4 * 4, ok);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  issue1(0, 0);
#pragma unroll
  for (int i = 0; i < COT; ++i) {
    const int o = warp * COT + i;
    const float bv = __ldg(b7 + o);
#pragma unroll
    for (int q = 0; q < TQ; ++q) {
      float v = ((q & 1) ? acc[i][q >> 1].y : acc[i][q >> 1].x) + bv;
      v = v > 0.f ? v : expm1f(v);
      mid[o * G::T_TILE + lane + 32 * q] = v;
    }
  }
#pragma unroll
  for (int i = 0; i < COT; ++i)
#pragma unroll
    for (int q = 0; q < TQ / 2; ++q) acc[i][q] = make_float2(0.f, 0.f);
  // ---------------- phase C: 1x1 conv over the tile ----------------
  constexpr int n_st1 = (C + G::CI2 - 1) / G::CI2;
  for (int st = 0; st < n_st1; ++st) {
    if (st + 1 < n_st1) {
      issue1((st + 1) * G::CI2, (st + 1) & 1);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();  // (first iteration: also publishes the mid tile)
    const float* ws = smem + (st & 1) * STAGE;
    const int c_lim = min(G::CI2, C - st * G::CI2);
#pragma unroll 2
    for (int c = 0; c < c_lim; ++c) {
      const float* mc = mid + (st * G::CI2 + c) * G::T_TILE + lane;
      const float* wc = ws + c * C + warp * COT;
      float2 xv[TQ / 2];
#pragma unroll
      for (int q = 0; q < TQ / 2; ++q) xv[q] = make_float2(mc[32 * (2 * q)], mc[32 * (2 * q + 1)]);
#pragma unroll
      for (int i4 = 0; i4 < COT / 4; ++i4) {
        const float4 t4 = *reinterpret_cast<const float4*>(wc + i4 * 4);
        const float wv[4] = {t4.x, t4.y, t4.z, t4.w};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float2 w2 = make_float2(wv[u], wv[u]);
#pragma unroll
          for (int q = 0; q < TQ / 2; ++q) acc[i4 * 4 + u][q] = ffma2(w2, xv[q], acc[i4 * 4 + u][q]);
        }
      }
    }
    __syncthreads();
  }
  // ---------------- phase D: bias + ELU + skip ----------------
#pragma unroll
  for (int i = 0; i < COT; ++i) {
    const int o = warp * COT + i;
    const float bv = __ldg(b1 + o);
#pragma unroll
    for (int q = 0; q < TQ; ++q) {
      const int t = t0 + lane + 32 * q;
      if (t >= T) continue;
      float v = ((q & 1) ? acc[i][q >> 1].y : acc[i][q >> 1].x) + bv;
      v = v > 0.f ? v : expm1f(v);
      const size_t idx = ((size_t)b * C + o) * T + t;
      y[idx] = v + __ldg(x + idx);
    }
  }
}

template <int C, int D>
inline int launch_ru(const float* x, const float* w7, const float* b7, const float* w1, const float* b1, float* y,
                     int B, int T, int pad_mode, cudaStream_t stream) {
  using G = RuGeo<C, D>;
  static_assert(G::SMEM <= 200 * 1024, "residual unit tile does not fit shared memory");
  static bool attr = false;
  if (!attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(residual_unit_kernel<C, D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)G::SMEM));
    attr = true;
  }
  dim3 grid(ceil_div(T, G::T_TILE), B);
  residual_unit_kernel<C, D><<<grid, THREADS, G::SMEM, stream>>>(x, w7, b7, w1, b1, y, T, pad_mode);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// -1: no specialisation for (C, dilation)
inline int dispatch_ru(const float* x, const float* w7, const float* b7, const float* w1, const float* b1, float* y,
                       int B, int C, int T, int dil, int pad_mode, cudaStream_t stream) {
#define RU_CASE(CC, DD) \
  if (C == CC && dil == DD) return launch_ru<CC, DD>(x, w7, b7, w1, b1, y, B, T, pad_mode, stream);
  RU_CASE(32, 1) RU_CASE(32, 3) RU_CASE(32, 9)
  RU_CASE(64, 1) RU_CASE(64, 3) RU_CASE(64, 9)
  RU_CASE(128, 1) RU_CASE(128, 3) RU_CASE(128, 9)
  RU_CASE(256, 1) RU_CASE(256, 3) RU_CASE(256, 9)
#undef RU_CASE
  return -1;
}

template <int K, int S, int D, int COT, int TQ, bool VEC>
inline int launch(const float* x, const float* w, const float* bias, const float* residual, float* y, int B, int Cin,
                  int Cout, int T, int Tout, int pad, int pad_mode, int act, cudaStream_t stream) {
  constexpr size_t smem = smem_bytes<K, S, D, COT, TQ>();
  static_assert(smem <= 100 * 1024, "conv tile does not fit two CTAs per SM");
  static bool attr = false;
  if (!attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(conv_kernel<K, S, D, COT, TQ, VEC>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)smem));
    attr = true;
  }
  dim3 grid(ceil_div(Tout, Geo<K, S, D, TQ>::T_TILE), ceil_div(Cout, 8 * COT), B);
  conv_kernel<K, S, D, COT, TQ, VEC><<<grid, THREADS, smem, stream>>>(x, w, bias, residual, y, Cin, Cout, T, Tout, pad,
                                                                       pad_mode, act);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// w must be the packed [Cin][K][Cout] copy.  Returns -1 when (K, stride, dilation) has no specialisation.
inline int dispatch(const float* x, const float* w, const float* bias, const float* residual, float* y, int B, int Cin,
                    int Cout, int T, int Tout, int K, int stride, int dil, int pad, int pad_mode, int act,
                    cudaStream_t stream) {
  const bool vec = Cout % 4 == 0 && (reinterpret_cast<uintptr_t>(w) & 15u) == 0;
#define CVT_ARGS x, w, bias, residual, y, B, Cin, Cout, T, Tout, pad, pad_mode, act, stream
#define CVT_CASE(KK, SS, DD, TQQ)                                             \
  if (K == KK && stride == SS && dil == DD) {                                 \
    if (!vec) return launch<KK, SS, DD, 4, TQQ, false>(CVT_ARGS);             \
    if (Cout >= 64) return launch<KK, SS, DD, 8, TQQ, true>(CVT_ARGS);        \
    return launch<KK, SS, DD, 4, TQQ, true>(CVT_ARGS);                        \
  }
  CVT_CASE(7, 1, 1, 8)
  CVT_CASE(7, 1, 3, 8)
  CVT_CASE(7, 1, 9, 8)
  CVT_CASE(1, 1, 1, 8)
  CVT_CASE(3, 1, 1, 8)
  CVT_CASE(4, 2, 1, 8)
  CVT_CASE(6, 3, 1, 4)
  CVT_CASE(8, 4, 1, 4)
  CVT_CASE(10, 5, 1, 4)
  CVT_CASE(16, 8, 1, 4)
#undef CVT_CASE
#undef CVT_ARGS
  return -1;
}

}  // namespace cvt
}  // namespace alm
