// HuBERT feature path (fairseq HubertModel.extract_features as called by HubertWithKmeans, hubert_kmeans.py:107-112):
// the norm, activation and layout kernels around the split-bf16 GEMMs of audiolm_pytorch_b200/hubert.py.
//
// Every conv and linear of the network runs on alm_gemm_bf16 with the split folded into K, as in rvq_tc.cu: the
// activation operand of a GEMM holds rows [x_hi | x_lo | x_hi] ("split layout", bf16 [rows, 3C]) against weight rows
// [w_hi | w_hi | w_lo].  The kernels here produce that layout from the fp32 residual stream; all arithmetic between
// the GEMMs (bias, GroupNorm, LayerNorm, GELU, residual adds) is fp32.  Reductions run in a fixed order (warp trees,
// fixed-stride per-thread sums, no atomics), so every output is a function of its own clip alone.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace hubert {

constexpr float EPS = 1e-5f;  // every GroupNorm / LayerNorm of fairseq's HuBERT

// F.gelu (erf form), fp32
__device__ __forceinline__ float gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }

__device__ __forceinline__ void store_split(__nv_bfloat16* row, int C, int c, float v) {
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  row[c] = hi;
  row[C + c] = lo;
  row[2 * C + c] = hi;
}

// y[b, t, c] = bias[c] + sum_j w[c, j] x[b, t * stride + j]   (conv 0: one input channel)
__global__ void conv0_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ bias,
                             float* __restrict__ y, int B, int T, int T1, int C, int K, int stride) {
  const long long n = (long long)B * T1 * C;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const long long bt = i / C;
    const int t = (int)(bt % T1);
    const int b = (int)(bt / T1);
    const float* xs = x + (long long)b * T + (long long)t * stride;
    const float* ws = w + (long long)c * K;
    float acc = 0.f;
    for (int j = 0; j < K; ++j) acc = fmaf(ws[j], xs[j], acc);
    y[i] = bias ? acc + bias[c] : acc;
  }
}

// GroupNorm(C, C) statistics over time: stats[b, c] = {mean, 1 / sqrt(var + eps)} of y[b, :, c] (two passes).
// Block (32 channels, 16 time lanes); lane t sums rows t, t + 16, ... in order, then lane 0 sums the 16 partials in order.
__global__ void __launch_bounds__(512) chan_stats_kernel(const float* __restrict__ y, float* __restrict__ stats, int T,
                                                         int C) {
  __shared__ float part[16][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int b = blockIdx.y;
  const float* ys = y + (long long)b * T * C + c;
  const bool ok = c < C;
  float s = 0.f;
  if (ok)
    for (int t = threadIdx.y; t < T; t += 16) s += ys[(long long)t * C];
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  float mean = 0.f;
  for (int i = 0; i < 16; ++i) mean += part[i][threadIdx.x];
  mean /= (float)T;
  __syncthreads();
  float q = 0.f;
  if (ok)
    for (int t = threadIdx.y; t < T; t += 16) {
      const float d = ys[(long long)t * C] - mean;
      q = fmaf(d, d, q);
    }
  part[threadIdx.y][threadIdx.x] = q;
  __syncthreads();
  if (threadIdx.y == 0 && ok) {
    float var = 0.f;
    for (int i = 0; i < 16; ++i) var += part[i][threadIdx.x];
    var /= (float)T;
    stats[((long long)b * C + c) * 2] = mean;
    stats[((long long)b * C + c) * 2 + 1] = 1.f / sqrtf(var + EPS);
  }
}

// mean and 1 / sqrt(var + eps) of a row held in global memory (one warp; two passes; fixed-order warp trees)
__device__ __forceinline__ void row_stats(const float* row, int C, float& mean, float& rstd) {
  const int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += row[c];
  mean = warp_sum(s) / (float)C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = row[c] - mean;
    q = fmaf(d, d, q);
  }
  rstd = 1.f / sqrtf(warp_sum(q) / (float)C + EPS);
}

// one warp per row m of y [M, C]:  v = y (+ bias);  mode 1: v = (v - mean[b, c]) rstd[b, c] gamma + beta with
// b = m / rows_per_batch (GroupNorm);  mode 2: LayerNorm over the row;  v = gelu(v) if gelu;  -> out fp32 and / or
// the split layout.  In mode 2 the biased row is first written to `out` (which must then be given) and re-read.
__global__ void __launch_bounds__(256)
norm_act_kernel(const float* __restrict__ y, const float* __restrict__ bias, int mode, const float* __restrict__ stats,
                long long rows_per_batch, const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                float* out, __nv_bfloat16* __restrict__ split, long long M, int C) {
  const long long m = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (m >= M) return;
  const float* yr = y + m * C;
  float* orow = out ? out + m * C : nullptr;
  __nv_bfloat16* srow = split ? split + m * 3 * C : nullptr;
  float mean = 0.f, rstd = 1.f;
  const float* st = mode == 1 ? stats + (m / rows_per_batch) * C * 2 : nullptr;
  if (mode == 2) {
    if (bias) {
      for (int c = lane; c < C; c += 32) orow[c] = yr[c] + bias[c];
      __syncwarp();
      yr = orow;
    }
    row_stats(yr, C, mean, rstd);
  }
  for (int c = lane; c < C; c += 32) {
    float v = yr[c];
    if (bias && mode != 2) v += bias[c];
    if (mode == 1) v = (v - st[2 * c]) * st[2 * c + 1] * gamma[c] + beta[c];
    if (mode == 2) v = (v - mean) * rstd * gamma[c] + beta[c];
    if (act) v = gelu(v);
    if (orow) orow[c] = v;
    if (srow) store_split(srow, C, c, v);
  }
}

// one warp per row m = b * T + t of the residual stream r [M, D]:
//   r_new = r + act(y + y_bias)   (y may be null; y is [M, D], or with groups > 1 the grouped conv output
//                                  [B, groups, T, D / groups]; act = gelu if y_gelu)
//   gamma == null: r_out = r_new.   Otherwise ln = LayerNorm(r_new) gamma + beta, split <- ln (if given) and
//   r_out = keep_ln ? ln : r_new.  r_out may alias r.
__global__ void __launch_bounds__(256)
add_ln_kernel(const float* r, const float* __restrict__ y, int groups, int T, const float* __restrict__ y_bias,
              int y_gelu, const float* __restrict__ gamma, const float* __restrict__ beta, int keep_ln, float* r_out,
              __nv_bfloat16* __restrict__ split, long long M, int D) {
  const long long m = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (m >= M) return;
  const float* rr = r + m * D;
  float* ro = r_out + m * D;
  const int Dg = D / groups;
  const long long b = m / T, t = m % T;
  for (int c = lane; c < D; c += 32) {
    float v = rr[c];
    if (y) {
      const float yv = groups > 1 ? y[((b * groups + c / Dg) * T + t) * Dg + c % Dg] : y[m * D + c];
      float u = y_bias ? yv + y_bias[c] : yv;
      if (y_gelu) u = gelu(u);
      v += u;
    }
    ro[c] = v;
  }
  if (!gamma) return;
  __syncwarp();
  float mean, rstd;
  row_stats(ro, D, mean, rstd);
  __nv_bfloat16* srow = split ? split + m * 3 * D : nullptr;
  for (int c = lane; c < D; c += 32) {
    const float v = (ro[c] - mean) * rstd * gamma[c] + beta[c];
    if (srow) store_split(srow, D, c, v);
    if (keep_ln) ro[c] = v;
  }
}

// group-major, zero-padded split copy of x [B, T, D] for the grouped positional conv:
// xp[b, g, p, :] = split(x[b, p - pad, g * Dg : (g + 1) * Dg]) for p in [0, Tp), zeros outside [0, T)
__global__ void pos_pack_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ xp, int B, int T, int D,
                                int groups, int pad, int Tp) {
  const int Dg = D / groups;
  const long long n = (long long)B * groups * Tp * Dg;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % Dg);
    const long long row = i / Dg;  // (b * groups + g) * Tp + p
    const int p = (int)(row % Tp);
    const long long bg = row / Tp;
    const int g = (int)(bg % groups);
    const long long b = bg / groups;
    const int t = p - pad;
    const float v = (t >= 0 && t < T) ? x[(b * T + t) * D + g * Dg + c] : 0.f;
    store_split(xp + row * 3 * Dg, Dg, c, v);
  }
}

// qkv fp32 [B, T, 3D] (q | k | v, biases included) -> q, k, v bf16 [B, heads, T, dh], the per-head sequences of an
// attention call with batch B * heads and one head
__global__ void qkv_heads_kernel(const float* __restrict__ qkv, __nv_bfloat16* __restrict__ q,
                                 __nv_bfloat16* __restrict__ k, __nv_bfloat16* __restrict__ v, int B, int T, int D,
                                 int heads) {
  const int dh = D / heads;
  const long long n = (long long)B * T * 3 * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int col = (int)(i % (3 * D));
    const long long bt = i / (3 * D);
    const long long t = bt % T, b = bt / T;
    const int which = col / D, h = (col % D) / dh, d = col % dh;
    __nv_bfloat16* dst = which == 0 ? q : which == 1 ? k : v;
    dst[((b * heads + h) * T + t) * dh + d] = __float2bfloat16_rn(qkv[i]);
  }
}

// attention output o bf16 [B, heads, T, dh] -> split layout [B, T, 3D] of the concatenated heads: a bf16 value is
// its own hi half, so the row is [o | 0 | o]
__global__ void merge_heads_kernel(const __nv_bfloat16* __restrict__ o, __nv_bfloat16* __restrict__ split, int B,
                                   int T, int D, int heads) {
  const int dh = D / heads;
  const long long n = (long long)B * T * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % D);
    const long long bt = i / D;
    const long long t = bt % T, b = bt / T;
    const __nv_bfloat16 val = o[((b * heads + c / dh) * T + t) * dh + c % dh];
    __nv_bfloat16* row = split + bt * 3 * D;
    row[c] = val;
    row[D + c] = __float2bfloat16_rn(0.f);
    row[2 * D + c] = val;
  }
}

inline unsigned grid_for(long long n, int threads) {
  const long long blocks = ceil_div<long long>(n, threads);
  const long long cap = (long long)num_sms() * 32;
  return (unsigned)(blocks < cap ? blocks : cap);
}

}  // namespace hubert
}  // namespace alm

using alm::ceil_div;

extern "C" int alm_hubert_conv0(const float* wave, const float* w, const float* bias, float* y, int B, int T, int C,
                                int K, int stride, alm_stream_t stream_) {
  ALM_REQUIRE(wave && w && y && B > 0 && C > 0 && K > 0 && stride > 0 && T >= K, ALM_ERR_ARG);
  const int T1 = (T - K) / stride + 1;
  const long long n = (long long)B * T1 * C;
  alm::hubert::conv0_kernel<<<alm::hubert::grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      wave, w, bias, y, B, T, T1, C, K, stride);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_hubert_chan_stats(const float* y, float* stats, int B, int T, int C, alm_stream_t stream_) {
  ALM_REQUIRE(y && stats && B > 0 && T > 0 && C > 0 && B <= 65535, ALM_ERR_ARG);
  alm::hubert::chan_stats_kernel<<<dim3(ceil_div(C, 32), B), dim3(32, 16), 0,
                                   reinterpret_cast<cudaStream_t>(stream_)>>>(y, stats, T, C);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_hubert_norm_act(const float* y, const float* bias, int mode, const float* stats,
                                   int64_t rows_per_batch, const float* gamma, const float* beta, int gelu, float* out,
                                   void* split, int64_t M, int C, alm_stream_t stream_) {
  ALM_REQUIRE(y && M > 0 && C > 0 && (out || split) && mode >= 0 && mode <= 2, ALM_ERR_ARG);
  ALM_REQUIRE(mode == 0 || (gamma && beta), ALM_ERR_ARG);
  ALM_REQUIRE(mode != 1 || (stats && rows_per_batch > 0), ALM_ERR_ARG);
  ALM_REQUIRE(mode != 2 || !bias || out, ALM_ERR_ARG);
  const int wpb = 8;
  alm::hubert::norm_act_kernel<<<(unsigned)ceil_div<long long>(M, wpb), wpb * 32, 0,
                                 reinterpret_cast<cudaStream_t>(stream_)>>>(
      y, bias, mode, stats, rows_per_batch, gamma, beta, gelu, out, reinterpret_cast<__nv_bfloat16*>(split), M, C);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_hubert_add_ln(const float* r, const float* y, int groups, int T, const float* y_bias, int y_gelu,
                                 const float* gamma, const float* beta, int keep_ln, float* r_out, void* split,
                                 int64_t M, int D, alm_stream_t stream_) {
  ALM_REQUIRE(r && r_out && M > 0 && D > 0 && T > 0 && M % T == 0 && groups >= 1 && D % groups == 0, ALM_ERR_ARG);
  ALM_REQUIRE(!gamma == !beta, ALM_ERR_ARG);
  const int wpb = 8;
  alm::hubert::add_ln_kernel<<<(unsigned)ceil_div<long long>(M, wpb), wpb * 32, 0,
                               reinterpret_cast<cudaStream_t>(stream_)>>>(
      r, y, groups, T, y_bias, y_gelu, gamma, beta, keep_ln, r_out, reinterpret_cast<__nv_bfloat16*>(split), M, D);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_hubert_pos_pack(const float* x, void* xp, int B, int T, int D, int groups, int pad, int Tp,
                                   alm_stream_t stream_) {
  ALM_REQUIRE(x && xp && B > 0 && T > 0 && groups > 0 && D % groups == 0 && pad >= 0 && Tp >= T + pad, ALM_ERR_ARG);
  const long long n = (long long)B * Tp * D;
  alm::hubert::pos_pack_kernel<<<alm::hubert::grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      x, reinterpret_cast<__nv_bfloat16*>(xp), B, T, D, groups, pad, Tp);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_hubert_qkv_heads(const float* qkv, void* q, void* k, void* v, int B, int T, int D, int heads,
                                    alm_stream_t stream_) {
  ALM_REQUIRE(qkv && q && k && v && B > 0 && T > 0 && heads > 0 && D % heads == 0, ALM_ERR_ARG);
  const long long n = (long long)B * T * 3 * D;
  alm::hubert::qkv_heads_kernel<<<alm::hubert::grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      qkv, reinterpret_cast<__nv_bfloat16*>(q), reinterpret_cast<__nv_bfloat16*>(k),
      reinterpret_cast<__nv_bfloat16*>(v), B, T, D, heads);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_hubert_merge_heads(const void* o, void* split, int B, int T, int D, int heads,
                                      alm_stream_t stream_) {
  ALM_REQUIRE(o && split && B > 0 && T > 0 && heads > 0 && D % heads == 0, ALM_ERR_ARG);
  const long long n = (long long)B * T * D;
  alm::hubert::merge_heads_kernel<<<alm::hubert::grid_for(n, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream_)>>>(
      reinterpret_cast<const __nv_bfloat16*>(o), reinterpret_cast<__nv_bfloat16*>(split), B, T, D, heads);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
