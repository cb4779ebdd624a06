// vq-wav2vec feature path (fairseq's wav2vec ConvFeatureExtractionModel and KmeansVectorQuantizer as called by
// FairseqVQWav2Vec, vq_wav2vec.py:75-76): the GroupNorm statistics and the fused norm / activation / skip / log kernel
// around the split-bf16 GEMMs of audiolm_pytorch_b200/vq_wav2vec.py.
//
// wav2vec (v1) normalises every conv output with GroupNorm(1, C) - one mean and variance per clip over all C x T - and
// the quantizer's projection with GroupNorm(G, C).  Both use alm_w2v_group_stats, which reduces in a fixed order with
// no atomics: a first kernel sums fixed chunks of W2V_STATS_ROWS rows in fp64 (shifted by the group's first element),
// a second merges a group's chunks in chunk order.  The chunking depends only on T and C / G, so the statistics of a
// clip are bitwise the same whatever the batch.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace w2v {

constexpr float EPS = 1e-5f;  // fairseq's Fp32GroupNorm (torch's GroupNorm default)
constexpr int ROWS = ALM_W2V_STATS_ROWS;
constexpr int THREADS = 256;

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// fixed-order sum of one double per thread over the block (warp trees, then warp 0 over the warp partials in order)
__device__ __forceinline__ double block_sum_f64(double v, double* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum_f64(v);
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  double s = 0.0;
  if (warp == 0) {
    s = lane < (int)(blockDim.x >> 5) ? sh[lane] : 0.0;
    s = warp_sum_f64(s);
  }
  return s;  // valid in warp 0
}

// one block per (b, g, chunk): part[(bg * nchunk + chunk) * 2 + {0, 1}] = sum (y - shift), sum (y - shift)^2 over rows
// [chunk * ROWS, min(T, (chunk + 1) * ROWS)) and channels [g Cg, (g + 1) Cg), shift = y[b, 0, g Cg]
__global__ void __launch_bounds__(THREADS)
stats_partial_kernel(const float* __restrict__ y, double* __restrict__ part, int T, int C, int G, int nchunk) {
  __shared__ double sh[2][THREADS / 32];
  const long long blk = blockIdx.x;
  const int chunk = (int)(blk % nchunk);
  const long long bg = blk / nchunk;
  const int g = (int)(bg % G);
  const long long b = bg / G;
  const int Cg = C / G, Cg4 = Cg / 4;
  const float* base = y + b * T * C + (long long)g * Cg;
  const double shift = base[0];
  const int t0 = chunk * ROWS;
  const int rows = min(ROWS, T - t0);
  const int n4 = rows * Cg4;
  double s1 = 0.0, s2 = 0.0;
  for (int e = threadIdx.x; e < n4; e += THREADS) {
    const int t = t0 + e / Cg4, c = (e % Cg4) * 4;
    const float4 v = *reinterpret_cast<const float4*>(base + (long long)t * C + c);
    const double d0 = v.x - shift, d1 = v.y - shift, d2 = v.z - shift, d3 = v.w - shift;
    s1 += (d0 + d1) + (d2 + d3);
    s2 = fma(d0, d0, fma(d1, d1, fma(d2, d2, fma(d3, d3, s2))));
  }
  s1 = block_sum_f64(s1, sh[0]);
  s2 = block_sum_f64(s2, sh[1]);
  if (threadIdx.x == 0) {
    part[blk * 2] = s1;
    part[blk * 2 + 1] = s2;
  }
}

// one block per (b, g): merge the chunks in chunk order -> stats[b, g] = {mean, 1 / sqrt(var + eps)} (biased var)
__global__ void __launch_bounds__(THREADS)
stats_merge_kernel(const float* __restrict__ y, const double* __restrict__ part, float* __restrict__ stats, int T,
                   int C, int G, int nchunk) {
  __shared__ double sh[2][THREADS / 32];
  const long long bg = blockIdx.x;
  const int g = (int)(bg % G);
  const long long b = bg / G;
  const int Cg = C / G;
  const double shift = y[b * T * C + (long long)g * Cg];
  const double* p = part + bg * nchunk * 2;
  double s1 = 0.0, s2 = 0.0;
  for (int i = threadIdx.x; i < nchunk; i += THREADS) {
    s1 += p[2 * i];
    s2 += p[2 * i + 1];
  }
  s1 = block_sum_f64(s1, sh[0]);
  s2 = block_sum_f64(s2, sh[1]);
  if (threadIdx.x == 0) {
    const double n = (double)T * Cg;
    const double m = s1 / n;
    const double var = fmax(s2 / n - m * m, 0.0);
    stats[bg * 2] = (float)(shift + m);
    stats[bg * 2 + 1] = (float)(1.0 / sqrt(var + (double)EPS));
  }
}

// F.gelu (erf form), fp32
__device__ __forceinline__ float gelu(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }

__device__ __forceinline__ uint2 pack4(__nv_bfloat16 a, __nv_bfloat16 b, __nv_bfloat16 c, __nv_bfloat16 d) {
  return make_uint2((uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16),
                    (uint32_t)__bfloat16_as_ushort(c) | ((uint32_t)__bfloat16_as_ushort(d) << 16));
}

// four channels [c, c + 4) of row (b, t) per thread:
//   v = (y - mean[b, g]) rstd[b, g] (gamma[c] + beta[c]);  v = act(v)  (0 none, 1 ReLU, 2 GELU)
//   v = (v + residual[b, t * step, c]) * scale   (if residual)
//   v = log(|v| + 1)                              (if log_compress)
// -> out fp32 [B, T, C] and / or split bf16 [B, T, 3C] = [v_hi | v_lo | v_hi]
__global__ void __launch_bounds__(THREADS)
norm_act_kernel(const float* __restrict__ y, const float* __restrict__ stats, const float* __restrict__ gamma,
                const float* __restrict__ beta, int act, const float* __restrict__ residual, int Tr, int step,
                float scale, int log_compress, float* __restrict__ out, __nv_bfloat16* __restrict__ split, int B, int T,
                int C, int G) {
  const int C4 = C / 4, Cg = C / G;
  const long long n = (long long)B * T * C4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4) * 4;
    const long long bt = i / C4;
    const long long t = bt % T, b = bt / T;
    const float* st = stats + (b * G + c / Cg) * 2;
    const float mean = st[0], rstd = st[1];
    const float4 yv = *reinterpret_cast<const float4*>(y + bt * C + c);
    float v[4] = {yv.x, yv.y, yv.z, yv.w};
    float4 rv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (residual) rv = *reinterpret_cast<const float4*>(residual + (b * Tr + t * step) * C + c);
    const float r[4] = {rv.x, rv.y, rv.z, rv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float u = (v[j] - mean) * rstd;
      if (gamma) u = fmaf(u, gamma[c + j], beta[c + j]);
      if (act == 1) u = fmaxf(u, 0.f);
      else if (act == 2) u = gelu(u);
      if (residual) u = (u + r[j]) * scale;
      if (log_compress) u = log1pf(fabsf(u));
      v[j] = u;
    }
    if (out) *reinterpret_cast<float4*>(out + bt * C + c) = make_float4(v[0], v[1], v[2], v[3]);
    if (split) {
      __nv_bfloat16 hi[4], lo[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) split_bf16(v[j], hi[j], lo[j]);
      __nv_bfloat16* row = split + bt * 3 * C;
      const uint2 h = pack4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<uint2*>(row + c) = h;
      *reinterpret_cast<uint2*>(row + C + c) = pack4(lo[0], lo[1], lo[2], lo[3]);
      *reinterpret_cast<uint2*>(row + 2 * C + c) = h;
    }
  }
}

inline unsigned grid_for(long long n, int threads) {
  const long long blocks = ceil_div<long long>(n, threads);
  const long long cap = (long long)num_sms() * 32;
  return (unsigned)(blocks < cap ? blocks : cap);
}

}  // namespace w2v
}  // namespace alm

using alm::ceil_div;

extern "C" int alm_w2v_group_stats(const float* y, float* stats, double* work, int B, int T, int C, int G,
                                   alm_stream_t stream_) {
  ALM_REQUIRE(y && stats && work && B > 0 && T > 0 && C > 0 && G > 0 && C % G == 0 && (C / G) % 4 == 0, ALM_ERR_ARG);
  const int nchunk = ceil_div(T, alm::w2v::ROWS);
  const long long groups = (long long)B * G;
  ALM_REQUIRE(groups * nchunk < (1LL << 31), ALM_ERR_ARG);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream_);
  alm::w2v::stats_partial_kernel<<<(unsigned)(groups * nchunk), alm::w2v::THREADS, 0, s>>>(y, work, T, C, G, nchunk);
  ALM_CHECK_LAUNCH();
  alm::w2v::stats_merge_kernel<<<(unsigned)groups, alm::w2v::THREADS, 0, s>>>(y, work, stats, T, C, G, nchunk);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(2);
  return ALM_OK;
}

extern "C" int alm_w2v_norm_act(const float* y, const float* stats, const float* gamma, const float* beta, int act,
                                const float* residual, int Tr, int step, float scale, int log_compress, float* out,
                                void* split, int B, int T, int C, int G, alm_stream_t stream_) {
  ALM_REQUIRE(y && stats && (out || split) && B > 0 && T > 0 && C > 0 && C % 4 == 0, ALM_ERR_ARG);
  ALM_REQUIRE(G > 0 && C % G == 0 && (C / G) % 4 == 0 && act >= 0 && act <= 2 && !gamma == !beta, ALM_ERR_ARG);
  ALM_REQUIRE(!residual || (step > 0 && (long long)(T - 1) * step < Tr), ALM_ERR_ARG);
  const long long n = (long long)B * T * (C / 4);
  alm::w2v::norm_act_kernel<<<alm::w2v::grid_for(n, alm::w2v::THREADS), alm::w2v::THREADS, 0,
                              reinterpret_cast<cudaStream_t>(stream_)>>>(
      y, stats, gamma, beta, act, residual, Tr, step, scale, log_compress, out,
      reinterpret_cast<__nv_bfloat16*>(split), B, T, C, G);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
