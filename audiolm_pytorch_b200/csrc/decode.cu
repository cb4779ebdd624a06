// Incremental (one new token per sequence) attention against a STATIC key/value cache whose fill level lives in
// device memory - the pieces that let a whole decode step be captured once in a CUDA graph and replayed per token
// (config C5: AudioLM.generate with use_kv_cache, audiolm_pytorch.py:1406-1511, 1608-1740, 1896-2039; the
// reference re-concatenates the cache with torch.cat per layer per step, :363-365).
//
//   alm_kv_append        : k_cache[b, *len, :] = kv_new[b, 0:D], v_cache[b, *len, :] = kv_new[b, D:2D]  (D = dim_head)
//   alm_mqa_attn_decode  : o[b, h, :] = softmax_j<=*len( q[b,h,:] . k_cache[b,j,:] * scale (+ bias[h, j]) ) v_cache[b,j,:]
//   alm_decode_bias_row  : bias[h, j] for the new token at position *len (relative-position / cross / fine 2-D bias)
// All three read the cache length from `len` at run time, so the launch parameters never change between steps.
// One warp per (batch, head): lanes stride over the keys with a private online softmax (fp32), then the 32
// partial states are merged with shuffles.  K/V rows are shared by all heads (MQA) and stay in L1/L2.
// The head width D (32, 64 or 128) is a template parameter of the attention kernels; at D = 128 the scaled query sits in
// shared memory (every lane reads the same element: a broadcast) so that the 128 accumulators stay in registers.
#include "alm_common.cuh"

namespace alm {

__global__ void kv_append_kernel(const __nv_bfloat16* __restrict__ kv_new, long long ld, __nv_bfloat16* __restrict__ kc,
                                 __nv_bfloat16* __restrict__ vc, long long cache_bstride, const int* __restrict__ len,
                                 int max_len, int b, int DEC_D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= b * 2 * DEC_D) return;
  const int pos = *len;
  if (pos < 0 || pos >= max_len) return;  // a full cache drops the token (the host sizes the cache for max_length)
  const int bb = i / (2 * DEC_D), c = i % (2 * DEC_D);
  const __nv_bfloat16 v = kv_new[(size_t)bb * ld + c];
  if (c < DEC_D) kc[(size_t)bb * cache_bstride + (size_t)pos * DEC_D + c] = v;
  else vc[(size_t)bb * cache_bstride + (size_t)pos * DEC_D + (c - DEC_D)] = v;
}

// HAS_BIAS: an additive fp32 score bias, one row per head (bias[head * bias_ld + j]) shared by every sequence of the
// batch; the scores are in log2 units (q carries scale * log2 e), so the bias enters as bias * log2 e.
template <int DEC_D, bool HAS_BIAS>
__global__ void __launch_bounds__(256)
mqa_attn_decode_kernel(const __nv_bfloat16* __restrict__ q, long long ldq, const __nv_bfloat16* __restrict__ kc,
                       const __nv_bfloat16* __restrict__ vc, long long cache_bstride, const int* __restrict__ len,
                       int max_len, const uint8_t* __restrict__ key_mask, long long mask_bstride,
                       const float* __restrict__ bias, long long bias_ld, __nv_bfloat16* __restrict__ o, long long ldo,
                       float* __restrict__ partial, int h, float scale_log2) {
  // grid (b, splits): each CTA covers one contiguous slice of the keys (flash-decoding); with splits > 1 the
  // per-slice softmax states go to `partial` [b, splits, h, D + 2] = {m, l, acc[D]} and a second kernel merges them
  const int b = blockIdx.x, split = blockIdx.y, splits = gridDim.y;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int n_all = min(*len + 1, max_len);  // the new token was appended at position *len
  const int chunk = ((n_all + splits - 1) / splits + 31) & ~31;
  const int j_begin = split * chunk;
  const int n_k = min(n_all, j_begin + chunk);
  const __nv_bfloat16* kb = kc + (size_t)b * cache_bstride;
  const __nv_bfloat16* vb = vc + (size_t)b * cache_bstride;
  const uint8_t* mrow = key_mask ? key_mask + (size_t)b * mask_bstride : nullptr;
  constexpr bool Q_SMEM = DEC_D > 64;
  constexpr int QR = Q_SMEM ? 1 : DEC_D;
  __shared__ float q_sh[Q_SMEM ? 8 * DEC_D : 1];   // [warp][D]: launches use at most 8 warps
  for (int head = warp; head < h; head += nwarps) {
    float qreg[QR];
    float* qv = Q_SMEM ? q_sh + warp * DEC_D : qreg;
    {
      const uint4* qp = reinterpret_cast<const uint4*>(q + (size_t)b * ldq + head * DEC_D);
#pragma unroll
      for (int i = 0; i < DEC_D / 8; ++i) {
        const uint4 u = __ldg(qp + i);
        qv[i * 8 + 0] = bf16_lo(u.x) * scale_log2; qv[i * 8 + 1] = bf16_hi(u.x) * scale_log2;
        qv[i * 8 + 2] = bf16_lo(u.y) * scale_log2; qv[i * 8 + 3] = bf16_hi(u.y) * scale_log2;
        qv[i * 8 + 4] = bf16_lo(u.z) * scale_log2; qv[i * 8 + 5] = bf16_hi(u.z) * scale_log2;
        qv[i * 8 + 6] = bf16_lo(u.w) * scale_log2; qv[i * 8 + 7] = bf16_hi(u.w) * scale_log2;
      }
    }
    if constexpr (Q_SMEM) __syncwarp();
    float m = -INFINITY, l = 0.f, acc[DEC_D];
#pragma unroll
    for (int d = 0; d < DEC_D; ++d) acc[d] = 0.f;
    for (int j = j_begin + lane; j < n_k; j += 32) {
      if (mrow != nullptr && mrow[j] == 0) continue;
      const uint4* kp = reinterpret_cast<const uint4*>(kb + (size_t)j * DEC_D);
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < DEC_D / 8; ++i) {
        const uint4 u = kp[i];
        s = fmaf(qv[i * 8 + 0], bf16_lo(u.x), s); s = fmaf(qv[i * 8 + 1], bf16_hi(u.x), s);
        s = fmaf(qv[i * 8 + 2], bf16_lo(u.y), s); s = fmaf(qv[i * 8 + 3], bf16_hi(u.y), s);
        s = fmaf(qv[i * 8 + 4], bf16_lo(u.z), s); s = fmaf(qv[i * 8 + 5], bf16_hi(u.z), s);
        s = fmaf(qv[i * 8 + 6], bf16_lo(u.w), s); s = fmaf(qv[i * 8 + 7], bf16_hi(u.w), s);
      }
      if constexpr (HAS_BIAS) s = fmaf(__ldg(bias + (size_t)head * bias_ld + j), 1.4426950408889634f, s);
      const float m_new = fmaxf(m, s);
      const float alpha = exp2f(m - m_new), p = exp2f(s - m_new);
      l = fmaf(l, alpha, p);
      const uint4* vp = reinterpret_cast<const uint4*>(vb + (size_t)j * DEC_D);
#pragma unroll
      for (int i = 0; i < DEC_D / 8; ++i) {
        const uint4 u = vp[i];
        acc[i * 8 + 0] = fmaf(acc[i * 8 + 0], alpha, p * bf16_lo(u.x)); acc[i * 8 + 1] = fmaf(acc[i * 8 + 1], alpha, p * bf16_hi(u.x));
        acc[i * 8 + 2] = fmaf(acc[i * 8 + 2], alpha, p * bf16_lo(u.y)); acc[i * 8 + 3] = fmaf(acc[i * 8 + 3], alpha, p * bf16_hi(u.y));
        acc[i * 8 + 4] = fmaf(acc[i * 8 + 4], alpha, p * bf16_lo(u.z)); acc[i * 8 + 5] = fmaf(acc[i * 8 + 5], alpha, p * bf16_hi(u.z));
        acc[i * 8 + 6] = fmaf(acc[i * 8 + 6], alpha, p * bf16_lo(u.w)); acc[i * 8 + 7] = fmaf(acc[i * 8 + 7], alpha, p * bf16_hi(u.w));
      }
      m = m_new;
    }
    // merge the 32 per-lane softmax states
    const float m_all = warp_max(m);
    const float f = (m == -INFINITY) ? 0.f : exp2f(m - m_all);
    const float l_all = warp_sum(l * f);
    // lane l keeps channels 64 r + 2 l + {0, 1} of every 64-channel group r (lanes 16.. hold nothing at D = 32)
    constexpr int GROUPS = (DEC_D + 63) / 64;
    float mine0[GROUPS], mine1[GROUPS];
#pragma unroll
    for (int r = 0; r < GROUPS; ++r) mine0[r] = mine1[r] = 0.f;
#pragma unroll
    for (int d = 0; d < DEC_D; ++d) {
      const float t = warp_sum(acc[d] * f);
      if (((d & 63) >> 1) == lane) { if (d & 1) mine1[d >> 6] = t; else mine0[d >> 6] = t; }
    }
    const bool owner = 2 * lane < DEC_D;
    if (partial != nullptr) {
      float* ps = partial + (((size_t)b * splits + split) * h + head) * (DEC_D + 2);
      if (lane == 0) { ps[0] = m_all; ps[1] = l_all; }
#pragma unroll
      for (int r = 0; r < GROUPS; ++r)
        if (owner) { ps[2 + 64 * r + 2 * lane] = mine0[r]; ps[3 + 64 * r + 2 * lane] = mine1[r]; }
    } else {
      const float inv = l_all > 0.f ? 1.f / l_all : 0.f;  // fully masked row -> zeros (as alm_mqa_attn_fwd)
#pragma unroll
      for (int r = 0; r < GROUPS; ++r)
        if (owner)
          *reinterpret_cast<__nv_bfloat162*>(o + (size_t)b * ldo + head * DEC_D + 64 * r + 2 * lane) =
              __floats2bfloat162_rn(mine0[r] * inv, mine1[r] * inv);
    }
    if constexpr (Q_SMEM) __syncwarp();  // the next head of this warp overwrites its q_sh row
  }
}

// o[b, head, :] = sum_s acc_s 2^(m_s - m) / sum_s l_s 2^(m_s - m): one thread per (head, channel)
__global__ void mqa_attn_decode_combine_kernel(const float* __restrict__ partial, __nv_bfloat16* __restrict__ o,
                                               long long ldo, int h, int splits, int DEC_D) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < h * DEC_D; i += blockDim.x) {
    const int head = i / DEC_D, d = i % DEC_D;
    const float* ps = partial + ((size_t)b * splits * h + head) * (DEC_D + 2);
    const size_t sstride = (size_t)h * (DEC_D + 2);
    float m = -INFINITY;
    for (int s2 = 0; s2 < splits; ++s2) m = fmaxf(m, ps[s2 * sstride]);
    float l = 0.f, a = 0.f;
    for (int s2 = 0; s2 < splits; ++s2) {
      const float ms = ps[s2 * sstride];
      const float f = (ms == -INFINITY) ? 0.f : exp2f(ms - m);
      l = fmaf(ps[s2 * sstride + 1], f, l);
      a = fmaf(ps[s2 * sstride + 2 + d], f, a);
    }
    o[(size_t)b * ldo + i] = __float2bfloat16(l > 0.f ? a / l : 0.f);
  }
}

// bias[h, j] (j <= L = *len) of the token at cache position L.  Every bias of the models reduces to one rule over
// per-position int32 coordinates u[t] and classes cls[t]:
//   bias[h, j] = (cls[L] != cls[j] || cls[L] < 0) ? override[h] : table[u[L] - u[j] + c, h]
// (table [rows, h] fp32, override [h] fp32 or null = 0).  A table row outside [0, rows) writes NaN rather than
// reading out of bounds.  Entries j > L are not written (the attention never reads them).
__global__ void decode_bias_row_kernel(const float* __restrict__ table, int rows, const float* __restrict__ override_h,
                                       const int* __restrict__ u, const int* __restrict__ cls, int c,
                                       const int* __restrict__ len, int max_len, float* __restrict__ out, long long ld,
                                       int h) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x, head = blockIdx.y;
  const int L = *len;
  if (L < 0 || L >= max_len || j > L) return;
  const int cl = cls[L];
  float v;
  if (cl < 0 || cls[j] != cl) {
    v = override_h ? override_h[head] : 0.f;
  } else {
    const int r = u[L] - u[j] + c;
    v = (r >= 0 && r < rows) ? table[(size_t)r * h + head] : __int_as_float(0x7fc00000);
  }
  out[(size_t)head * ld + j] = v;
}


// ------------------------------------------------------------------------------------------------
// out[r, n] = sum_k x[r, k] * W[n, k] (+ bias[n])  for a handful of rows r (decode: r = batch <= 8).
// With one or a few rows a "GEMM" is a matrix-vector product bound by reading W once; the 128-row wgmma tile
// kernel would put N/256 CTAs on it (4 CTAs for the FFN down projection).  Here every warp owns output columns
// n, n + warps, ... and streams W rows with 16-byte loads from all SMs; x sits in shared memory.
// Replaces the nn.Linear calls of a decode step (audiolm_pytorch.py:293-303, 255-259, 621).
// ------------------------------------------------------------------------------------------------
constexpr int GV_MAXR = 8, GV_THREADS = 256;

template <int R>
__global__ void __launch_bounds__(GV_THREADS)
gemv_bf16_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, const __nv_bfloat16* __restrict__ W, long long ldw,
                 void* __restrict__ out, int c_fp32, long long ldo, const float* __restrict__ bias, int N, int K) {
  extern __shared__ __align__(16) __nv_bfloat16 xs[];  // [R][Kp]
  const int Kp = (K + 7) & ~7;
  for (int i = threadIdx.x; i < R * Kp; i += GV_THREADS) {
    const int r = i / Kp, k = i - r * Kp;
    xs[i] = k < K ? x[(size_t)r * ldx + k] : __float2bfloat16(0.f);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_warps = gridDim.x * (GV_THREADS / 32);
  for (int n = blockIdx.x * (GV_THREADS / 32) + warp; n < N; n += n_warps) {
    const uint4* wrow = reinterpret_cast<const uint4*>(W + (size_t)n * ldw);
    float acc[R];
#pragma unroll
    for (int r = 0; r < R; ++r) acc[r] = 0.f;
    for (int c = lane; c < Kp / 8; c += 32) {
      const uint4 wv = __ldg(wrow + c);
      const float w8[8] = {bf16_lo(wv.x), bf16_hi(wv.x), bf16_lo(wv.y), bf16_hi(wv.y),
                           bf16_lo(wv.z), bf16_hi(wv.z), bf16_lo(wv.w), bf16_hi(wv.w)};
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const uint4 xv = *reinterpret_cast<const uint4*>(xs + r * Kp + c * 8);
        float a = acc[r];
        a = fmaf(w8[0], bf16_lo(xv.x), a); a = fmaf(w8[1], bf16_hi(xv.x), a);
        a = fmaf(w8[2], bf16_lo(xv.y), a); a = fmaf(w8[3], bf16_hi(xv.y), a);
        a = fmaf(w8[4], bf16_lo(xv.z), a); a = fmaf(w8[5], bf16_hi(xv.z), a);
        a = fmaf(w8[6], bf16_lo(xv.w), a); a = fmaf(w8[7], bf16_hi(xv.w), a);
        acc[r] = a;
      }
    }
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float v = warp_sum(acc[r]) + (bias ? bias[n] : 0.f);
      if (lane == 0) {
        if (c_fp32) reinterpret_cast<float*>(out)[(size_t)r * ldo + n] = v;
        else reinterpret_cast<__nv_bfloat16*>(out)[(size_t)r * ldo + n] = __float2bfloat16(v);
      }
    }
  }
}

}  // namespace alm

using namespace alm;

extern "C" int alm_kv_append_dh(const void* kv_new, int64_t ld, void* k_cache, void* v_cache, int64_t cache_bstride,
                                const int32_t* len, int max_len, int b, int dim_head, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(dim_head == 32 || dim_head == 64 || dim_head == 128, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(kv_new && k_cache && v_cache && len && b > 0 && max_len > 0, ALM_ERR_ARG);
  const int n = b * 2 * dim_head;
  kv_append_kernel<<<ceil_div(n, 256), 256, 0, stream>>>((const __nv_bfloat16*)kv_new, ld, (__nv_bfloat16*)k_cache,
                                                         (__nv_bfloat16*)v_cache, cache_bstride, len, max_len, b,
                                                         dim_head);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_kv_append(const void* kv_new, int64_t ld, void* k_cache, void* v_cache, int64_t cache_bstride,
                             const int32_t* len, int max_len, int b, alm_stream_t stream_) {
  return alm_kv_append_dh(kv_new, ld, k_cache, v_cache, cache_bstride, len, max_len, b, 64, stream_);
}

extern "C" int alm_mqa_attn_decode_dh(const void* q, int64_t ldq, const void* k_cache, const void* v_cache,
                                      int64_t cache_bstride, const int32_t* len, int max_len, const void* key_mask,
                                      int64_t mask_bstride, const float* bias, int64_t bias_ld, void* o, int64_t ldo,
                                      float* workspace, int splits, int b, int h, float scale, int dim_head,
                                      alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(dim_head == 32 || dim_head == 64 || dim_head == 128, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(q && k_cache && v_cache && len && o && b > 0 && h > 0 && max_len > 0, ALM_ERR_ARG);
  ALM_REQUIRE(splits >= 1 && splits <= 64 && (splits == 1 || workspace != nullptr), ALM_ERR_ARG);
  ALM_REQUIRE(bias == nullptr || bias_ld >= max_len, ALM_ERR_ARG);
  ALM_REQUIRE(ldq % 8 == 0 && ldo % 2 == 0 && cache_bstride % 8 == 0, ALM_ERR_ALIGN);
  ALM_REQUIRE((reinterpret_cast<uintptr_t>(q) & 15u) == 0 && (reinterpret_cast<uintptr_t>(k_cache) & 15u) == 0 &&
                  (reinterpret_cast<uintptr_t>(v_cache) & 15u) == 0, ALM_ERR_ALIGN);
  const int threads = 32 * min(h, 8);
  dim3 grid(b, splits);
  auto kernel = dim_head == 32    ? (bias ? mqa_attn_decode_kernel<32, true> : mqa_attn_decode_kernel<32, false>)
                : dim_head == 64  ? (bias ? mqa_attn_decode_kernel<64, true> : mqa_attn_decode_kernel<64, false>)
                                  : (bias ? mqa_attn_decode_kernel<128, true> : mqa_attn_decode_kernel<128, false>);
  kernel<<<grid, threads, 0, stream>>>((const __nv_bfloat16*)q, ldq, (const __nv_bfloat16*)k_cache,
                                       (const __nv_bfloat16*)v_cache, cache_bstride, len, max_len,
                                       (const uint8_t*)key_mask, mask_bstride, bias, bias_ld, (__nv_bfloat16*)o, ldo,
                                       splits > 1 ? workspace : nullptr, h, scale * 1.4426950408889634f);
  ALM_CHECK_LAUNCH();
  if (splits > 1) {
    mqa_attn_decode_combine_kernel<<<b, 256, 0, stream>>>(workspace, (__nv_bfloat16*)o, ldo, h, splits, dim_head);
    ALM_CHECK_LAUNCH();
  }
  ALM_LAUNCHED(splits > 1 ? 2 : 1);
  return ALM_OK;
}

extern "C" int alm_mqa_attn_decode(const void* q, int64_t ldq, const void* k_cache, const void* v_cache,
                                   int64_t cache_bstride, const int32_t* len, int max_len, const void* key_mask,
                                   int64_t mask_bstride, const float* bias, int64_t bias_ld, void* o, int64_t ldo,
                                   float* workspace, int splits, int b, int h, float scale, alm_stream_t stream_) {
  return alm_mqa_attn_decode_dh(q, ldq, k_cache, v_cache, cache_bstride, len, max_len, key_mask, mask_bstride, bias,
                                bias_ld, o, ldo, workspace, splits, b, h, scale, 64, stream_);
}

extern "C" int alm_decode_bias_row(const float* table, int rows, const float* override_h, const int32_t* u,
                                   const int32_t* cls, int c, const int32_t* len, int max_len, float* out, int64_t ld,
                                   int h, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(table && u && cls && len && out && rows > 0 && max_len > 0 && h > 0 && h <= 65535 && ld >= max_len,
              ALM_ERR_ARG);
  dim3 grid(ceil_div(max_len, 256), h);
  decode_bias_row_kernel<<<grid, 256, 0, stream>>>(table, rows, override_h, u, cls, c, len, max_len, out, ld, h);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_gemv_bf16(const void* x, int64_t ldx, const void* W, int64_t ldw, void* out, int c_fp32, int64_t ldo,
                             const float* bias, int rows, int N, int K, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && W && out && rows >= 1 && rows <= GV_MAXR && N > 0 && K > 0, ALM_ERR_ARG);
  ALM_REQUIRE(ldw % 8 == 0 && ldw >= ((K + 7) & ~7) && (reinterpret_cast<uintptr_t>(W) & 15u) == 0, ALM_ERR_ALIGN);
  const int Kp = (K + 7) & ~7;
  const size_t smem = (size_t)rows * Kp * sizeof(__nv_bfloat16);
  ALM_REQUIRE(smem <= 96 * 1024, ALM_ERR_UNSUPPORTED);
  const int grid = min(ceil_div(N, GV_THREADS / 32), 4 * num_sms());
  auto* xp = (const __nv_bfloat16*)x;
  auto* wp = (const __nv_bfloat16*)W;
#define GV_LAUNCH(RR)                                                                                              \
  {                                                                                                                \
    static bool attr = false;                                                                                      \
    if (!attr) {                                                                                                   \
      ALM_CUDA_OK(cudaFuncSetAttribute(gemv_bf16_kernel<RR>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024)); \
      attr = true;                                                                                                 \
    }                                                                                                              \
    gemv_bf16_kernel<RR><<<grid, GV_THREADS, smem, stream>>>(xp, ldx, wp, ldw, out, c_fp32, ldo, bias, N, K);       \
  }
  switch (rows) {
    case 1: GV_LAUNCH(1) break;
    case 2: GV_LAUNCH(2) break;
    case 3: GV_LAUNCH(3) break;
    case 4: GV_LAUNCH(4) break;
    case 5: GV_LAUNCH(5) break;
    case 6: GV_LAUNCH(6) break;
    case 7: GV_LAUNCH(7) break;
    default: GV_LAUNCH(8) break;
  }
#undef GV_LAUNCH
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
