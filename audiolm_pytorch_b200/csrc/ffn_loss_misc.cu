// HBM-bound companions of the tensor-core GEMMs on the transformer path:
//   geglu_ln   : GEGLU + inner LayerNorm of FeedForward (audiolm_pytorch.py:246-260), fwd + bwd
//   ce         : cross entropy with ignore_index, fused forward + d(logits) (audiolm_pytorch.py:1561-1565,
//                1836-1854, 2119-2137)
//   attn_delta : rowsum(dO * O) for the attention backward
//   axpby      : value-residual mix v = 0.5 (v + v_first) (audiolm_pytorch.py:355-358) and its backward
//   cast_pad   : fp32 master weights -> zero-padded bf16 operand copies for the TMA/wgmma GEMMs
#include <stdlib.h>

#include "alm_common.cuh"

namespace alm {

constexpr int FF_THREADS = 256;
constexpr int FF_MAX_CHUNKS = 4;  // inner_pad <= 256*8*4 = 8192

__device__ __forceinline__ void unpack8b(const uint4& u, float (&f)[8]) {
  f[0] = bf16_lo(u.x); f[1] = bf16_hi(u.x); f[2] = bf16_lo(u.y); f[3] = bf16_hi(u.y);
  f[4] = bf16_lo(u.z); f[5] = bf16_hi(u.z); f[6] = bf16_lo(u.w); f[7] = bf16_hi(u.w);
}
__device__ __forceinline__ uint32_t pk2b(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ uint4 pack8b(const float (&f)[8]) {
  return make_uint4(pk2b(f[0], f[1]), pk2b(f[2], f[3]), pk2b(f[4], f[5]), pk2b(f[6], f[7]));
}

template <int N>
__device__ __forceinline__ void block_sum256(float (&v)[N], float* buf /*[N][8]*/) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();  // protect buf from the previous use
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) buf[i * 8 + warp] = v[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < FF_THREADS / 32; ++w) s += buf[i * 8 + w];
    v[i] = s;
  }
}

template <int N, int NT>
__device__ __forceinline__ void block_sum_nt(float (&v)[N], float* buf /*[N][NT/32]*/) {
  constexpr int NW = NT / 32;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = warp_sum(v[i]);
  __syncthreads();  // protect buf from the previous use
  if (lane == 0) {
#pragma unroll
    for (int i = 0; i < N; ++i) buf[i * NW + warp] = v[i];
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < N; ++i) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < NW; ++w) s += buf[i * NW + w];
    v[i] = s;
  }
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.7071067811865476f)); }

__device__ __forceinline__ float gelu_erf_grad(float x) {
  const float cdf = 0.5f * (1.f + erff(x * 0.7071067811865476f));
  const float pdf = 0.3989422804014327f * __expf(-0.5f * x * x);
  return cdf + x * pdf;
}

// h [M, ldh]: a = h[:, 0:inner], gate = h[:, gate_off : gate_off+inner]   ->  gn [M, ldg] (cols >= inner are 0)
template <int NCH, int NT>
__global__ void __launch_bounds__(NT)
geglu_ln_fwd_kernel(const __nv_bfloat16* __restrict__ h, long long ldh, int gate_off,
                    const float* __restrict__ gamma, __nv_bfloat16* __restrict__ gn, long long ldg,
                    float* __restrict__ stats, int M, int inner, int inner_pad) {
  __shared__ float buf[2 * (NT / 32)];
  // software pipeline: the NEXT row's operands are loaded into registers before this row is reduced, so the
  // load latency overlaps the erf / reduction / store phases of the current row (the row after that is pulled
  // towards L2)
  uint4 pa[NCH], pgt[NCH];
  auto load_row = [&](int row, uint4* xa, uint4* xg) {
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
      if (c0 < inner_pad) {
        xa[k] = *reinterpret_cast<const uint4*>(h + (size_t)row * ldh + c0);
        xg[k] = *reinterpret_cast<const uint4*>(h + (size_t)row * ldh + gate_off + c0);
      }
    }
  };
  if ((int)blockIdx.x < M) load_row(blockIdx.x, pa, pgt);
  for (int m = blockIdx.x; m < M; m += gridDim.x) {
    uint4 na[NCH], ngt[NCH];
    if (m + (int)gridDim.x < M) load_row(m + gridDim.x, na, ngt);
    if (m + 2 * (int)gridDim.x < M && (threadIdx.x & 7) == 0) {  // L2 prefetch of the row after next
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const int c0 = (threadIdx.x + k * NT) * 8;
        if (c0 < inner_pad) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(h + (size_t)(m + 2 * gridDim.x) * ldh + c0));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(h + (size_t)(m + 2 * gridDim.x) * ldh + gate_off + c0));
        }
      }
    }
    float g[NCH][8];
    float s12[2] = {0.f, 0.f};  // sum, sum of squares: one block reduction per row
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) g[k][e] = 0.f;
      if (c0 < inner_pad) {
        float a[8], gt[8];
        unpack8b(pa[k], a);
        unpack8b(pgt[k], gt);
        const int nv = min(8, inner - c0);  // 8 except in the row's last (padded) chunk
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float cdf, xpdf;
          gelu_parts(gt[e], cdf, xpdf);
          const float v = e < nv ? gt[e] * cdf * a[e] : 0.f;
          g[k][e] = v;
          s12[0] += v;
          s12[1] = fmaf(v, v, s12[1]);
        }
      }
    }
    block_sum_nt<2, NT>(s12, buf);
    const float mean = s12[0] / inner;
    const float rstd = rsqrtf(fmaxf(s12[1] / inner - mean * mean, 0.f) + 1e-5f);
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
      if (c0 < inner_pad) {
        const int nv = min(8, inner - c0);
        float gm[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (nv == 8) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0));
          const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
          gm[0] = g0.x; gm[1] = g0.y; gm[2] = g0.z; gm[3] = g0.w; gm[4] = g1.x; gm[5] = g1.y; gm[6] = g1.z; gm[7] = g1.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (e < nv) gm[e] = __ldg(gamma + c0 + e);
        }
        float o[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = e < nv ? (g[k][e] - mean) * rstd * gm[e] : 0.f;
        *reinterpret_cast<uint4*>(gn + (size_t)m * ldg + c0) = pack8b(o);
      }
    }
    if (threadIdx.x == 0) {
      stats[(size_t)m * 2] = mean;
      stats[(size_t)m * 2 + 1] = rstd;
    }
#pragma unroll
    for (int k = 0; k < NCH; ++k) { pa[k] = na[k]; pgt[k] = ngt[k]; }
  }
}

template <int NCH, int NT>
__global__ void __launch_bounds__(NT, NT == 512 ? 2 : 1)
geglu_ln_bwd_kernel(const __nv_bfloat16* __restrict__ h, long long ldh, int gate_off,
                    const float* __restrict__ gamma, const float* __restrict__ stats,
                    const __nv_bfloat16* __restrict__ dgn, long long ldg, __nv_bfloat16* __restrict__ dh,
                    float* __restrict__ g_gamma, int M, int inner, int inner_pad) {
  __shared__ float buf[2 * (NT / 32)];
  float gacc[NCH][8];
#pragma unroll
  for (int k = 0; k < NCH; ++k)
#pragma unroll
    for (int e = 0; e < 8; ++e) gacc[k][e] = 0.f;
  for (int m = blockIdx.x; m < M; m += gridDim.x) {
    if (m + (int)gridDim.x < M && (threadIdx.x & 7) == 0) {  // L2 prefetch of this CTA's next row
#pragma unroll
      for (int k = 0; k < NCH; ++k) {
        const int c0 = (threadIdx.x + k * NT) * 8;
        if (c0 < inner_pad) {
          asm volatile("prefetch.global.L2 [%0];" ::"l"(h + (size_t)(m + gridDim.x) * ldh + c0));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(h + (size_t)(m + gridDim.x) * ldh + gate_off + c0));
          asm volatile("prefetch.global.L2 [%0];" ::"l"(dgn + (size_t)(m + gridDim.x) * ldg + c0));
        }
      }
    }
    const float mean = stats[(size_t)m * 2], rstd = stats[(size_t)m * 2 + 1];
    // phase 1 keeps per element: a, ge = gelu(gate), gp = gelu'(gate) and gl = dgn * gamma (one exponential each)
    float a[NCH][8], gp[NCH][8], gl[NCH][8], ge[NCH][8];
    float r2[2] = {0.f, 0.f};
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
#pragma unroll
      for (int e = 0; e < 8; ++e) { a[k][e] = gp[k][e] = gl[k][e] = ge[k][e] = 0.f; }
      if (c0 < inner_pad) {
        float dv[8], gt[8];
        unpack8b(*reinterpret_cast<const uint4*>(h + (size_t)m * ldh + c0), a[k]);
        unpack8b(*reinterpret_cast<const uint4*>(h + (size_t)m * ldh + gate_off + c0), gt);
        unpack8b(*reinterpret_cast<const uint4*>(dgn + (size_t)m * ldg + c0), dv);
        const int nv = min(8, inner - c0);
        float gm[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        if (nv == 8) {
          const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c0));
          const float4 g1 = __ldg(reinterpret_cast<const float4*>(gamma + c0 + 4));
          gm[0] = g0.x; gm[1] = g0.y; gm[2] = g0.z; gm[3] = g0.w; gm[4] = g1.x; gm[5] = g1.y; gm[6] = g1.z; gm[7] = g1.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (e < nv) gm[e] = __ldg(gamma + c0 + e);
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float cdf, xpdf;
          gelu_parts(gt[e], cdf, xpdf);
          const bool ok = e < nv;
          ge[k][e] = ok ? gt[e] * cdf : 0.f;
          gp[k][e] = ok ? cdf + xpdf : 0.f;
          if (!ok) { a[k][e] = 0.f; dv[e] = 0.f; }
          const float xh = (ge[k][e] * a[k][e] - mean) * rstd;
          gl[k][e] = dv[e] * gm[e];
          gacc[k][e] = fmaf(dv[e], xh, gacc[k][e]);
          r2[0] += gl[k][e];
          r2[1] = fmaf(gl[k][e], xh, r2[1]);
        }
      }
    }
    block_sum_nt<2, NT>(r2, buf);
    const float m1 = r2[0] / inner, m2 = r2[1] / inner;
#pragma unroll
    for (int k = 0; k < NCH; ++k) {
      const int c0 = (threadIdx.x + k * NT) * 8;
      if (c0 < inner_pad) {
        const int nv = min(8, inner - c0);
        float da[8], dg8[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float xh = (ge[k][e] * a[k][e] - mean) * rstd;
          const float dg = e < nv ? rstd * (gl[k][e] - m1 - xh * m2) : 0.f;
          da[e] = dg * ge[k][e];
          dg8[e] = dg * a[k][e] * gp[k][e];
        }
        *reinterpret_cast<uint4*>(dh + (size_t)m * ldh + c0) = pack8b(da);
        *reinterpret_cast<uint4*>(dh + (size_t)m * ldh + gate_off + c0) = pack8b(dg8);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < NCH; ++k) {
    const int c0 = (threadIdx.x + k * NT) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e)
      if (c0 + e < inner) atomicAdd(g_gamma + c0 + e, gacc[k][e]);
  }
}


// (The row-per-CTA layout above is the one dispatched; a two-warps-per-row variant was slower at C3 and removed.)

// ---- cross entropy: one CTA per row -----------------------------------------------------------
// loss_rows[r] = lse - logit[label]  (0 when label == ignore)
// dlogits[r, c] = (softmax - onehot) * (*scale_num) / (*scale_den)   as bf16 (0 row when ignored)
__global__ void __launch_bounds__(FF_THREADS)
ce_fwd_bwd_kernel(const float* __restrict__ logits, long long ldl, const long long* __restrict__ labels,
                  long long ignore_index, float* __restrict__ loss_rows, __nv_bfloat16* __restrict__ dlogits,
                  long long ldd, const float* __restrict__ scale_num, const float* __restrict__ scale_den, int V,
                  int Vpad) {
  __shared__ float buf[2 * 8];
  const int r = blockIdx.x;
  const float* row = logits + (size_t)r * ldl;
  const long long label = labels[r];
  const bool ignored = (label == ignore_index);
  float mx[1] = {-INFINITY};
  for (int c = threadIdx.x; c < V; c += FF_THREADS) mx[0] = fmaxf(mx[0], row[c]);
  // block max via the sum helper's buffer
  {
    float v = warp_max(mx[0]);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) buf[threadIdx.x >> 5] = v;
    __syncthreads();
    float m = buf[0];
#pragma unroll
    for (int w = 1; w < FF_THREADS / 32; ++w) m = fmaxf(m, buf[w]);
    mx[0] = m;
  }
  float sm[1] = {0.f};
  for (int c = threadIdx.x; c < V; c += FF_THREADS) sm[0] += __expf(row[c] - mx[0]);
  block_sum256<1>(sm, buf);
  const float lse = mx[0] + logf(sm[0]);
  if (threadIdx.x == 0) loss_rows[r] = ignored ? 0.f : (lse - row[label]);
  if (dlogits != nullptr) {
    const float sc = ignored ? 0.f : (*scale_num) / (*scale_den);
    __nv_bfloat16* drow = dlogits + (size_t)r * ldd;
    for (int c = threadIdx.x; c < Vpad; c += FF_THREADS) {
      float g = 0.f;
      if (c < V && !ignored) g = (__expf(row[c] - lse) - (c == label ? 1.f : 0.f)) * sc;
      drow[c] = __float2bfloat16_rn(g);
    }
  }
}

// ---- delta[b,h,i] = sum_d dO[b,i,h,d] * O[b,i,h,d]   (one warp per (token, head), d = 64) --------
// also zeroes the same (token, head) row of the fp32 dQ workspace of the attention backward (when given)
__global__ void attn_delta_kernel(const __nv_bfloat16* __restrict__ o, long long ldo,
                                  const __nv_bfloat16* __restrict__ d_o, long long lddo, float* __restrict__ delta,
                                  long long dstride, float* __restrict__ dq_acc, int b, int h, int n) {
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int total = b * n * h;
  if (gw >= total) return;
  const int head = gw % h;
  const int tok = gw / h;  // b*n + i
  const uint32_t uo = *reinterpret_cast<const uint32_t*>(o + (size_t)tok * ldo + head * 64 + lane * 2);
  const uint32_t ud = *reinterpret_cast<const uint32_t*>(d_o + (size_t)tok * lddo + head * 64 + lane * 2);
  float v = bf16_lo(uo) * bf16_lo(ud) + bf16_hi(uo) * bf16_hi(ud);
  if (dq_acc != nullptr)
    *reinterpret_cast<float2*>(dq_acc + ((size_t)tok * h + head) * 64 + lane * 2) = make_float2(0.f, 0.f);
  v = warp_sum(v);
  if (lane == 0) {
    const int bi = tok / n, i = tok - bi * n;
    delta[((size_t)bi * h + head) * dstride + i] = v;
  }
}

// ---- out[r, c] = alpha * x[r, c] + beta * y[r, c]   (bf16, 2-D strided, cols % 2 == 0) ---------
__global__ void axpby_bf16_kernel(const __nv_bfloat16* __restrict__ x, long long ldx, float alpha,
                                  const __nv_bfloat16* __restrict__ y, long long ldy, float beta,
                                  __nv_bfloat16* __restrict__ out, long long ldout, long long rows, int cols) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int half = cols / 2;
  if (i >= rows * half) return;
  const long long r = i / half;
  const int c = (int)(i - r * half) * 2;
  const uint32_t ux = *reinterpret_cast<const uint32_t*>(x + r * ldx + c);
  float lo = alpha * bf16_lo(ux), hi = alpha * bf16_hi(ux);
  if (y != nullptr) {
    const uint32_t uy = *reinterpret_cast<const uint32_t*>(y + r * ldy + c);
    lo += beta * bf16_lo(uy);
    hi += beta * bf16_hi(uy);
  }
  *reinterpret_cast<uint32_t*>(out + r * ldout + c) = pk2b(lo, hi);
}

// ---- dst_bf16[r, 0:cols_pad] = src_f32[r, 0:cols] zero padded -----------------------------------
__global__ void cast_pad_kernel(const float* __restrict__ src, long long lds, __nv_bfloat16* __restrict__ dst,
                                long long ldd, long long rows, int cols, int cols_pad) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols_pad) return;
  const long long r = i / cols_pad;
  const int c = (int)(i - r * cols_pad);
  dst[r * ldd + c] = __float2bfloat16_rn(c < cols ? src[r * lds + c] : 0.f);
}

// ---- x[i] *= *s (bf16, contiguous) ---------------------------------------------------------------
__global__ void scale_by_scalar_kernel(__nv_bfloat16* __restrict__ x, const float* __restrict__ s, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  x[i] = __float2bfloat16_rn(__bfloat162float(x[i]) * (*s));
}


// ---- top-k filter + Gumbel-max sampling, one CTA per row (audiolm_pytorch.py:98-117, 1498-1499, 1702-1703) ----
// ids[r] = argmax_c ( keep(c) ? logits[r,c]/temperature + g(uniform[r,c]) : -inf ),  g(u) = -log(-log(u+1e-20)+1e-20)
// keep = the k largest logits of the row (ties at the threshold resolved towards lower indices).
constexpr int SMP_THREADS = 256, SMP_MAXV = 2048;
__global__ void __launch_bounds__(SMP_THREADS)
topk_gumbel_kernel(const float* __restrict__ logits, long long ldl, const float* __restrict__ uniform, long long ldu,
                   long long* __restrict__ ids, int V, int k, float inv_temperature) {
  __shared__ float keys[SMP_MAXV];
  __shared__ float red_v[SMP_THREADS / 32];
  __shared__ int red_i[SMP_THREADS / 32];
  __shared__ int cnt_gt;
  __shared__ unsigned hist[256];
  __shared__ unsigned sel_prefix, sel_remaining;
  const int r = blockIdx.x;
  const float* row = logits + (size_t)r * ldl;
  float thr;
  if (V <= SMP_MAXV) {
    int P = 1;
    while (P < V) P <<= 1;
    for (int i = threadIdx.x; i < P; i += SMP_THREADS) keys[i] = i < V ? row[i] : -INFINITY;
    if (threadIdx.x == 0) cnt_gt = 0;
    __syncthreads();
    // bitonic sort, descending
    for (int size = 2; size <= P; size <<= 1)
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int i = threadIdx.x; i < P / 2; i += SMP_THREADS) {
          const int lo = 2 * i - (i & (stride - 1));
          const int hi = lo + stride;
          const bool desc = ((lo & size) == 0);
          const float a = keys[lo], b = keys[hi];
          if (desc ? (a < b) : (a > b)) { keys[lo] = b; keys[hi] = a; }
        }
        __syncthreads();
      }
    thr = keys[min(k, V) - 1];
  } else {
    // large vocabularies: k-th largest by a 4-pass radix select over the order-preserving integer image of the floats
    auto okey = [](float f) -> unsigned {
      const unsigned u = __float_as_uint(f);
      return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    };
    if (threadIdx.x == 0) { cnt_gt = 0; sel_prefix = 0; sel_remaining = (unsigned)min(k, V); }
    __syncthreads();
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 24 - 8 * pass;
      for (int i = threadIdx.x; i < 256; i += SMP_THREADS) hist[i] = 0;
      __syncthreads();
      const unsigned prefix = sel_prefix;
      const unsigned pmask = pass == 0 ? 0u : (0xFFFFFFFFu << (shift + 8));
      for (int c = threadIdx.x; c < V; c += SMP_THREADS) {
        const unsigned kk = okey(row[c]);
        if ((kk & pmask) == prefix) atomicAdd(&hist[(kk >> shift) & 0xFFu], 1u);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        unsigned rem = sel_remaining;
        int b = 255;
        for (; b > 0; --b) {
          if (hist[b] >= rem) break;
          rem -= hist[b];
        }
        sel_prefix = prefix | ((unsigned)b << shift);
        sel_remaining = rem;
      }
      __syncthreads();
    }
    const unsigned kt = sel_prefix;  // integer image of the k-th largest logit
    thr = __uint_as_float((kt & 0x80000000u) ? (kt & 0x7FFFFFFFu) : ~kt);
  }
  int local = 0;
  for (int c = threadIdx.x; c < V; c += SMP_THREADS) local += row[c] > thr;
  local = (int)warp_sum((float)local);
  if ((threadIdx.x & 31) == 0) atomicAdd(&cnt_gt, local);
  __syncthreads();
  const int ties_allowed = k - cnt_gt;  // how many entries equal to thr are kept (lowest indices first)
  // rank of each tie among ties = number of equal entries with a lower index (V is small: O(V) scan per tie)
  float best = -INFINITY;
  int best_i = 0x7fffffff;
  const float* urow = uniform + (size_t)r * ldu;
  for (int c = threadIdx.x; c < V; c += SMP_THREADS) {
    const float v = row[c];
    bool keep = v > thr;
    if (!keep && v == thr) {
      int before = 0;
      for (int j = 0; j < c; ++j) before += row[j] == thr;
      keep = before < ties_allowed;
    }
    if (keep) {
      const float g = -logf(-logf(urow[c] + 1e-20f) + 1e-20f);
      const float val = v * inv_temperature + g;
      if (val > best || (val == best && c < best_i)) { best = val; best_i = c; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_i, o);
    if (ov > best || (ov == best && oi < best_i)) { best = ov; best_i = oi; }
  }
  if ((threadIdx.x & 31) == 0) { red_v[threadIdx.x >> 5] = best; red_i[threadIdx.x >> 5] = best_i; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < SMP_THREADS / 32; ++w)
      if (red_v[w] > best || (red_v[w] == best && red_i[w] < best_i)) { best = red_v[w]; best_i = red_i[w]; }
    ids[r] = best_i;
  }
}


// ---- plain residual + LayerNorm (num_residual_streams == 1: hyper-connections disabled, the reference wraps each
// branch in Residual(branch), audiolm_pytorch.py:446): r_new = r (+ y);  xn = LN(r_new) * gamma ------------------
// one warp per row, fp32 residual stream, bf16 branch output y / normed output xn / raw copy `rb` (kv projection input)
__global__ void resid_ln_fwd_kernel(const float* __restrict__ r, const __nv_bfloat16* __restrict__ y,
                                    const float* __restrict__ gamma, float* __restrict__ r_new,
                                    __nv_bfloat16* __restrict__ xn, __nv_bfloat16* __restrict__ rb,
                                    float* __restrict__ stats, int M, int d) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* rr = r + (size_t)row * d;
  float s = 0.f;
  for (int c = lane; c < d; c += 32) {
    float v = rr[c] + (y ? __bfloat162float(y[(size_t)row * d + c]) : 0.f);
    if (r_new) r_new[(size_t)row * d + c] = v;
    s += v;
  }
  const float mean = warp_sum(s) / d;
  float q = 0.f;
  for (int c = lane; c < d; c += 32) {
    const float v = rr[c] + (y ? __bfloat162float(y[(size_t)row * d + c]) : 0.f);
    q = fmaf(v - mean, v - mean, q);
  }
  const float rstd = rsqrtf(warp_sum(q) / d + 1e-5f);
  for (int c = lane; c < d; c += 32) {
    const float v = rr[c] + (y ? __bfloat162float(y[(size_t)row * d + c]) : 0.f);
    xn[(size_t)row * d + c] = __float2bfloat16_rn((v - mean) * rstd * gamma[c]);
    if (rb) rb[(size_t)row * d + c] = __float2bfloat16_rn(v);
  }
  if (lane == 0) { stats[(size_t)row * 2] = mean; stats[(size_t)row * 2 + 1] = rstd; }
}

// dr = dr_out (+) LN-backward(dxn) (+) dextra ; g_gamma += dxn * xhat      (r_new is the forward's output)
__global__ void resid_ln_bwd_kernel(const float* __restrict__ r_new, const float* __restrict__ gamma,
                                    const float* __restrict__ stats, const float* __restrict__ dr_out,
                                    const __nv_bfloat16* __restrict__ dxn, const __nv_bfloat16* __restrict__ dextra,
                                    float* __restrict__ dr, __nv_bfloat16* __restrict__ dr_bf16,
                                    float* __restrict__ g_gamma, float out_scale, int M, int d) {
  const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (row >= M) return;
  const float mean = stats[(size_t)row * 2], rstd = stats[(size_t)row * 2 + 1];
  float s1 = 0.f, s2 = 0.f;
  for (int c = lane; c < d; c += 32) {
    const float xh = (r_new[(size_t)row * d + c] - mean) * rstd;
    const float dx = __bfloat162float(dxn[(size_t)row * d + c]);
    const float gl = dx * gamma[c];
    atomicAdd(g_gamma + c, dx * xh);
    s1 += gl;
    s2 = fmaf(gl, xh, s2);
  }
  const float m1 = warp_sum(s1) / d, m2 = warp_sum(s2) / d;
  for (int c = lane; c < d; c += 32) {
    const size_t i = (size_t)row * d + c;
    const float xh = (r_new[i] - mean) * rstd;
    const float gl = __bfloat162float(dxn[i]) * gamma[c];
    float v = rstd * (gl - m1 - xh * m2);
    if (dr_out) v += dr_out[i];
    if (dextra) v += __bfloat162float(dextra[i]);
    v *= out_scale;
    dr[i] = v;
    if (dr_bf16) dr_bf16[i] = __float2bfloat16_rn(v);
  }
}

}  // namespace alm

using namespace alm;

extern "C" int alm_geglu_ln_fwd(const void* h, int64_t ldh, int gate_off, const float* gamma, void* gn, int64_t ldg,
                                float* stats, int M, int inner, int inner_pad, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(M > 0 && inner > 0 && inner_pad >= inner && inner_pad % 8 == 0, ALM_ERR_ARG);
  ALM_REQUIRE(ldh % 8 == 0 && ldg % 8 == 0 && gate_off % 8 == 0, ALM_ERR_ALIGN);
  const int nch = ceil_div(inner_pad / 8, FF_THREADS);
  ALM_REQUIRE(nch <= FF_MAX_CHUNKS, ALM_ERR_UNSUPPORTED);
  const int grid = min(M, num_sms() * 8);
  auto* hp = (const __nv_bfloat16*)h;
  auto* gp = (__nv_bfloat16*)gn;
  if (nch <= 1) geglu_ln_fwd_kernel<1, 256><<<grid, FF_THREADS, 0, stream>>>(hp, ldh, gate_off, gamma, gp, ldg, stats, M, inner, inner_pad);
  else if (nch == 2) geglu_ln_fwd_kernel<2, 256><<<grid, FF_THREADS, 0, stream>>>(hp, ldh, gate_off, gamma, gp, ldg, stats, M, inner, inner_pad);
  else geglu_ln_fwd_kernel<4, 256><<<grid, FF_THREADS, 0, stream>>>(hp, ldh, gate_off, gamma, gp, ldg, stats, M, inner, inner_pad);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_geglu_ln_bwd(const void* h, int64_t ldh, int gate_off, const float* gamma, const float* stats,
                                const void* dgn, int64_t ldg, void* dh, float* g_gamma, int M, int inner,
                                int inner_pad, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(M > 0 && inner > 0 && inner_pad >= inner && inner_pad % 8 == 0, ALM_ERR_ARG);
  ALM_REQUIRE(ldh % 8 == 0 && ldg % 8 == 0 && gate_off % 8 == 0, ALM_ERR_ALIGN);
  const int nch = ceil_div(inner_pad / 8, FF_THREADS);
  ALM_REQUIRE(nch <= FF_MAX_CHUNKS, ALM_ERR_UNSUPPORTED);
  auto* hp = (const __nv_bfloat16*)h;
  auto* dg = (const __nv_bfloat16*)dgn;
  auto* dhp = (__nv_bfloat16*)dh;
  static const int bwd_threads = getenv("ALM_GEGLU_BWD_THREADS") ? atoi(getenv("ALM_GEGLU_BWD_THREADS")) : 512;
  if (bwd_threads == 512 && inner_pad > 2048 && inner_pad <= 4096) {
    // one 8-column chunk per thread: half the registers of the 256-thread layout -> 2 x 512 threads per SM
    const int grid = min(M, num_sms() * 2);
    geglu_ln_bwd_kernel<1, 512><<<grid, 512, 0, stream>>>(hp, ldh, gate_off, gamma, stats, dg, ldg, dhp, g_gamma, M, inner, inner_pad);
    ALM_CHECK_LAUNCH();
    ALM_LAUNCHED(1);
    return ALM_OK;
  }
  const int grid = min(M, num_sms() * 4);
  if (nch <= 1) geglu_ln_bwd_kernel<1, 256><<<grid, FF_THREADS, 0, stream>>>(hp, ldh, gate_off, gamma, stats, dg, ldg, dhp, g_gamma, M, inner, inner_pad);
  else if (nch == 2) geglu_ln_bwd_kernel<2, 256><<<grid, FF_THREADS, 0, stream>>>(hp, ldh, gate_off, gamma, stats, dg, ldg, dhp, g_gamma, M, inner, inner_pad);
  else geglu_ln_bwd_kernel<4, 256><<<grid, FF_THREADS, 0, stream>>>(hp, ldh, gate_off, gamma, stats, dg, ldg, dhp, g_gamma, M, inner, inner_pad);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_ce_fwd_bwd(const float* logits, int64_t ldl, const int64_t* labels, int64_t ignore_index,
                              float* loss_rows, void* dlogits, int64_t ldd, const float* scale_num,
                              const float* scale_den, int rows, int V, int Vpad, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(rows > 0 && V > 0 && Vpad >= V, ALM_ERR_ARG);
  ALM_REQUIRE(dlogits == nullptr || (scale_num && scale_den), ALM_ERR_ARG);
  ce_fwd_bwd_kernel<<<rows, FF_THREADS, 0, stream>>>(logits, ldl, (const long long*)labels, ignore_index,
                                                    loss_rows, (__nv_bfloat16*)dlogits, ldd, scale_num, scale_den, V,
                                                    Vpad);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_attn_delta(const void* o, int64_t ldo, const void* d_o, int64_t lddo, float* delta,
                              int64_t delta_stride, float* dq_acc, int b, int h, int n, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(b > 0 && h > 0 && n > 0, ALM_ERR_ARG);
  const long long warps = (long long)b * h * n;
  const int threads = 256;
  const long long blocks = ceil_div(warps * 32, (long long)threads);
  attn_delta_kernel<<<(unsigned)blocks, threads, 0, stream>>>((const __nv_bfloat16*)o, ldo,
                                                              (const __nv_bfloat16*)d_o, lddo, delta, delta_stride, dq_acc, b, h, n);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_axpby_bf16(const void* x, int64_t ldx, float alpha, const void* y, int64_t ldy, float beta,
                              void* out, int64_t ldout, int64_t rows, int cols, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(rows > 0 && cols > 0 && cols % 2 == 0, ALM_ERR_ARG);
  ALM_REQUIRE(ldx % 2 == 0 && ldy % 2 == 0 && ldout % 2 == 0, ALM_ERR_ALIGN);
  const long long n = rows * (cols / 2);
  axpby_bf16_kernel<<<(unsigned)ceil_div(n, 256LL), 256, 0, stream>>>(
      (const __nv_bfloat16*)x, ldx, alpha, (const __nv_bfloat16*)y, ldy, beta, (__nv_bfloat16*)out, ldout, rows, cols);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_cast_pad_bf16(const float* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int cols,
                                 int cols_pad, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(rows > 0 && cols > 0 && cols_pad >= cols, ALM_ERR_ARG);
  const long long n = rows * cols_pad;
  cast_pad_kernel<<<(unsigned)ceil_div(n, 256LL), 256, 0, stream>>>(src, lds, (__nv_bfloat16*)dst, ldd, rows, cols,
                                                                   cols_pad);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// every weight of a model in ONE launch: desc[i] = {src, dst, rows, cols, cols_pad, lds, ldd} (int64 each), blockIdx.y = i
namespace alm {
__global__ void __launch_bounds__(256) cast_pad_multi_kernel(const long long* __restrict__ desc) {
  const long long* d = desc + 7 * (long long)blockIdx.y;
  const float* src = reinterpret_cast<const float*>(d[0]);
  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(d[1]);
  const long long rows = d[2], cols = d[3], cols_pad = d[4], lds = d[5], ldd = d[6];
  const long long pairs = cols_pad / 2;  // cols_pad is even (multiple of 8)
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < rows * pairs;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / pairs, c = (i - r * pairs) * 2;
    const float a = c < cols ? src[r * lds + c] : 0.f;
    const float b = c + 1 < cols ? src[r * lds + c + 1] : 0.f;
    *reinterpret_cast<__nv_bfloat162*>(dst + r * ldd + c) = __floats2bfloat162_rn(a, b);
  }
}
}  // namespace alm

extern "C" int alm_cast_pad_multi(const int64_t* desc_dev, int n, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(desc_dev && n > 0 && n <= 65535, ALM_ERR_ARG);
  alm::cast_pad_multi_kernel<<<dim3(96, n), 256, 0, stream>>>(reinterpret_cast<const long long*>(desc_dev));
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_scale_by_scalar_bf16(void* x, const float* s, int64_t n, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(n > 0 && s, ALM_ERR_ARG);
  scale_by_scalar_kernel<<<(unsigned)ceil_div((long long)n, 256LL), 256, 0, stream>>>((__nv_bfloat16*)x, s, n);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_topk_gumbel_sample(const float* logits, int64_t ldl, const float* uniform, int64_t ldu, int64_t* ids,
                                      int rows, int V, int k, float temperature, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(logits && uniform && ids && rows > 0 && V > 0 && k > 0 && temperature > 0.f, ALM_ERR_ARG);
  topk_gumbel_kernel<<<rows, SMP_THREADS, 0, stream>>>(logits, ldl, uniform, ldu, reinterpret_cast<long long*>(ids), V,
                                                       k, 1.f / temperature);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_resid_ln_fwd(const float* r, const void* y, const float* gamma, float* r_new, void* xn, void* rb,
                                float* stats, int M, int d, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(r && gamma && xn && stats && M > 0 && d > 0, ALM_ERR_ARG);
  resid_ln_fwd_kernel<<<ceil_div(M * 32, 256), 256, 0, stream>>>(r, (const __nv_bfloat16*)y, gamma, r_new,
                                                                 (__nv_bfloat16*)xn, (__nv_bfloat16*)rb, stats, M, d);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_resid_ln_bwd(const float* r_new, const float* gamma, const float* stats, const float* dr_out,
                                const void* dxn, const void* dextra, float* dr, void* dr_bf16, float* g_gamma,
                                float out_scale, int M, int d, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(r_new && gamma && stats && dxn && dr && g_gamma && M > 0 && d > 0, ALM_ERR_ARG);
  resid_ln_bwd_kernel<<<ceil_div(M * 32, 256), 256, 0, stream>>>(
      r_new, gamma, stats, dr_out, (const __nv_bfloat16*)dxn, (const __nv_bfloat16*)dextra, dr,
      (__nv_bfloat16*)dr_bf16, g_gamma, out_scale, M, d);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// ---- fused head + cross entropy, second half of the forward: soft-max partials of alm_gemm_head_ce(mode 1) -> row LSE / loss
namespace alm {
__global__ void ce_finish_kernel(const float* __restrict__ part, int tiles, const float* __restrict__ lab,
                                 const long long* __restrict__ labels, long long ignore, float* __restrict__ lse,
                                 float* __restrict__ loss_rows, int M) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= M) return;
  const float* pr = part + (size_t)r * tiles * 2;
  float m = -INFINITY;
  for (int t = 0; t < tiles; ++t) m = fmaxf(m, pr[2 * t]);
  float s = 0.f;
  for (int t = 0; t < tiles; ++t) s += pr[2 * t + 1] * exp2f(pr[2 * t] - m);
  const float l = (m + log2f(s)) * 0.6931471805599453f;
  lse[r] = l;
  loss_rows[r] = labels[r] == ignore ? 0.f : l - lab[r];
}
}  // namespace alm

extern "C" int alm_ce_finish(const float* part, int tiles, const float* lab_logit, const int64_t* labels,
                             int64_t ignore_index, float* lse, float* loss_rows, int M, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(part && lab_logit && labels && lse && loss_rows && M > 0 && tiles > 0, ALM_ERR_ARG);
  alm::ce_finish_kernel<<<alm::ceil_div(M, 256), 256, 0, stream>>>(part, tiles, lab_logit,
                                                                   reinterpret_cast<const long long*>(labels),
                                                                   (long long)ignore_index, lse, loss_rows, M);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
