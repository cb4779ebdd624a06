// Residual VQ nearest-code search with the distance GEMM on the tensor cores.
//
// Reference: vector-quantize-pytorch ResidualVQ eval path as called at soundstream.py:840 (restated in
// oracle/third_party.py::euclid_nearest): per stage  idx = argmin_c sqrt(max(|r|^2 + |e_c|^2 - 2 r.e_c, 0)),
// lowest index on ties;  r -= e_idx;  quantized += e_idx.
//
// The 2 N C D flops of r.e_c (8.4 MFLOP per frame) are what made the fp32 CUDA-core kernel (codec.cu) FMA-bound.
// Here, per stage:
//   1. S = R' B'^T on the wgmma GEMM (alm_gemm_bf16) with the split-bf16 trick folded into K:
//        R' = [r_hi | r_lo | r_hi]  (N x 3D),  B' = [e_hi | e_hi | e_lo]  (C x 3D)   =>  S ~ r.e to ~2^-16 relative
//   2. rvq_select_kernel (one warp per row): approximate scores a_c = |e_c|^2 - 2 S_c pick the CANDIDATES
//      (everything within the bf16x3 error bound of the best); each candidate's distance is then re-evaluated in
//      fp32 with the reference's expansion and the winner (lowest index on ties) is chosen among them, so the emitted
//      index is the fp32 argmin, not the approximate one.  The warp then updates r, quantized and the next stage's R'.
//
// Cosine mode (VectorQuantize(use_cosine_sim=True), restated in oracle/third_party.py::cosine_nearest): per stage
// idx = argmax_c r^.e_c with r^ = r / max(|r|, 1e-12) (F.normalize), lowest index on ties; e_c is the stored row, not
// re-normalised, and r -= e_idx, quantized += e_idx as above.  R' holds the split of r^ instead of r; the score GEMM is
// unchanged (S ~ r^.e).  Select takes every code within the bf16x3 error window of the best MAXIMUM score, re-ranks
// the candidates by r.e_c in fp32 (r^ is r over a positive scalar, so the ranking is that of r^.e_c, and a zero row
// gives 0 everywhere, so code 0 wins as argmax does), then writes the split of the next r^ after one extra pass for
// its norm.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace rvq {

// one warp per code row: e2 = |e|^2 (fp32, sequential-per-lane + tree), packed = [hi | hi | lo]
__global__ void pack_codebooks_kernel(const float* __restrict__ cb, __nv_bfloat16* __restrict__ packed,
                                      float* __restrict__ e2, long long rows, int D) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float* src = cb + row * D;
  __nv_bfloat16* dst = packed + row * 3 * D;
  float acc = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = src[d];
    acc = fmaf(v, v, acc);
    __nv_bfloat16 hi, lo;
    split_bf16(v, hi, lo);
    dst[d] = hi;
    dst[D + d] = hi;
    dst[2 * D + d] = lo;
  }
  acc = warp_sum(acc);
  if (lane == 0) e2[row] = acc;
}

__device__ __forceinline__ void write_split(__nv_bfloat16* dst, int D, int d, float v) {
  __nv_bfloat16 hi, lo;
  split_bf16(v, hi, lo);
  dst[d] = hi;
  dst[D + d] = lo;
  dst[2 * D + d] = hi;
}

// F.normalize's scale of a row from its squared norm: 1 / max(|r|, 1e-12)
__device__ __forceinline__ float inv_norm(float n2) { return 1.f / fmaxf(sqrtf(n2), 1e-12f); }

// r = x, quantized = 0, R' = [hi | lo | hi] of x (COS: of x / max(|x|, 1e-12)); the Dp - Dx columns past x's width
// are zero
template <bool COS>
__global__ void prepare_kernel(const float* __restrict__ x, long long ldx, float* __restrict__ r,
                               float* __restrict__ quant, long long ldq, __nv_bfloat16* __restrict__ rp, int N, int Dx,
                               int D) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  __nv_bfloat16* dst = rp + (long long)row * 3 * D;
  float n2 = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = d < Dx ? x[(long long)row * ldx + d] : 0.f;
    r[(long long)row * D + d] = v;
    quant[(long long)row * ldq + d] = 0.f;
    if constexpr (COS) n2 = fmaf(v, v, n2);
    else write_split(dst, D, d, v);
  }
  if constexpr (COS) {
    const float s = inv_norm(warp_sum(n2));
    for (int d = lane; d < D; d += 32) write_split(dst, D, d, r[(long long)row * D + d] * s);
  }
}

// >> the error of the bf16x3 scores: the dropped lo x lo terms (~2^-18) plus the fp32 accumulation over K = 3D in the
// GEMM.  Measured max |S - r.e| / (|r|^2 + |e|^2) up to D = 1024: 5.8e-6, i.e. 17x headroom (H100 80GB HBM3, 700 W;
// tests/test_nearest_code_envelope_gpu.py::test_score_window_headroom asserts 4x).
constexpr float CAND_TOL = 1e-4f;

// >> cosine window.  The same GEMM error, |S_c - r^.e_c| <= eps (|r^|^2 + |e_c|^2) with eps <= 5.8e-6 measured, holds
// for the best-scoring code a and for the fp32 winner b, so S_b >= S_a - eps (2 |r^|^2 + |e_a|^2 + |e_b|^2) up to the
// fp32 re-rank's own error; taking every c with S_c >= max S - CAND_TOL_COS (|r^|^2 + max_c |e_c|^2) covers that with
// CAND_TOL_COS / (2 eps) >= 8x headroom for any codebook norms (|r^|^2 is 1, or 0 for a zero row, where every score is 0;
// the window takes 1).  Measured eps on normalised rows up to D = 1024, with unit, generated and rescaled codebooks:
// 6.0e-6, i.e. 17x headroom per code (H100 80GB HBM3, 700 W;
// tests/test_codec_rvq_options_gpu.py::test_cosine_score_window_headroom asserts 4x).
constexpr float CAND_TOL_COS = 1e-4f;

template <bool COS>
__global__ void __launch_bounds__(256)
select_kernel(const float* __restrict__ S, long long ldS, const float* __restrict__ e2, const float* __restrict__ cb,
              float* __restrict__ r, float* __restrict__ quant, long long ldq, __nv_bfloat16* __restrict__ rp,
              long long* __restrict__ idx, long long ldi, int N, int D, int C, int write_rp) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  float* rr = r + (long long)row * D;
  const float* Sr = S + (long long)row * ldS;
  int best_c = 0;
  if constexpr (COS) {
    // pass 1: best approximate score and the largest |e|^2
    float m = -INFINITY, em = 0.f;
    for (int c = lane; c < C; c += 32) {
      m = fmaxf(m, Sr[c]);
      em = fmaxf(em, e2[c]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      em = fmaxf(em, __shfl_xor_sync(0xffffffffu, em, o));
    }
    const float thr = m - CAND_TOL_COS * (1.f + em) - 1e-30f;
    // pass 2: fp32 r.e of every candidate, ascending code index, strict > => lowest index wins ties
    float best = -INFINITY;
    for (int c0 = 0; c0 < C; c0 += 32) {
      const int c = c0 + lane;
      unsigned mask = __ballot_sync(0xffffffffu, c < C && Sr[c] >= thr);
      while (mask) {
        const int cc = c0 + __ffs(mask) - 1;
        mask &= mask - 1;
        const float* e = cb + (long long)cc * D;
        float dot = 0.f;
        for (int d = lane; d < D; d += 32) dot = fmaf(rr[d], e[d], dot);
        dot = warp_sum(dot);
        if (dot > best) {
          best = dot;
          best_c = cc;
        }
      }
    }
  } else {
    float r2 = 0.f;
    for (int d = lane; d < D; d += 32) r2 = fmaf(rr[d], rr[d], r2);
    r2 = warp_sum(r2);
    // pass 1: best approximate score
    float m = INFINITY;
    for (int c = lane; c < C; c += 32) m = fminf(m, e2[c] - 2.f * Sr[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // pass 2: exact fp32 distance of every candidate, ascending code index => lowest index wins ties
    float best = INFINITY;
    for (int c0 = 0; c0 < C; c0 += 32) {
      const int c = c0 + lane;
      bool cand = false;
      if (c < C) {
        const float ec = e2[c];
        cand = (ec - 2.f * Sr[c]) <= m + CAND_TOL * (r2 + ec) + 1e-30f;
      }
      unsigned mask = __ballot_sync(0xffffffffu, cand);
      while (mask) {
        const int bit = __ffs(mask) - 1;
        mask &= mask - 1;
        const int cc = c0 + bit;
        const float* e = cb + (long long)cc * D;
        float dot = 0.f;
        for (int d = lane; d < D; d += 32) dot = fmaf(rr[d], e[d], dot);
        dot = warp_sum(dot);
        const float dist = sqrtf(fmaxf(r2 + e2[cc] - 2.f * dot, 0.f));
        if (dist < best) {
          best = dist;
          best_c = cc;
        }
      }
    }
  }
  if (lane == 0) idx[(long long)row * ldi] = best_c;
  const float* e = cb + (long long)best_c * D;
  __nv_bfloat16* dst = rp + (long long)row * 3 * D;
  float n2 = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float ev = e[d];
    const float nr = rr[d] - ev;
    rr[d] = nr;
    quant[(long long)row * ldq + d] += ev;
    if constexpr (COS) n2 = fmaf(nr, nr, n2);
    else if (write_rp) write_split(dst, D, d, nr);
  }
  if constexpr (COS) {
    if (write_rp) {
      const float s = inv_norm(warp_sum(n2));
      for (int d = lane; d < D; d += 32) write_split(dst, D, d, rr[d] * s);
    }
  }
}

// [hi | lo | hi] of fp32 rows: the A operand of a split-bf16 GEMM (the projections around a residual VQ)
__global__ void split_rows_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ out, int N,
                                  int D) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  for (int d = lane; d < D; d += 32) write_split(out + (long long)row * 3 * D, D, d, x[(long long)row * ldx + d]);
}

}  // namespace rvq
}  // namespace alm

extern "C" int alm_rvq_pack_codebooks(const float* codebooks, void* packed, float* e2, int64_t rows, int D,
                                      alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(codebooks && packed && e2 && rows > 0 && D > 0, ALM_ERR_ARG);
  const int wpb = 8;
  rvq::pack_codebooks_kernel<<<(unsigned)ceil_div<long long>(rows, wpb), wpb * 32, 0, stream>>>(
      codebooks, reinterpret_cast<__nv_bfloat16*>(packed), e2, rows, D);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_rvq_prepare(const float* x, int64_t ldx, float* r, float* quantized, int64_t ldq, void* rp, int N,
                               int Dx, int D, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && r && quantized && rp && N > 0 && Dx > 0 && D >= Dx && ldx >= Dx && ldq >= D, ALM_ERR_ARG);
  const int wpb = 8;
  rvq::prepare_kernel<false><<<ceil_div(N, wpb), wpb * 32, 0, stream>>>(x, ldx, r, quantized, ldq,
                                                                         reinterpret_cast<__nv_bfloat16*>(rp), N, Dx, D);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_rvq_prepare_cos(const float* x, int64_t ldx, float* r, float* quantized, int64_t ldq, void* rp,
                                   int N, int Dx, int D, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && r && quantized && rp && N > 0 && Dx > 0 && D >= Dx && ldx >= Dx && ldq >= D, ALM_ERR_ARG);
  const int wpb = 8;
  rvq::prepare_kernel<true><<<ceil_div(N, wpb), wpb * 32, 0, stream>>>(x, ldx, r, quantized, ldq,
                                                                        reinterpret_cast<__nv_bfloat16*>(rp), N, Dx, D);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

template <bool COS>
static int rvq_select_launch(const float* scores, int64_t lds, const float* e2, const float* codebook, float* r,
                             float* quantized, int64_t ldq, void* rp, int64_t* indices, int64_t ldi, int N, int D,
                             int C, int write_rp, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(scores && e2 && codebook && r && quantized && rp && indices && N > 0 && D > 0 && C > 0, ALM_ERR_ARG);
  const int wpb = 8;
  rvq::select_kernel<COS><<<ceil_div(N, wpb), wpb * 32, 0, stream>>>(
      scores, lds, e2, codebook, r, quantized, ldq, reinterpret_cast<__nv_bfloat16*>(rp),
      reinterpret_cast<long long*>(indices), ldi, N, D, C, write_rp);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_rvq_select(const float* scores, int64_t lds, const float* e2, const float* codebook, float* r,
                              float* quantized, int64_t ldq, void* rp, int64_t* indices, int64_t ldi, int N, int D,
                              int C, int write_rp, alm_stream_t stream) {
  return rvq_select_launch<false>(scores, lds, e2, codebook, r, quantized, ldq, rp, indices, ldi, N, D, C, write_rp,
                                  stream);
}

extern "C" int alm_rvq_select_cos(const float* scores, int64_t lds, const float* e2, const float* codebook, float* r,
                                  float* quantized, int64_t ldq, void* rp, int64_t* indices, int64_t ldi, int N, int D,
                                  int C, int write_rp, alm_stream_t stream) {
  return rvq_select_launch<true>(scores, lds, e2, codebook, r, quantized, ldq, rp, indices, ldi, N, D, C, write_rp,
                                 stream);
}

extern "C" int alm_split_rows(const float* x, int64_t ldx, void* out, int N, int D, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && out && N > 0 && D > 0 && ldx >= D, ALM_ERR_ARG);
  const int wpb = 8;
  rvq::split_rows_kernel<<<ceil_div(N, wpb), wpb * 32, 0, stream>>>(x, ldx, reinterpret_cast<__nv_bfloat16*>(out), N,
                                                                     D);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
