// Residual scalar quantizers of SoundStream, eval path (vector-quantize-pytorch GroupedResidualFSQ / GroupedResidualLFQ
// as called at soundstream.py:563-587, 839-845 and decoded at :691-699), fp32 on CUDA cores.
//
// Both quantize every one of dc dimensions on its own behind the same optional projections, so one kernel pair serves
// both, selected by `mode`:
//   r = project_in(x_g); acc = 0
//   for q < Q:  c = stage(r, q); r -= c; acc += c; index[q] = sum_j digit_j * basis_j
//   quantized_g = project_out(acc)
// FSQ stage (per dimension j): z = r / scale[q][j]; z' = rint(tanh(z + shift) * half_l - offset); c = z' / (L // 2) * scale;
//   digit = z' + L // 2.
// LFQ stage: c = r > 0 ? scale[q][j] : -scale[q][j]; digit = r > 0.
// The per-dimension constants come from the host (torch fp32, the expressions the quantizers use), so nothing here
// recomputes pow / atanh.  Every stage operation is a separately rounded IEEE op (__fmul_rn, __fsub_rn, __fdiv_rn,
// tanhf, rintf): a contracted fma or an approximate tanh moves a rounding boundary and with it an index.
//
// One warp per (row, group).  Lane j < dc owns dimension j through all Q stages; the index of a stage is a warp
// integer sum.  project_in is a lane-strided dot product per output reduced by a butterfly (every lane ends with the
// same sum); project_out broadcasts acc and each lane writes its strided output columns.  The decoder rebuilds every
// code from its index with the same operations and runs the same code-sum + project_out function, so decoding the
// encoder's own indices reproduces its `quantized` bit for bit.
#include "alm_common.cuh"

namespace alm {

constexpr int SQ_MAX_DC = 16;
constexpr int SQ_MAX_Q = 32;
constexpr int SQ_MAX_DG = 1024;
constexpr int SQ_WARPS = 8;
constexpr int SQ_FSQ = 0;
constexpr int SQ_LFQ = 1;

// consts: fp32 [4 + Q, dc] = half_l, offset, shift, L // 2, then scale[q]; ints: int32 [2, dc] = levels, basis.
struct SqParams {
  int N, groups, Dg, dc, Q, mode;
  const float* w_in;     // [groups, dc, Dg]; the projections exist iff Dg != dc (else both are identities)
  const float* b_in;     // [groups, dc]
  const float* w_out_t;  // [groups, dc, Dg] = project_out.weight transposed
  const float* b_out;    // [groups, Dg]
  const float* consts;
  const int* ints;
};

// code of stage q for this lane's dimension (FSQ from z', LFQ from the sign bit); the one place codes are formed
__device__ __forceinline__ float sq_code(const SqParams& p, int j, int q, float zq_or_bit) {
  const float scale = __ldg(p.consts + (size_t)(4 + q) * p.dc + j);
  if (p.mode == SQ_LFQ) return zq_or_bit > 0.f ? scale : -scale;
  return __fmul_rn(__fdiv_rn(zq_or_bit, __ldg(p.consts + 3 * p.dc + j)), scale);
}

// quantized_g[d] = b_out[d] + sum_k W_out[d, k] acc[k] for this warp's row (identity: acc itself); acc lives in lane k
__device__ __forceinline__ void sq_project_out(const SqParams& p, int g, float acc, float* __restrict__ out, int lane) {
  if (p.Dg == p.dc) {
    if (lane < p.dc) out[lane] = acc;
    return;
  }
  float a[SQ_MAX_DC];
#pragma unroll
  for (int k = 0; k < SQ_MAX_DC; ++k) a[k] = __shfl_sync(0xffffffffu, acc, k);
  const float* wt = p.w_out_t + (size_t)g * p.dc * p.Dg;
  const float* bo = p.b_out + (size_t)g * p.Dg;
  for (int d = lane; d < p.Dg; d += 32) {
    float o = __ldg(bo + d);
#pragma unroll
    for (int k = 0; k < SQ_MAX_DC; ++k)
      if (k < p.dc) o = fmaf(__ldg(wt + (size_t)k * p.Dg + d), a[k], o);
    out[d] = o;
  }
}

__global__ void __launch_bounds__(SQ_WARPS * 32)
sq_encode_kernel(SqParams p, const float* __restrict__ x, long long ldx, float* __restrict__ quant, long long ldq,
                 void* __restrict__ indices, int idx64) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * SQ_WARPS + (threadIdx.x >> 5);
  if (wid >= (long long)p.N * p.groups) return;
  const int g = (int)(wid / p.N);
  const int n = (int)(wid - (long long)g * p.N);
  const float* xr = x + (size_t)n * ldx + (size_t)g * p.Dg;
  const int j = lane < p.dc ? lane : 0;

  // r = project_in(x_g), held by lane j
  float r;
  if (p.Dg == p.dc) {
    r = lane < p.dc ? xr[lane] : 0.f;
  } else {
    float part[SQ_MAX_DC];
#pragma unroll
    for (int k = 0; k < SQ_MAX_DC; ++k) part[k] = 0.f;
    const float* wi = p.w_in + (size_t)g * p.dc * p.Dg;
    for (int d = lane; d < p.Dg; d += 32) {
      const float xv = xr[d];
#pragma unroll
      for (int k = 0; k < SQ_MAX_DC; ++k)
        if (k < p.dc) part[k] = fmaf(__ldg(wi + (size_t)k * p.Dg + d), xv, part[k]);
    }
    r = 0.f;
#pragma unroll
    for (int k = 0; k < SQ_MAX_DC; ++k) {
      if (k < p.dc) {
        float v = part[k];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == k) r = v;
      }
    }
    if (lane < p.dc) r = __fadd_rn(r, __ldg(p.b_in + (size_t)g * p.dc + lane));
  }

  const float half_l = __ldg(p.consts + j), offset = __ldg(p.consts + p.dc + j);
  const float shift = __ldg(p.consts + 2 * p.dc + j), hw = __ldg(p.consts + 3 * p.dc + j);
  const int basis = __ldg(p.ints + p.dc + j);
  float acc = 0.f;
  unsigned my_idx = 0;
  for (int q = 0; q < p.Q; ++q) {
    float zq_or_bit;
    if (p.mode == SQ_LFQ) {
      zq_or_bit = r > 0.f ? 1.f : 0.f;
    } else {
      const float z = __fdiv_rn(r, __ldg(p.consts + (size_t)(4 + q) * p.dc + j));
      zq_or_bit = rintf(__fsub_rn(__fmul_rn(tanhf(__fadd_rn(z, shift)), half_l), offset));
    }
    const float c = sq_code(p, j, q, zq_or_bit);
    r = __fsub_rn(r, c);
    acc = __fadd_rn(acc, c);
    const int digit = p.mode == SQ_LFQ ? (int)zq_or_bit : (int)zq_or_bit + (int)hw;
    const unsigned v = __reduce_add_sync(0xffffffffu, lane < p.dc ? (unsigned)(digit * basis) : 0u);
    if (lane == q) my_idx = v;
  }
  if (lane < p.Q) {
    const size_t o = ((size_t)g * p.N + n) * p.Q + lane;
    if (idx64) reinterpret_cast<long long*>(indices)[o] = (long long)my_idx;
    else reinterpret_cast<int*>(indices)[o] = (int)my_idx;
  }
  sq_project_out(p, g, lane < p.dc ? acc : 0.f, quant + (size_t)n * ldq + (size_t)g * p.Dg, lane);
}

// indices [groups, N, Qi] (Qi <= Q leading stages; -1 = dropped) -> out [N, groups * Dg]
__global__ void __launch_bounds__(SQ_WARPS * 32)
sq_decode_kernel(SqParams p, const void* __restrict__ indices, int idx64, int Qi, float* __restrict__ out,
                 long long ldo) {
  const int lane = threadIdx.x & 31;
  const long long wid = (long long)blockIdx.x * SQ_WARPS + (threadIdx.x >> 5);
  if (wid >= (long long)p.N * p.groups) return;
  const int g = (int)(wid / p.N);
  const int n = (int)(wid - (long long)g * p.N);
  const int j = lane < p.dc ? lane : 0;
  const size_t row = ((size_t)g * p.N + n) * Qi;
  long long mine = -1;
  if (lane < Qi)
    mine = idx64 ? reinterpret_cast<const long long*>(indices)[row + lane]
                 : (long long)reinterpret_cast<const int*>(indices)[row + lane];
  const int level = __ldg(p.ints + j), basis = __ldg(p.ints + p.dc + j);
  const int hw = (int)__ldg(p.consts + 3 * p.dc + j);
  float acc = 0.f;
  for (int q = 0; q < Qi; ++q) {
    const long long id = __shfl_sync(0xffffffffu, mine, q);
    if (id < 0) continue;
    const float zq_or_bit = p.mode == SQ_LFQ ? (float)((id / basis) & 1) : (float)((int)((id / basis) % level) - hw);
    acc = __fadd_rn(acc, sq_code(p, j, q, zq_or_bit));
  }
  sq_project_out(p, g, lane < p.dc ? acc : 0.f, out + (size_t)n * ldo + (size_t)g * p.Dg, lane);
}

// the envelope both entries share; ALM_ERR_UNSUPPORTED outside it
static int sq_check(const SqParams& p) {
  ALM_REQUIRE(p.N > 0 && p.consts && p.ints && (p.mode == SQ_FSQ || p.mode == SQ_LFQ), ALM_ERR_ARG);
  ALM_REQUIRE(p.dc >= 1 && p.dc <= SQ_MAX_DC && p.Q >= 1 && p.Q <= SQ_MAX_Q, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(p.groups == 1 || p.groups == 2 || p.groups == 4, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(p.Dg == p.dc || (p.Dg % 4 == 0 && p.Dg <= SQ_MAX_DG), ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(p.Dg == p.dc || (p.w_out_t && p.b_out), ALM_ERR_ARG);
  return ALM_OK;
}

}  // namespace alm

using namespace alm;

extern "C" int alm_sq_encode(const float* x, int64_t ldx, int N, int groups, int Dg, int mode, const float* w_in,
                             const float* b_in, const float* w_out_t, const float* b_out, const float* consts,
                             const int32_t* ints, int dc, int Q, float* quantized, int64_t ldq, void* indices,
                             int idx64, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const SqParams p{N, groups, Dg, dc, Q, mode, w_in, b_in, w_out_t, b_out, consts, ints};
  const int rc = sq_check(p);
  if (rc != ALM_OK) return rc;
  ALM_REQUIRE(p.Dg == p.dc || (w_in && b_in), ALM_ERR_ARG);
  ALM_REQUIRE(x && quantized && indices && ldx >= (int64_t)groups * Dg && ldq >= (int64_t)groups * Dg, ALM_ERR_ARG);
  const long long warps = (long long)N * groups;
  sq_encode_kernel<<<(unsigned)ceil_div<long long>(warps, SQ_WARPS), SQ_WARPS * 32, 0, stream>>>(
      p, x, ldx, quantized, ldq, indices, idx64);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_sq_decode(const void* indices, int idx64, int Qi, int N, int groups, int Dg, int mode,
                             const float* w_out_t, const float* b_out, const float* consts, const int32_t* ints, int dc,
                             int Q, float* out, int64_t ldo, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  const SqParams p{N, groups, Dg, dc, Q, mode, nullptr, nullptr, w_out_t, b_out, consts, ints};
  const int rc = sq_check(p);
  if (rc != ALM_OK) return rc;
  ALM_REQUIRE(indices && out && ldo >= (int64_t)groups * Dg, ALM_ERR_ARG);
  ALM_REQUIRE(Qi >= 1 && Qi <= Q, ALM_ERR_UNSUPPORTED);
  const long long warps = (long long)N * groups;
  sq_decode_kernel<<<(unsigned)ceil_div<long long>(warps, SQ_WARPS), SQ_WARPS * 32, 0, stream>>>(p, indices, idx64, Qi,
                                                                                               out, ldo);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
