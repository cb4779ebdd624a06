// EnCodec 24 kHz (EncodecWrapper, encodec.py) kernels on CUDA cores: the 2-layer LSTM block (fp32 or C8S in and out),
// the fp32 SEANet resnet block of the CUDA-core plan, and the reflect padding of inputs too short for a plain reflect.
// The tensor-core resnet block is ru_tc_kernel's RB mode (codec_tc.cu); the convs run on the SoundStream kernels.
// See include/alm_b200.h for the contracts.
#include <algorithm>

#include "alm_common.cuh"

namespace alm {
namespace encodec {

__device__ __forceinline__ float elu(float v) { return v > 0.f ? v : expm1f(v); }

// ---- reflect padding ------------------------------------------------------------------------------
// EnCodec's _pad1d: when L <= max(pl, pr) the input is first zero-extended to max(pl, pr) + 1 samples, reflected,
// and the extension trimmed off again.  Position q of the padded row (q = -pl .. L + pr - 1) reads x[j] with j the
// reflection of q in the extended row, and 0 where j lands in the extension.
__global__ void pad1d_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t rows, int L, int pl, int pr) {
  const int Lp = L + pl + pr;
  const int mx = pl > pr ? pl : pr;
  const int L0 = L <= mx ? mx + 1 : L;
  const int64_t n = rows * Lp;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / Lp;
    const int q = (int)(e - r * Lp) - pl;
    const int j = q < 0 ? -q : (q < L0 ? q : 2 * (L0 - 1) - q);
    y[e] = j < L ? x[r * L + j] : 0.f;
  }
}

// ---- SEANet resnet block --------------------------------------------------------------------------
// y = Ws x + bs + W1 ELU(W3 * ELU(x) + b3) + b1 (ELU(y) when elu_out); W3 k3 causal, reflect-left pad 2.
// A CTA owns RB_TT time steps of one clip and every channel: x (raw and ELU'd, with the 2-sample halo) and the hidden
// activations stay in shared memory.  Every sum runs over its inputs in one fixed order.
constexpr int RB_TT = 32;
constexpr int RB_THREADS = 256;

__global__ void __launch_bounds__(RB_THREADS) resblock_kernel(const float* __restrict__ x, const float* __restrict__ w3,
                                                              const float* __restrict__ b3, const float* __restrict__ w1,
                                                              const float* __restrict__ ws, const float* __restrict__ bo,
                                                              float* __restrict__ y, int C, int T, int elu_out) {
  extern __shared__ float sm[];
  const int H = C / 2, W = RB_TT + 2;
  float* xs = sm;            // [C][W] raw x
  float* es = xs + C * W;    // [C][W] ELU(x)
  float* hs = es + C * W;    // [H][RB_TT]
  const int b = blockIdx.y, t0 = blockIdx.x * RB_TT;
  const float* xb = x + (int64_t)b * C * T;
  for (int e = threadIdx.x; e < C * W; e += RB_THREADS) {
    const int c = e / W, tt = t0 + e % W - 2;
    float v = 0.f;
    if (tt < 0) {
      if (-tt < T) v = xb[(int64_t)c * T - tt];  // reflect (the zero-extension of _pad1d when T <= 2)
    } else if (tt < T) {
      v = xb[(int64_t)c * T + tt];
    }
    xs[e] = v;
    es[e] = elu(v);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = warp; j < H; j += RB_THREADS / 32) {
    float acc = b3[j];
    const float* wj = w3 + (int64_t)j * C * 3;
    for (int c = 0; c < C; ++c) {
      const float* e = es + c * W + lane;
      acc = fmaf(wj[3 * c], e[0], acc);
      acc = fmaf(wj[3 * c + 1], e[1], acc);
      acc = fmaf(wj[3 * c + 2], e[2], acc);
    }
    hs[j * RB_TT + lane] = elu(acc);
  }
  __syncthreads();
  const int t = t0 + lane;
  for (int o = warp; o < C; o += RB_THREADS / 32) {
    float acc = bo[o];
    const float* w1o = w1 + (int64_t)o * H;
    for (int j = 0; j < H; ++j) acc = fmaf(w1o[j], hs[j * RB_TT + lane], acc);
    const float* wso = ws + (int64_t)o * C;
    for (int c = 0; c < C; ++c) acc = fmaf(wso[c], xs[c * W + lane + 2], acc);
    if (t < T) y[((int64_t)b * C + o) * T + t] = elu_out ? elu(acc) : acc;
  }
}

// ---- LSTM block -----------------------------------------------------------------------------------
// y = LSTM2(LSTM1(x)) + x over H = 512 channels, zero initial state, one persistent cooperative grid of H / 4 CTAs.
// CTA k owns hidden units 4k..4k+3 of both layers: 32 gate rows (layer, gate i/f/g/o, unit) whose [W_ih | W_hh] rows
// (1024 floats each) stay in shared memory.  Phase s (0..T) runs layer 1 at step s and layer 2 at step s - 1, so the
// two layers share T + 1 device-wide barriers; h of both layers is double-buffered in global memory.
constexpr int LH = 512;
constexpr int L_UNITS = 4;
constexpr int L_GRID = LH / L_UNITS;
constexpr int L_ROWS = 32;
constexpr int L_K = 2 * LH;
constexpr int L_NB = 8;  // batch items per pass: a warp's 4 units x 8 items = one value per lane after the reduction
constexpr int L_THREADS = 256;
constexpr size_t L_SMEM = (size_t)(L_ROWS * L_K + L_NB * 3 * LH + 2 * 4 * L_UNITS * L_NB) * sizeof(float);

struct LstmArgs {
  const void* x;       // fp32 [B][H][T], or C8S bf16 [B][2H/8][T][8] when c8s
  const float* w;      // [L_GRID][L_ROWS][L_K] (ops.encodec_lstm_pack)
  const float* bias;   // [L_GRID][L_ROWS], b_ih + b_hh
  void* y;             // the layout of x
  float* xt;           // [T][B][H]
  float* h1;           // [2][B][H]
  float* h2;           // [2][B][H]
  float* c;            // [2][B][H]
  unsigned* counter;
  int* err;
  int B, T, elu_out, c8s;
};

// element (b, c, t) of a C8S tensor with P = 1 and H channels: hi at chunk c / 8, lo at chunk H / 8 + c / 8
__device__ __forceinline__ size_t c8s_at(int b, int c, int t, int T) {
  return (((size_t)b * (2 * LH / 8) + c / 8) * T + t) * 8 + c % 8;
}

__device__ __forceinline__ float sigm(float v) { return 1.f / (1.f + expf(-v)); }

// 32 values per lane -> lane L holds the warp total of value L; the association is the same for every L
__device__ __forceinline__ float reduce32(float (&v)[32], int lane) {
#pragma unroll
  for (int o = 16; o >= 1; o >>= 1) {
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = up ? v[i] : v[i + o];
      const float keep = up ? v[i + o] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return v[0];
}

__global__ void __launch_bounds__(L_THREADS, 1) lstm_kernel(LstmArgs a) {
  extern __shared__ float sm[];
  float* ws = sm;                      // [L_ROWS][L_K]
  float* vs = ws + L_ROWS * L_K;       // [L_NB][x_s | h1_{s-1} | h2_{s-2}]
  float* gs = vs + L_NB * 3 * LH;      // [layer][gate][unit][item]
  const int B = a.B, T = a.T, cta = blockIdx.x, tid = threadIdx.x;
  const int lane = tid & 31, warp = tid >> 5;
  unsigned epoch = 0;
  {
    const float4* src = reinterpret_cast<const float4*>(a.w + (size_t)cta * L_ROWS * L_K);
    for (int e = tid; e < L_ROWS * L_K / 4; e += L_THREADS) reinterpret_cast<float4*>(ws)[e] = src[e];
  }
  // x [B][H][T] -> xt [T][B][H] through 32 x 32 tiles, and zero state
  {
    float(*tile)[33] = reinterpret_cast<float(*)[33]>(vs);
    const int tt = (T + 31) / 32, ntiles = B * (LH / 32) * tt;
    for (int i = cta; i < ntiles; i += gridDim.x) {
      const int b = i / ((LH / 32) * tt), r = i % ((LH / 32) * tt), c0 = (r / tt) * 32, s0 = (r % tt) * 32;
      __syncthreads();
      for (int e = tid; e < 1024; e += L_THREADS) {
        const int ci = e / 32, si = e % 32;
        if (s0 + si >= T) continue;
        if (a.c8s) {
          const __nv_bfloat16* xb = reinterpret_cast<const __nv_bfloat16*>(a.x);
          const size_t o = c8s_at(b, c0 + ci, s0 + si, T);
          tile[ci][si] = __bfloat162float(xb[o]) + __bfloat162float(xb[o + (size_t)(LH / 8) * T * 8]);
        } else {
          tile[ci][si] = reinterpret_cast<const float*>(a.x)[((size_t)b * LH + c0 + ci) * T + s0 + si];
        }
      }
      __syncthreads();
      for (int e = tid; e < 1024; e += L_THREADS) {
        const int si = e / 32, ci = e % 32;
        if (s0 + si < T) a.xt[((size_t)(s0 + si) * B + b) * LH + c0 + ci] = tile[ci][si];
      }
    }
    for (int e = tid; e < L_UNITS * B; e += L_THREADS) {
      const int b = e / L_UNITS, h = cta * L_UNITS + e % L_UNITS;
      for (int k = 0; k < 2; ++k) {
        a.h1[((size_t)k * B + b) * LH + h] = 0.f;
        a.h2[((size_t)k * B + b) * LH + h] = 0.f;
        a.c[((size_t)k * B + b) * LH + h] = 0.f;
      }
    }
  }
  __threadfence();
  grid_barrier(a.counter, epoch, a.err);

  // warps 0-3: layer 1, gate = warp; warps 4-7: layer 2, gate = warp - 4.  Rows of a warp: units 0..3.
  const int layer = warp >> 2, gate = warp & 3;
  const float* wrow = ws + (size_t)warp * L_UNITS * L_K;
  const float* vbase = vs + layer * LH;  // layer 1 reads [x | h1], layer 2 [h1 | h2]
  for (int s = 0; s <= T; ++s) {
    const bool on1 = s < T, on2 = s >= 1;
    const float* h1r = a.h1 + (size_t)((s + 1) & 1) * B * LH;  // h1_{s-1}
    const float* h2r = a.h2 + (size_t)(s & 1) * B * LH;        // h2_{s-2}
    for (int b0 = 0; b0 < B; b0 += L_NB) {
      const int nb = min(L_NB, B - b0);
      for (int e = tid; e < L_NB * 3 * LH / 4; e += L_THREADS) {
        const int bi = e / (3 * LH / 4), k = (e % (3 * LH / 4)) * 4;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (bi < nb) {
          const int b = b0 + bi;
          if (k < LH) {
            if (on1) v = __ldcg(reinterpret_cast<const float4*>(a.xt + ((size_t)s * B + b) * LH + k));
          } else if (k < 2 * LH) {
            v = __ldcg(reinterpret_cast<const float4*>(h1r + (size_t)b * LH + k - LH));
          } else {
            v = __ldcg(reinterpret_cast<const float4*>(h2r + (size_t)b * LH + k - 2 * LH));
          }
        }
        reinterpret_cast<float4*>(vs)[e] = v;
      }
      __syncthreads();
      if (layer == 0 ? on1 : on2) {
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        for (int i = 0; i < L_K / 32; ++i) {
          const int k = lane + 32 * i;
          float wv[L_UNITS];
#pragma unroll
          for (int u = 0; u < L_UNITS; ++u) wv[u] = wrow[u * L_K + k];
#pragma unroll
          for (int bi = 0; bi < L_NB; ++bi) {
            const float v = vbase[bi * 3 * LH + k];
#pragma unroll
            for (int u = 0; u < L_UNITS; ++u) acc[u * L_NB + bi] = fmaf(wv[u], v, acc[u * L_NB + bi]);
          }
        }
        const float g = reduce32(acc, lane);
        const int u = lane / L_NB, bi = lane % L_NB;
        gs[((layer * 4 + gate) * L_UNITS + u) * L_NB + bi] = g + a.bias[cta * L_ROWS + (layer * 4 + gate) * L_UNITS + u];
      }
      __syncthreads();
      if (tid < 2 * L_UNITS * L_NB) {
        const int ly = tid / (L_UNITS * L_NB), u = (tid / L_NB) % L_UNITS, bi = tid % L_NB;
        if (bi < nb && (ly == 0 ? on1 : on2)) {
          const float* g = gs + ly * 4 * L_UNITS * L_NB + u * L_NB + bi;
          const float ig = sigm(g[0]), fg = sigm(g[L_UNITS * L_NB]), gg = tanhf(g[2 * L_UNITS * L_NB]),
                      og = sigm(g[3 * L_UNITS * L_NB]);
          const int b = b0 + bi, h = cta * L_UNITS + u;
          float* cp = a.c + ((size_t)ly * B + b) * LH + h;
          const float c = fmaf(fg, *cp, ig * gg);
          *cp = c;
          const float hv = og * tanhf(c);
          if (ly == 0) {
            a.h1[((size_t)(s & 1) * B + b) * LH + h] = hv;
          } else {
            a.h2[((size_t)((s + 1) & 1) * B + b) * LH + h] = hv;
            const float out = hv + __ldcg(a.xt + ((size_t)(s - 1) * B + b) * LH + h);
            const float v = a.elu_out ? elu(out) : out;
            if (a.c8s) {
              __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(a.y);
              const size_t o = c8s_at(b, h, s - 1, T);
              const __nv_bfloat16 hi = __float2bfloat16_rn(v);
              yb[o] = hi;
              yb[o + (size_t)(LH / 8) * T * 8] = __float2bfloat16_rn(v - __bfloat162float(hi));
            } else {
              reinterpret_cast<float*>(a.y)[((size_t)b * LH + h) * T + s - 1] = v;
            }
          }
        }
      }
      __syncthreads();
    }
    __threadfence();
    grid_barrier(a.counter, epoch, a.err);
  }
}

}  // namespace encodec
}  // namespace alm

using namespace alm;

extern "C" {

int alm_encodec_pad1d(const float* x, float* y, int64_t rows, int L, int pad_left, int pad_right, alm_stream_t stream) {
  ALM_REQUIRE(x && y && rows > 0 && L > 0 && pad_left >= 0 && pad_right >= 0, ALM_ERR_ARG);
  const int64_t n = rows * (int64_t)(L + pad_left + pad_right);
  const int grid = (int)std::min<int64_t>(ceil_div<int64_t>(n, 256), 8 * num_sms());
  encodec::pad1d_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, y, rows, L, pad_left, pad_right);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

int alm_encodec_resblock_fp32(const float* x, const float* w3, const float* b3, const float* w1, const float* ws,
                              const float* b_out, float* y, int B, int C, int T, int elu_out, alm_stream_t stream) {
  ALM_REQUIRE(x && w3 && b3 && w1 && ws && b_out && y && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(C >= 2 && C % 2 == 0 && C <= 512 && B <= 65535, ALM_ERR_UNSUPPORTED);
  const size_t smem = (size_t)(2 * C * (encodec::RB_TT + 2) + C / 2 * encodec::RB_TT) * sizeof(float);
  static bool attr = false;
  if (!attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(encodec::resblock_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  dim3 grid(ceil_div(T, encodec::RB_TT), B);
  encodec::resblock_kernel<<<grid, encodec::RB_THREADS, smem, (cudaStream_t)stream>>>(x, w3, b3, w1, ws, b_out, y, C, T,
                                                                                      elu_out);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

long long alm_encodec_lstm_workspace(int B, int T) {
  if (B <= 0 || T <= 0) return -1;
  // xt, h1, h2, c, then the barrier counter and error flag
  return (long long)((int64_t)T * B * encodec::LH + 6LL * B * encodec::LH) * 4 + 16;
}

int alm_encodec_lstm(const void* x, const float* w_packed, const float* bias_packed, void* y, void* workspace,
                     int B, int T, int elu_out, int c8s, alm_stream_t stream) {
  ALM_REQUIRE(x && w_packed && bias_packed && y && workspace && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE((reinterpret_cast<uintptr_t>(w_packed) & 15u) == 0 && (reinterpret_cast<uintptr_t>(workspace) & 15u) == 0,
              ALM_ERR_ALIGN);
  ALM_REQUIRE(num_sms() >= encodec::L_GRID, ALM_ERR_UNSUPPORTED);
  static bool attr = false;
  if (!attr) {
    ALM_CUDA_OK(cudaFuncSetAttribute(encodec::lstm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)encodec::L_SMEM));
    attr = true;
  }
  float* f = reinterpret_cast<float*>(workspace);
  encodec::LstmArgs a;
  a.x = x; a.w = w_packed; a.bias = bias_packed; a.y = y;
  a.xt = f;
  a.h1 = a.xt + (size_t)T * B * encodec::LH;
  a.h2 = a.h1 + 2 * (size_t)B * encodec::LH;
  a.c = a.h2 + 2 * (size_t)B * encodec::LH;
  a.counter = reinterpret_cast<unsigned*>(a.c + 2 * (size_t)B * encodec::LH);
  a.err = reinterpret_cast<int*>(a.counter + 1);
  a.B = B; a.T = T; a.elu_out = elu_out; a.c8s = c8s;
  // the counter restarts at 0 every launch; co-residency of the CTAs (one per SM) is what the barrier relies on
  ALM_CUDA_OK(cudaMemsetAsync(a.counter, 0, 8, (cudaStream_t)stream));
  void* kargs[] = {(void*)&a};
  ALM_CUDA_OK(cudaLaunchCooperativeKernel((const void*)encodec::lstm_kernel, dim3(encodec::L_GRID),
                                          dim3(encodec::L_THREADS), kargs, encodec::L_SMEM, (cudaStream_t)stream));
  ALM_LAUNCHED(1);
  return ALM_OK;
}

}  // extern "C"
