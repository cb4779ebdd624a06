// SoundStream encoder / decoder convs on the Hopper tensor cores (sm_90a wgmma): split-bf16 ("bf16x3") implicit-GEMM
// causal convs.
//
// Reference arithmetic: soundstream.py:332-345 (CausalConv1d), :362-369 (ResidualUnit), :371-383 (EncoderBlock).
//
// Why tensor cores: fp32 CUDA-core conv kernels (conv_tiled.cuh) are FMA-bound.  fp32 operands are split as
// x = x_hi + x_lo (two bf16, |x - x_hi - x_lo| <= 2^-17 |x|) and every product is evaluated as
//   x_hi w_hi + x_lo w_hi + x_hi w_lo          (three bf16 wgmmas, fp32 accumulation in registers)
// which keeps the result within ~2^-16 relative of the fp32 product (the dropped x_lo w_lo term is 2^-18).
//
// Activation format between the encoder's layers ("C8S", channels-8 split): bf16 [B][2C/8][P][T/P][8]
//   chunk c < C/8 holds the hi halves of channels 8c..8c+7, chunk C/8 + c their lo halves;
//   P = 1 normally; a layer feeding a stride-s conv writes P = s phase planes (row t -> plane t % s, row t / s) so
//   that every tap of the strided conv reads unit-stride rows.
// Same bytes as fp32 [B][C][T].  One time step of one chunk is 16 B = one row of a wgmma no-swizzle core matrix:
// a tile [chunk][row][8] is a K-major operand whose rows are 16 B apart (SBO = 128), so the start address of the
// A descriptor can point at ANY row.  One staged tile [rows + 6d] therefore serves all 7 taps of a dilated conv
// by shifting the descriptor start by j*d rows: no im2col, no per-tap reload.
//
// Kernels
//   first_conv_kernel      fp32 wave [B][T] (C_in = 1) -> C8S, CUDA cores (7 FMAs per output, HBM-bound on the write)
//   ru_tc_kernel<C, SE>    fused ResidualUnit: y = x + ELU(W1 ELU(W7 *_d x + b7) + b1); the k=7 result goes
//                          registers -> (bias, ELU, split) -> shared memory as the bf16 A operand of the 1x1 conv.
//                          SE = true adds the unit's SqueezeExcite (soundstream.py:145-169) as two more GEMMs per tile
//                          RB = true: EnCodec's SEANet resnet block instead (EncodecWrapper; see RuCfg)
//   conv_tc_kernel<..>     strided / plain causal conv as a pipelined implicit GEMM over (tap, k-step) units
// Activation tiles are staged with 16-B cp.async by whole producer warps, weights with large bulk copies.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {
namespace ctc {

constexpr int TILE_M = 128;
constexpr int MAX_HALO = 54;  // 6 * dilation 9

__device__ __forceinline__ float elu1(float v) { return v > 0.f ? v : (__expf(v) - 1.f); }
__device__ __forceinline__ float silu1(float v) { return v / (1.f + __expf(-v)); }
__device__ __forceinline__ float sigmoid1(float v) { return 1.f / (1.f + __expf(-v)); }

// 8 fp32 -> hi uint4, lo uint4 (bf16 pairs, channel e in the low half of word e/2 for even e)
__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    __nv_bfloat16 h0, l0, h1, l1;
    split_bf16(v[2 * i], h0, l0);
    split_bf16(v[2 * i + 1], h1, l1);
    h[i] = (uint32_t)__bfloat16_as_ushort(h0) | ((uint32_t)__bfloat16_as_ushort(h1) << 16);
    l[i] = (uint32_t)__bfloat16_as_ushort(l0) | ((uint32_t)__bfloat16_as_ushort(l1) << 16);
  }
  hi = make_uint4(h[0], h[1], h[2], h[3]);
  lo = make_uint4(l[0], l[1], l[2], l[3]);
}

// element offset of (batch b, chunk c, time t) in a C8S tensor with `nch` chunks, P phase planes, T time steps
__device__ __forceinline__ size_t c8s_off(int b, int c, int t, int nch, int P, int T) {
  return ((((size_t)b * nch + c) * P + (t % P)) * (size_t)(T / P) + (t / P)) * 8;
}

// ---------------------------------------------------------------------------------------------
// first conv: C_in = 1, kernel K <= 8, stride 1 -> C8S (P = 1)
// ---------------------------------------------------------------------------------------------
template <int COUT>
__global__ void __launch_bounds__(128) first_conv_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ bias, __nv_bfloat16* __restrict__ y,
                                                         int B, int T, int K, int pad_mode) {
  __shared__ float sw[COUT * 8];
  __shared__ float sb[COUT];
  for (int i = threadIdx.x; i < COUT * 8; i += blockDim.x) sw[i] = (i % 8) < K ? w[(i / 8) * K + (i % 8)] : 0.f;
  for (int i = threadIdx.x; i < COUT; i += blockDim.x) sb[i] = bias ? bias[i] : 0.f;
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int pad = K - 1;
  constexpr int NCH = COUT / 8;
  // grid.y is capped at 65535: a larger batch strides over it
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    float xv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      xv[j] = 0.f;
      if (j < K) {
        int u = t + j - pad;  // x index of tap j
        if (u < 0) {
          if (pad_mode == 0) u = -u;                 // reflect (edge sample excluded)
          else if (pad_mode == 2) u = 0;             // replicate
          else u = -1;                               // constant zero
        }
        if (u >= 0) xv[j] = __ldg(x + (size_t)b * T + u);
      }
    }
#pragma unroll 1
    for (int c = 0; c < NCH; ++c) {
      float v[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float acc = sb[c * 8 + e];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc = fmaf(sw[(c * 8 + e) * 8 + j], xv[j], acc);  // taps >= K: w = 0 and x = 0
        v[e] = acc;
      }
      uint4 hi, lo;
      split8(v, hi, lo);
      *reinterpret_cast<uint4*>(y + c8s_off(b, c, t, 2 * NCH, 1, T)) = hi;
      *reinterpret_cast<uint4*>(y + c8s_off(b, NCH + c, t, 2 * NCH, 1, T)) = lo;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// fp32 channels-last [B][n][C] (the quantizer's output) -> C8S (P = 1): the decoder's entry format
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pack_c8s_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, int B,
                                                       int n, int C) {
  const int nch = C / 8;
  const long long total = (long long)B * n * nch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % nch);
    const long long bt = i / nch;
    const int t = (int)(bt % n), b = (int)(bt / n);
    const float4 a0 = __ldg(reinterpret_cast<const float4*>(x + bt * C + c * 8));
    const float4 a1 = __ldg(reinterpret_cast<const float4*>(x + bt * C + c * 8 + 4));
    const float v[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    uint4 hi, lo;
    split8(v, hi, lo);
    *reinterpret_cast<uint4*>(y + c8s_off(b, c, t, 2 * nch, 1, n)) = hi;
    *reinterpret_cast<uint4*>(y + c8s_off(b, nch + c, t, 2 * nch, 1, n)) = lo;
  }
}

// ---------------------------------------------------------------------------------------------
// last decoder conv: CausalConv1d(CIN, 1, K <= 8) on C8S -> fp32 wave [B][T] (soundstream.py:626), CUDA cores
// ---------------------------------------------------------------------------------------------
template <int CIN>
__global__ void __launch_bounds__(128) last_conv_kernel(const __nv_bfloat16* __restrict__ x, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ y, int B,
                                                        int T, int K, int pad_mode) {
  __shared__ float sw[CIN * 8];  // [ci][tap]
  for (int i = threadIdx.x; i < CIN * 8; i += blockDim.x) sw[i] = (i % 8) < K ? w[(i / 8) * K + (i % 8)] : 0.f;
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  constexpr int NCH = CIN / 8;
  const int pad = K - 1;
  // grid.y is capped at 65535: a larger batch strides over it
  for (int b = blockIdx.y; b < B; b += gridDim.y) {
    float acc = bias ? bias[0] : 0.f;
    for (int j = 0; j < K; ++j) {
      int u = t + j - pad;
      if (u < 0) {
        if (pad_mode == 0) u = -u;
        else if (pad_mode == 2) u = 0;
        else continue;
      }
#pragma unroll
      for (int c = 0; c < NCH; ++c) {
        const uint4 h = __ldg(reinterpret_cast<const uint4*>(x + c8s_off(b, c, u, 2 * NCH, 1, T)));
        const uint4 l = __ldg(reinterpret_cast<const uint4*>(x + c8s_off(b, NCH + c, u, 2 * NCH, 1, T)));
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          acc = fmaf(sw[(c * 8 + 2 * e) * 8 + j], bf16_lo(hw[e]) + bf16_lo(lw[e]), acc);
          acc = fmaf(sw[(c * 8 + 2 * e + 1) * 8 + j], bf16_hi(hw[e]) + bf16_hi(lw[e]), acc);
        }
      }
    }
    y[(size_t)b * T + t] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// shared pieces
// ---------------------------------------------------------------------------------------------
// row `t` of a C8S tensor with P phase planes: element offset of chunk 0 (add c * chunk_stride for chunk c)
struct RowAddr {
  size_t off;           // ((b * nch) * P + t % P) * (T / P) + t / P, in 8-element rows, times 8
  size_t chunk_stride;  // elements between consecutive chunks
};
__device__ __forceinline__ RowAddr c8s_row(int b, int t, int nch, int P, int T) {
  const int rows = T / P;
  RowAddr a;
  a.chunk_stride = (size_t)P * rows * 8;
  a.off = (size_t)b * nch * a.chunk_stride + ((size_t)(t % P) * rows + (t / P)) * 8;
  return a;
}

// ---------------------------------------------------------------------------------------------
// fused ResidualUnit
//   warps 0 (and 3 when the weights are resident) : producers      warps 4-7 : one consumer warpgroup (wgmma + epilogues)
// One tile = RU_TILE_M time steps.  D1 (the k=7 dilated conv) accumulates in registers; E1 adds b7, applies ELU and
// writes the split bf16 activation to shared memory in the no-swizzle K-major layout, which is the A operand of the
// 1x1 conv (D2); E2 adds b1, applies ELU, adds the skip input and stores C8S.  One warpgroup per CTA keeps the
// register budget at 255 per thread, which the C = 256 layer (two 128-register accumulators in sequence) needs.
//
// SE = true (ResidualUnit(squeeze_excite=True), soundstream.py:362-369): the unit's output is x + y * gate(y) with
// y = ELU(D2 + b1).  The reference's "cumulative mean" runs over channels (SqueezeExcite.forward cumsums dim -2 of
// [B, C, T]), so the gate is pointwise in time and the mean folds into the first SE weight (ops.pack_ru_se_weights):
//   gate = sigmoid(W2 SiLU(W1' y + bs1) + bs2),  W1'[i, c'] = sum_{c >= c'} W1[i, c] / (c + 1).
// E2 writes split y to sA2 (as E1 does); D3 = y W1'^T (N = NS, the inner width zero-padded to >= 32, A from sA2);
// E3 adds bs1, applies SiLU and splits the accumulators straight into register A fragments (the m64nNk16 accumulator
// and the k16 register-A layouts coincide); D4 = s W2^T (N = C, K = NS, A from registers); E4 re-reads y from sA2,
// adds the skip input and stores.  Re-reading y keeps the C = 256 layer at one 128-register accumulator.  The SE
// weights stream through the same ring (or stay resident) after the conv units: KSTEPS W1' units, NS / 16 W2 units.
// ---------------------------------------------------------------------------------------------
constexpr int RU_TILE_M = 64;
constexpr int RU_THREADS = 256;

struct RuParams {
  const __nv_bfloat16* x;
  __nv_bfloat16* y;
  const __nv_bfloat16* w;  // units (tap j = 0..6 of the k=7 conv, 7 = the 1x1 conv) x (k-step): [part][2][C][8]
  const float* b7;
  const float* b1;
  int B, T, d, pad_mode, out_phases;
  int tiles_per_clip, total_tiles;
  int ar;      // rows of one staged chunk: RU_TILE_M + 6 d
  int na, nw;  // staged activation tiles (1 or 2), weight ring stages (streamed mode)
  const float* se_b1 = nullptr;  // SE only: biases of the two 1x1 convs ([se_ci], [C])
  const float* se_b2 = nullptr;
  int se_ci = 0;
  int elu_out = 0;  // RB only: ELU on the block's output
};

// RB = true: EnCodec's SEANet resnet block (EncodecWrapper) on the same pipeline,
//   y = [W1 | Ws] . [ELU(W3 *_k3 ELU(x) + b3) ; x] + b1 + bs   (ELU'd when elu_out), C -> C/2 -> C.
// The staged tile is raw x; the consumers write ELU(x) (re-split) into the sA2 region, which D1 reads; E1 then
// overwrites sA2 with the hidden activations.  D1 runs with N = C (W3's rows zero-padded from C/2), so the units, the
// accumulator and E1 are the ResidualUnit's; D2 runs K over the hidden k-steps (A = sA2) and then the shortcut's
// k-steps (A = the staged raw x, shifted by the 2-row halo), so the 1x1 shortcut folds into the second product.
// Units: 3 W3 taps, W1 (columns zero-padded from C/2), Ws: 5 KSTEPS.  The staged tile is released after D2.
template <int C, bool SE = false, bool RB = false>
struct RuCfg {
  static constexpr int NCHUNK = C / 8;
  static constexpr int KSTEPS = C / 16;
  static constexpr bool RESIDENT = C <= 64;       // all weights stay in shared memory for the CTA's lifetime
  static constexpr int UNIT_BYTES = 2 * 2 * C * 16;  // hi [2 chunks][C][16 B] + lo
  static constexpr int NUNITS = (RB ? 5 : 8) * KSTEPS;
  static constexpr int MAX_NW = 16;
  // E1 output: [hi / lo][chunk][64 rows][16 B]; RB: first ELU(x) with the 2-row halo
  static constexpr int A2_BYTES = 2 * NCHUNK * (RU_TILE_M + (RB ? 2 : 0)) * 16;
  // squeeze-excite: inner width padded to NS (a multiple of 16, >= 32 for the smallest wgmma tile in use)
  static constexpr int NS = SE ? (C / 4 > 32 ? C / 4 : 32) : 0;
  static constexpr int SE1_UNIT_BYTES = 2 * 2 * NS * 16;  // one k-step of W1': hi / lo [2 chunks][NS][16 B]
  static constexpr int SE_BYTES = KSTEPS * SE1_UNIT_BYTES + (NS / 16) * UNIT_BYTES;
  static constexpr int W_BYTES = NUNITS * UNIT_BYTES + SE_BYTES;  // the packed weights of one unit (resident image)
  static constexpr int BIAS_FLOATS = 2 * C + (SE ? NS + C : 0);  // b7, b1 (, bs1 padded to NS, bs2)
  static constexpr int FIXED_BYTES = A2_BYTES + BIAS_FLOATS * 4 + 512 + 128;  // A2, biases, barriers, alignment slack
  static constexpr int MAX_SMEM = 232448;
  // two CTAs per SM only where shared memory allows it at every dilation (resident weights, largest halo); the
  // occupancy hint of the kernel and the grid size of launch_ru both follow from it
  static constexpr int RESIDENT_MAX_SMEM =
      2 * (2 * NCHUNK * (RU_TILE_M + MAX_HALO) * 16) + W_BYTES + FIXED_BYTES;
  static constexpr int CTAS_PER_SM = RESIDENT && RESIDENT_MAX_SMEM <= 113 * 1024 ? 2 : 1;
  // weight unit u of the packed image: 8 KSTEPS conv units, then KSTEPS W1' units, then NS / 16 W2 units
  static constexpr int ALL_UNITS = NUNITS + (SE ? KSTEPS + NS / 16 : 0);
  __host__ __device__ static constexpr int unit_off(int u) {
    return u < NUNITS            ? u * UNIT_BYTES
           : u < NUNITS + KSTEPS ? NUNITS * UNIT_BYTES + (u - NUNITS) * SE1_UNIT_BYTES
                                 : NUNITS * UNIT_BYTES + KSTEPS * SE1_UNIT_BYTES + (u - NUNITS - KSTEPS) * UNIT_BYTES;
  }
  __host__ __device__ static constexpr int unit_bytes(int u) {
    return u >= NUNITS && u < NUNITS + KSTEPS ? SE1_UNIT_BYTES : UNIT_BYTES;
  }
};

template <int C, bool SE, bool RB>
__global__ void __launch_bounds__(RU_THREADS, RuCfg<C, SE, RB>::CTAS_PER_SM) ru_tc_kernel(const RuParams p) {
  using Cfg = RuCfg<C, SE, RB>;
  constexpr int TAPS = RB ? 3 : 7;
  constexpr int NCHUNK = Cfg::NCHUNK, KSTEPS = Cfg::KSTEPS;
  constexpr bool RESIDENT = Cfg::RESIDENT;
  const int NA = p.na, NW = p.nw, A_ROWS = p.ar;
  const int A_BYTES = 2 * NCHUNK * A_ROWS * 16;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  uint8_t* sA2 = smem;
  uint8_t* sA = sA2 + Cfg::A2_BYTES;
  uint8_t* sW = sA + NA * A_BYTES;
  float* sBias = reinterpret_cast<float*>(sW + (RESIDENT ? Cfg::W_BYTES : NW * Cfg::UNIT_BYTES));
  uint64_t* bars = reinterpret_cast<uint64_t*>(sBias + Cfg::BIAS_FLOATS);
  uint64_t* a_full = bars;              // [2]
  uint64_t* a_empty = bars + 2;         // [2]
  uint64_t* w_full = bars + 4;          // [<= 16] (resident: [0] only)
  uint64_t* w_empty = bars + 20;        // [<= 16]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < 2; ++i) {
      mbar_init(&a_full[i], 1);
      mbar_init(&a_empty[i], 4);  // one arrive per consumer warp
    }
    for (int i = 0; i < Cfg::MAX_NW; ++i) {
      mbar_init(&w_full[i], 1);
      mbar_init(&w_empty[i], 4);
    }
    fence_mbar_init();
  }
  for (int i = threadIdx.x; i < C; i += blockDim.x) {
    sBias[i] = p.b7 ? p.b7[i] : 0.f;
    sBias[C + i] = p.b1 ? p.b1[i] : 0.f;
  }
  if constexpr (SE) {
    for (int i = threadIdx.x; i < Cfg::NS; i += blockDim.x) sBias[2 * C + i] = i < p.se_ci ? p.se_b1[i] : 0.f;
    for (int i = threadIdx.x; i < C; i += blockDim.x) sBias[2 * C + Cfg::NS + i] = p.se_b2[i];
  }
  __syncthreads();

  const int halo = (TAPS - 1) * p.d;
  auto tile_of = [&](int i) { return (int)blockIdx.x + i * (int)gridDim.x; };
  auto has = [&](int i) { return i >= 0 && tile_of(i) < p.total_tiles; };

  if (warp < 4) {
    if (!(warp == 0 || (RESIDENT && warp == 3))) return;
    // ===================== producer(s) =====================
    // activation tiles: 16-B cp.async by all 32 lanes (the padding rule is just an address per row); weights: bulk copies.
    // Resident-weight layers (C <= 64) run TWO producer warps, warp 0 owning staging buffer 0 (even tiles) and warp 3
    // buffer 1 (odd tiles).
    if (RESIDENT && warp == 0 && lane == 0) {
      mbar_arrive_expect_tx(&w_full[0], Cfg::W_BYTES);
      constexpr int PIECE = 16384;  // few large copies
      for (int off = 0; off < Cfg::W_BYTES; off += PIECE)
        bulk_copy_g2s(sW + off, reinterpret_cast<const uint8_t*>(p.w) + off, min(PIECE, Cfg::W_BYTES - off),
                      &w_full[0]);
    }
    int wstage = 0;
    uint32_t wphase = 0;
    auto stream_units = [&](int u0, int u1) {  // lane 0 only
      for (int u = u0; u < u1; ++u) {
        mbar_wait(&w_empty[wstage], wphase ^ 1u);
        mbar_arrive_expect_tx(&w_full[wstage], Cfg::UNIT_BYTES);
        bulk_copy_g2s(sW + wstage * Cfg::UNIT_BYTES, p.w + (size_t)u * (Cfg::UNIT_BYTES / 2), Cfg::UNIT_BYTES,
                      &w_full[wstage]);
        if (++wstage == NW) { wstage = 0; wphase ^= 1u; }
      }
    };
    auto stream_se_units = [&](int u0, int u1) {  // lane 0 only; the W1' units are smaller than a ring slot
      for (int u = u0; u < u1; ++u) {
        mbar_wait(&w_empty[wstage], wphase ^ 1u);
        mbar_arrive_expect_tx(&w_full[wstage], Cfg::unit_bytes(u));
        bulk_copy_g2s(sW + wstage * Cfg::UNIT_BYTES, reinterpret_cast<const uint8_t*>(p.w) + Cfg::unit_off(u),
                      Cfg::unit_bytes(u), &w_full[wstage]);
        if (++wstage == NW) { wstage = 0; wphase ^= 1u; }
      }
    };
    auto issue_a = [&](int i) {
      const int ab = i % NA;
      mbar_wait(&a_empty[ab], (((uint32_t)(i / NA)) & 1u) ^ 1u);
      const int tile = tile_of(i);
      const int b = tile / p.tiles_per_clip;
      const int t0 = (tile - b * p.tiles_per_clip) * RU_TILE_M;
      const int rows = halo + min(RU_TILE_M, p.T - t0);  // smem row r <-> time t0 - halo + r
      uint8_t* dst = sA + ab * A_BYTES;
      for (int r = lane; r < rows; r += 32) {
        int tau = t0 - halo + r;
        uint32_t bytes = 16;
        if (tau < 0) {  // left padding (soundstream.py:339-344)
          if (p.pad_mode == 0) tau = -tau;            // reflect, edge sample excluded
          else if (p.pad_mode == 2) tau = 0;          // replicate
          else { tau = 0; bytes = 0; }                // constant zero
        }
        const __nv_bfloat16* src = p.x + ((size_t)b * 2 * NCHUNK * p.T + tau) * 8;
#pragma unroll 4
        for (int c = 0; c < 2 * NCHUNK; ++c)
          cp_async_16(dst + (c * A_ROWS + r) * 16, src + (size_t)c * p.T * 8, bytes);
      }
      cp_async_commit();
    };
    // HBM latency under load exceeds one tile period: pull the tiles PF steps ahead into L2 so that the cp.async of
    // the staged tile (and the epilogue's skip reads) hit L2
    constexpr int PF = 3;
    auto prefetch_tile = [&](int i) {
      const int tile = tile_of(i);
      const int b = tile / p.tiles_per_clip;
      const int t0 = (tile - b * p.tiles_per_clip) * RU_TILE_M;
      const int first = max(0, t0 - halo), last = min(p.T, t0 + RU_TILE_M);
      const int lpc = ((last - first) * 16 + 127) / 128 + 1;  // 128-B lines per chunk (+1: unaligned start)
      const uint8_t* base = reinterpret_cast<const uint8_t*>(p.x + ((size_t)b * 2 * NCHUNK * p.T + first) * 8);
      const size_t span = (size_t)(last - first) * 16 - 1;
      for (int idx = lane; idx < 2 * NCHUNK * lpc; idx += 32) {
        const int c = idx / lpc, l = idx - c * lpc;
        prefetch_l2(base + (size_t)c * p.T * 16 + min((size_t)l * 128, span));
      }
    };
    if (RESIDENT) {
      const int pid = warp == 0 ? 0 : 1;  // NA == 2: tile i lives in buffer i % 2, owned by producer i % 2
      if (has(pid + 2)) prefetch_tile(pid + 2);
      for (int i = pid; has(i); i += 2) {
        if (has(i + 4)) prefetch_tile(i + 4);
        issue_a(i);                  // waits until the consumer has released the buffer
        cp_async_wait<0>();
        fence_proxy_async_smem();    // cp.async writes (generic proxy) -> wgmma operand reads (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_full[i % NA]);
      }
    } else {
      if (has(0)) issue_a(0);
      for (int k = 1; k < PF; ++k)
        if (has(k)) prefetch_tile(k);
      for (int i = 0; has(i); ++i) {
        if (has(i + PF)) prefetch_tile(i + PF);
        cp_async_wait<0>();        // tile i (issued one step ago)
        fence_proxy_async_smem();  // cp.async writes (generic proxy) -> wgmma operand reads (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_full[i % NA]);
        // publish tile i BEFORE staging tile i + 1: the staging waits for a_empty and takes ~1 k clk of issue
        if (NA == 2 && has(i + 1)) issue_a(i + 1);
        if constexpr (SE) {
          if (lane == 0) stream_se_units(0, Cfg::ALL_UNITS);
        } else {
          if (lane == 0) stream_units(0, Cfg::NUNITS);
        }
        __syncwarp();
        if (NA == 1 && has(i + 1)) issue_a(i + 1);
      }
    }
    return;
  }

  // ===================== consumer warpgroup =====================
  // fragment: rows rl + 8 h (h = 0, 1) of the tile, of every 8-column group j the columns 8 j + c_lane + {0, 1}
  const int rl = (warp & 3) * 16 + (lane >> 2);
  const int c_lane = 2 * (lane & 3);
  if (RESIDENT) mbar_wait(&w_full[0], 0);
  int wstage = 0;
  uint32_t wphase = 0;
  int prev_w = -1;
  const uint32_t sw_addr = smem_u32(sW);
  const uint64_t b0 = wgmma_desc_nosw(sw_addr, 128, C * 16);
  const uint32_t a2_addr = smem_u32(sA2);
  // weights of unit u: resident at a fixed offset, else the next slot of the ring (released one unit later, when the
  // wgmma group that read it has retired)
  auto unit_b = [&](int u) -> uint64_t {
    if (RESIDENT) return b0 + (uint64_t)(u * (Cfg::UNIT_BYTES / 16));
    mbar_wait(&w_full[wstage], wphase);
    return b0 + (uint64_t)(wstage * (Cfg::UNIT_BYTES / 16));
  };
  // SE units: resident at their packed offset, else the next ring slot; `base` carries the operand's LBO
  auto se_unit = [&](int u, uint64_t base) -> uint64_t {
    if (RESIDENT) return base + (uint64_t)(Cfg::unit_off(u) / 16);
    mbar_wait(&w_full[wstage], wphase);
    return base + (uint64_t)(wstage * (Cfg::UNIT_BYTES / 16));
  };
  auto unit_done = [&]() {
    wgmma_commit();
    if (!RESIDENT) {
      wgmma_wait<1>();
      if (prev_w >= 0 && lane == 0) mbar_arrive(&w_empty[prev_w]);
      prev_w = wstage;
      if (++wstage == NW) { wstage = 0; wphase ^= 1u; }
    }
  };
  auto drain = [&]() {
    wgmma_wait<0>();
    if (!RESIDENT && prev_w >= 0 && lane == 0) mbar_arrive(&w_empty[prev_w]);
    prev_w = -1;
  };
  for (int i = 0; has(i); ++i) {
    const int ab = i % NA;
    mbar_wait(&a_full[ab], ((uint32_t)(i / NA)) & 1u);
    if constexpr (RB) {
      // ---- ELU(x) of the staged tile (halo included) -> sA2, same [hi / lo][chunk][A_ROWS][16 B] layout ----
      const uint8_t* src = sA + ab * A_BYTES;
      for (int e = threadIdx.x - 128; e < NCHUNK * A_ROWS; e += 128) {
        const uint4 h = *reinterpret_cast<const uint4*>(src + e * 16);
        const uint4 l = *reinterpret_cast<const uint4*>(src + (NCHUNK * A_ROWS + e) * 16);
        const uint32_t hw[4] = {h.x, h.y, h.z, h.w}, lw[4] = {l.x, l.y, l.z, l.w};
        float v[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          v[2 * k] = elu1(bf16_lo(hw[k]) + bf16_lo(lw[k]));
          v[2 * k + 1] = elu1(bf16_hi(hw[k]) + bf16_hi(lw[k]));
        }
        uint4 oh, ol;
        split8(v, oh, ol);
        *reinterpret_cast<uint4*>(sA2 + e * 16) = oh;
        *reinterpret_cast<uint4*>(sA2 + (NCHUNK * A_ROWS + e) * 16) = ol;
      }
      fence_proxy_async_smem();  // generic-proxy writes -> wgmma operand reads
      asm volatile("bar.sync 1, 128;" ::: "memory");
    }
    // ---- D1 = W7 *_d x: 7 taps x KSTEPS units, three bf16 products each (x_hi w_hi + x_lo w_hi + x_hi w_lo) ----
    float d[C / 2];
    {
      const uint32_t a_addr = RB ? a2_addr : smem_u32(sA + ab * A_BYTES);
      // descriptors are built once; between MMAs only the 14-bit start-address field (>> 4) of the low word moves
      const uint64_t a_hi0 = wgmma_desc_nosw(a_addr, 128, A_ROWS * 16);
      const uint64_t a_lo0 = wgmma_desc_nosw(a_addr + NCHUNK * (A_ROWS * 16), 128, A_ROWS * 16);
      const uint32_t kstep_units = 2 * A_ROWS;       // two chunks, in 16-B units
#pragma unroll 1
      for (int j = 0; j < TAPS; ++j) {
        const uint32_t row_units = (uint32_t)(j * p.d);
#pragma unroll
        for (int kk = 0; kk < KSTEPS; ++kk) {
          const uint64_t b_hi = unit_b(j * KSTEPS + kk);
          const uint64_t b_lo = b_hi + (uint64_t)(2 * C);
          const uint64_t off = (uint64_t)(kk * kstep_units + row_units);
          wgmma_fence();
          wgmma_ss<C>(d, a_hi0 + off, b_hi, (j > 0 || kk > 0) ? 1u : 0u);
          wgmma_ss<C>(d, a_lo0 + off, b_hi, 1u);
          wgmma_ss<C>(d, a_hi0 + off, b_lo, 1u);
          unit_done();
        }
      }
      drain();
      wgmma_fence_acc(d);
    }
    if (!RB && lane == 0) mbar_arrive(&a_empty[ab]);  // the staged tile may be overwritten
    if constexpr (RB) asm volatile("bar.sync 1, 128;" ::: "memory");  // every warp's D1 reads of ELU(x) have retired
    // ---- E1: D1 (+b7, ELU, split) -> sA2, [hi / lo][chunk][64 rows][16 B] ----
#pragma unroll
    for (int j = 0; j < C / 8; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int col = 8 * j + c_lane;
        uint32_t hi, lo;
        split_bf16x2(elu1(d[4 * j + 2 * h] + sBias[col]), elu1(d[4 * j + 2 * h + 1] + sBias[col + 1]), hi, lo);
        const uint32_t off = (uint32_t)(j * RU_TILE_M + rl + 8 * h) * 16 + c_lane * 2;
        *reinterpret_cast<uint32_t*>(sA2 + off) = hi;
        *reinterpret_cast<uint32_t*>(sA2 + NCHUNK * RU_TILE_M * 16 + off) = lo;
      }
    fence_proxy_async_smem();  // generic-proxy writes -> wgmma operand reads
    asm volatile("bar.sync 1, 128;" ::: "memory");
    // ---- D2 = W1 ELU(D1 + b7): A from sA2 ----
#pragma unroll
    for (int kk = 0; kk < KSTEPS; ++kk) {
      const uint64_t b_hi = unit_b((TAPS) * KSTEPS + kk);
      const uint64_t b_lo = b_hi + (uint64_t)(2 * C);
      const uint32_t a_off = a2_addr + kk * 2 * (RU_TILE_M * 16);
      const uint64_t a_hi = wgmma_desc_nosw(a_off, 128, RU_TILE_M * 16);
      const uint64_t a_lo = wgmma_desc_nosw(a_off + NCHUNK * (RU_TILE_M * 16), 128, RU_TILE_M * 16);
      wgmma_fence();
      wgmma_ss<C>(d, a_hi, b_hi, kk > 0 ? 1u : 0u);
      wgmma_ss<C>(d, a_lo, b_hi, 1u);
      wgmma_ss<C>(d, a_hi, b_lo, 1u);
      unit_done();
    }
    if constexpr (RB) {
      // ---- shortcut: D2 += Ws x, A = the staged raw x from row `halo` on ----
      const uint32_t a_addr = smem_u32(sA + ab * A_BYTES);
      const uint64_t a_hi0 = wgmma_desc_nosw(a_addr, 128, A_ROWS * 16);
      const uint64_t a_lo0 = wgmma_desc_nosw(a_addr + NCHUNK * (A_ROWS * 16), 128, A_ROWS * 16);
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        const uint64_t b_hi = unit_b(4 * KSTEPS + kk);
        const uint64_t b_lo = b_hi + (uint64_t)(2 * C);
        const uint64_t off = (uint64_t)(kk * 2 * A_ROWS + halo);
        wgmma_fence();
        wgmma_ss<C>(d, a_hi0 + off, b_hi, 1u);
        wgmma_ss<C>(d, a_lo0 + off, b_hi, 1u);
        wgmma_ss<C>(d, a_hi0 + off, b_lo, 1u);
        unit_done();
      }
    }
    drain();
    wgmma_fence_acc(d);
    if (RB && lane == 0) mbar_arrive(&a_empty[ab]);  // the staged tile may be overwritten
    const int tile = tile_of(i);
    const int b = tile / p.tiles_per_clip;
    const int t0 = (tile - b * p.tiles_per_clip) * RU_TILE_M;
    if constexpr (SE) {
      constexpr int NS = Cfg::NS;
      // ---- E2: y = ELU(D2 + b1) -> split -> sA2 (A operand of D3, re-read by E4) ----
      asm volatile("bar.sync 1, 128;" ::: "memory");  // every warp's D2 reads of sA2 have retired
#pragma unroll
      for (int j = 0; j < C / 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int col = 8 * j + c_lane;
          uint32_t hi, lo;
          split_bf16x2(elu1(d[4 * j + 2 * h] + sBias[C + col]), elu1(d[4 * j + 2 * h + 1] + sBias[C + col + 1]), hi,
                       lo);
          const uint32_t off = (uint32_t)(j * RU_TILE_M + rl + 8 * h) * 16 + c_lane * 2;
          *reinterpret_cast<uint32_t*>(sA2 + off) = hi;
          *reinterpret_cast<uint32_t*>(sA2 + NCHUNK * RU_TILE_M * 16 + off) = lo;
        }
      fence_proxy_async_smem();
      asm volatile("bar.sync 1, 128;" ::: "memory");
      // ---- D3 = W1' y: N = NS, K = C, A from sA2 ----
      float s[NS / 2];
      const uint64_t b3 = wgmma_desc_nosw(sw_addr, 128, NS * 16);
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        const uint64_t b_hi = se_unit(8 * KSTEPS + kk, b3);
        const uint64_t b_lo = b_hi + (uint64_t)(2 * NS);
        const uint32_t a_off = a2_addr + kk * 2 * (RU_TILE_M * 16);
        const uint64_t a_hi = wgmma_desc_nosw(a_off, 128, RU_TILE_M * 16);
        const uint64_t a_lo = wgmma_desc_nosw(a_off + NCHUNK * (RU_TILE_M * 16), 128, RU_TILE_M * 16);
        wgmma_fence();
        wgmma_ss<NS>(s, a_hi, b_hi, kk > 0 ? 1u : 0u);
        wgmma_ss<NS>(s, a_lo, b_hi, 1u);
        wgmma_ss<NS>(s, a_hi, b_lo, 1u);
        unit_done();
      }
      drain();
      wgmma_fence_acc(s);
      // ---- E3: SiLU(D3 + bs1) -> split register A fragments of D4: a[q] of k-step kk is accumulator group
      // j = 2 kk + q / 2, row half q % 2 (padded inner channels are SiLU(0) = 0) ----
      uint32_t s_hi[NS / 16][4], s_lo[NS / 16][4];
#pragma unroll
      for (int kk = 0; kk < NS / 16; ++kk)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int j = 2 * kk + q / 2, h = q % 2;
          const int col = 8 * j + c_lane;
          split_bf16x2(silu1(s[4 * j + 2 * h] + sBias[2 * C + col]), silu1(s[4 * j + 2 * h + 1] + sBias[2 * C + col + 1]),
                       s_hi[kk][q], s_lo[kk][q]);
        }
      // ---- D4 = W2 s: N = C, K = NS ----
#pragma unroll
      for (int kk = 0; kk < NS / 16; ++kk) {
        const uint64_t b_hi = se_unit(9 * KSTEPS + kk, b0);
        const uint64_t b_lo = b_hi + (uint64_t)(2 * C);
        wgmma_fence();
        wgmma_rs<C>(d, s_hi[kk], b_hi, kk > 0 ? 1u : 0u);
        wgmma_rs<C>(d, s_lo[kk], b_hi, 1u);
        wgmma_rs<C>(d, s_hi[kk], b_lo, 1u);
        unit_done();
      }
      drain();
      wgmma_fence_acc(d);
      // ---- E4: skip + y * sigmoid(D4 + bs2) -> split -> global (C8S); each thread re-reads the y it wrote ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = t0 + rl + 8 * h;
        if (t >= p.T) continue;
        const __nv_bfloat16* xrow = p.x + ((size_t)b * 2 * NCHUNK * p.T + t) * 8 + c_lane;
        const RowAddr ya = c8s_row(b, t, 2 * NCHUNK, p.out_phases, p.T);
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const int col = 8 * j + c_lane;
          const uint32_t hw = __ldg(reinterpret_cast<const uint32_t*>(xrow + (size_t)j * p.T * 8));
          const uint32_t lw = __ldg(reinterpret_cast<const uint32_t*>(xrow + (size_t)(NCHUNK + j) * p.T * 8));
          const uint32_t off = (uint32_t)(j * RU_TILE_M + rl + 8 * h) * 16 + c_lane * 2;
          const uint32_t yh = *reinterpret_cast<const uint32_t*>(sA2 + off);
          const uint32_t yl = *reinterpret_cast<const uint32_t*>(sA2 + NCHUNK * RU_TILE_M * 16 + off);
          const float v0 = bf16_lo(hw) + bf16_lo(lw) +
                           (bf16_lo(yh) + bf16_lo(yl)) * sigmoid1(d[4 * j + 2 * h] + sBias[2 * C + NS + col]);
          const float v1 = bf16_hi(hw) + bf16_hi(lw) +
                           (bf16_hi(yh) + bf16_hi(yl)) * sigmoid1(d[4 * j + 2 * h + 1] + sBias[2 * C + NS + col + 1]);
          uint32_t oh, ol;
          split_bf16x2(v0, v1, oh, ol);
          *reinterpret_cast<uint32_t*>(p.y + ya.off + (size_t)j * ya.chunk_stride + c_lane) = oh;
          *reinterpret_cast<uint32_t*>(p.y + ya.off + (size_t)(NCHUNK + j) * ya.chunk_stride + c_lane) = ol;
        }
      }
    } else if constexpr (RB) {
      // ---- E2: D2 + (b1 + bs) (ELU if elu_out) -> split -> global (C8S) ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = t0 + rl + 8 * h;
        if (t >= p.T) continue;
        const RowAddr ya = c8s_row(b, t, 2 * NCHUNK, p.out_phases, p.T);
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const int col = 8 * j + c_lane;
          float v0 = d[4 * j + 2 * h] + sBias[C + col], v1 = d[4 * j + 2 * h + 1] + sBias[C + col + 1];
          if (p.elu_out) {
            v0 = elu1(v0);
            v1 = elu1(v1);
          }
          uint32_t oh, ol;
          split_bf16x2(v0, v1, oh, ol);
          *reinterpret_cast<uint32_t*>(p.y + ya.off + (size_t)j * ya.chunk_stride + c_lane) = oh;
          *reinterpret_cast<uint32_t*>(p.y + ya.off + (size_t)(NCHUNK + j) * ya.chunk_stride + c_lane) = ol;
        }
      }
    } else {
      // ---- E2: D2 (+b1, ELU, + skip) -> split -> global (C8S) ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int t = t0 + rl + 8 * h;
        if (t >= p.T) continue;
        const __nv_bfloat16* xrow = p.x + ((size_t)b * 2 * NCHUNK * p.T + t) * 8 + c_lane;
        const RowAddr ya = c8s_row(b, t, 2 * NCHUNK, p.out_phases, p.T);
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
          const int col = 8 * j + c_lane;
          const uint32_t hw = __ldg(reinterpret_cast<const uint32_t*>(xrow + (size_t)j * p.T * 8));
          const uint32_t lw = __ldg(reinterpret_cast<const uint32_t*>(xrow + (size_t)(NCHUNK + j) * p.T * 8));
          const float v0 = bf16_lo(hw) + bf16_lo(lw) + elu1(d[4 * j + 2 * h] + sBias[C + col]);
          const float v1 = bf16_hi(hw) + bf16_hi(lw) + elu1(d[4 * j + 2 * h + 1] + sBias[C + col + 1]);
          uint32_t oh, ol;
          split_bf16x2(v0, v1, oh, ol);
          *reinterpret_cast<uint32_t*>(p.y + ya.off + (size_t)j * ya.chunk_stride + c_lane) = oh;
          *reinterpret_cast<uint32_t*>(p.y + ya.off + (size_t)(NCHUNK + j) * ya.chunk_stride + c_lane) = ol;
        }
    }
    }
    // every thread's sA2 reads by the D2 (D3) wgmmas have retired (drain above); E1 of the next tile may overwrite it
    asm volatile("bar.sync 1, 128;" ::: "memory");
  }
}

template <int C, bool SE = false, bool RB = false>
static int launch_ru(RuParams p, cudaStream_t stream) {
  using Cfg = RuCfg<C, SE, RB>;
  auto kfn = ru_tc_kernel<C, SE, RB>;
  p.ar = RU_TILE_M + (RB ? 2 : 6 * p.d);
  const int a_bytes = 2 * Cfg::NCHUNK * p.ar * 16;
  int smem;
  if (Cfg::RESIDENT) {
    p.na = 2;
    p.nw = 0;
    smem = 2 * a_bytes + Cfg::W_BYTES + Cfg::FIXED_BYTES;
  } else {
    // the weight ring must cover the L2 latency of the streamed units: as many stages as fit; a second staged
    // activation tile only if that still leaves at least 48 KB of ring
    auto stages = [&](int na) {
      return min(Cfg::MAX_NW, (Cfg::MAX_SMEM - na * a_bytes - Cfg::FIXED_BYTES) / Cfg::UNIT_BYTES);
    };
    p.na = stages(2) * Cfg::UNIT_BYTES >= 48 * 1024 ? 2 : 1;
    p.nw = stages(p.na);
    if (p.nw < 2) return ALM_ERR_UNSUPPORTED;
    smem = p.na * a_bytes + p.nw * Cfg::UNIT_BYTES + Cfg::FIXED_BYTES;
  }
  if (smem > Cfg::MAX_SMEM) return ALM_ERR_UNSUPPORTED;
  static int attr_smem = 0;
  if (smem > attr_smem) {
    ALM_CUDA_OK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_smem = smem;
  }
  const int grid = min(p.total_tiles, num_sms() * Cfg::CTAS_PER_SM);
  kfn<<<grid, RU_THREADS, smem, stream>>>(p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// ---------------------------------------------------------------------------------------------
// plain / strided causal conv (dilation 1) as a pipelined implicit GEMM
//   out[t, co] = b[co] + sum_{j < K} sum_ci W[co, ci, j] xp[ci, t*s + j],  xp[u] = x[u - (K - s)]  (soundstream.py:332-345)
// Input: C8S with P = s phase planes, so tap j of output row t reads plane ((j - pad) mod s), row t + floor((j - pad) / s):
// unit-stride rows for every tap.  One pipeline stage = one (tap, 16-channel k-step) unit: A hi/lo [2][128][16 B] each
// (cp.async, 16 B per lane), W hi/lo [2][BN][16 B] each (one bulk copy); three wgmmas per stage and consumer warpgroup.
// Warps 0 and 3: producers; warps 4-7 / 8-11: consumer warpgroups for tile rows [0, 64) / [64, 128).
// ---------------------------------------------------------------------------------------------
constexpr int CTA_THREADS = 384;

struct ConvParams {
  const __nv_bfloat16* x;   // C8S [B][2 Cin/8][s][Tin/s][8]
  void* y;                  // C8S (out_phases) or fp32 [B][n_out][Cout]
  const __nv_bfloat16* w;   // [ntile][tap][kstep][part][2][BN][8]
  const float* bias;
  int B, Cin, Cout, Tin, n_out, K, s, pad_mode, out_phases, out_fp32;
  int up;  // > 1: the Cout = up * C' output columns are `up` consecutive time steps of C' channels (transposed conv)
  int m_tiles, n_tiles, total_tiles;
};

template <int BN>
struct ConvCfg {
  static constexpr int A_BYTES = 4 * TILE_M * 16;       // hi c0, hi c1, lo c0, lo c1
  static constexpr int W_BYTES = 4 * BN * 16;
  static constexpr int STAGE_BYTES = A_BYTES + W_BYTES;
  static constexpr int STAGES = BN == 256 ? 8 : 10;
  static constexpr int LOOKAHEAD = 3;                   // cp.async groups in flight PER PRODUCER WARP before its oldest is published
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 512 + 128;
};

template <int BN>
__global__ void __launch_bounds__(CTA_THREADS, 1) conv_tc_kernel(const ConvParams p) {
  using Cfg = ConvCfg<BN>;
  constexpr int STAGES = Cfg::STAGES, LA = Cfg::LOOKAHEAD;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;                  // [STAGES]  count 2: W bulk copy (expect_tx) + A (cp.async groups)
  uint64_t* empty = bars + STAGES;        // [STAGES]  one arrive per consumer warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 2);
      mbar_init(&empty[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int ksteps = p.Cin / 16;
  const int nch = p.Cin / 8;            // chunks per part
  const int units = p.K * ksteps;
  const int pad = p.K - p.s;
  const int rows_in = p.Tin / p.s;      // rows of one phase plane
  // tile -> (b, mt, nt): n fastest so the two N halves of a wide layer run back to back on the same A rows (L2 reuse)
  auto decode = [&](int tile, int& b, int& mt, int& nt) {
    nt = tile % p.n_tiles;
    const int r = tile / p.n_tiles;
    mt = r % p.m_tiles;
    b = r / p.m_tiles;
  };

  if (warp < 4) {
    if (warp == 1 || warp == 2) return;
    // ===================== two producer warps (all 32 lanes each): warp 0 stages the even units, warp 3 the odd ones
    // (one warp's address arithmetic + issue of 16 cp.async per stage cannot keep the small-N layers fed) ============
    const int pid = warp == 0 ? 0 : 1;
    int stage = 0, pending = 0, k = 0, done_m = 0;
    uint32_t phase = 0;
    auto publish_oldest = [&]() {  // this warp's oldest cp.async group has landed: make it visible to wgmma, signal
      fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[(2 * done_m + pid) % STAGES]);
      ++done_m;
      --pending;
    };
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      int b, mt, nt;
      decode(tile, b, mt, nt);
      const int t0 = mt * TILE_M;
      const int nrows = min(TILE_M, p.n_out - t0);
      const __nv_bfloat16* xb = p.x + (size_t)b * 2 * nch * p.s * (size_t)rows_in * 8;
      for (int j = 0; j < p.K; ++j) {
        const int q = j - pad;
        const int plane = ((q % p.s) + p.s) % p.s;
        const int shift = (q - plane) / p.s;   // floor(q / s)
        // per-lane source rows of this tap (row r of the tile -> x row, or the padding rule when it is negative)
        size_t src_row[TILE_M / 32];
        uint32_t src_bytes[TILE_M / 32];
#pragma unroll
        for (int it = 0; it < TILE_M / 32; ++it) {
          const int r = it * 32 + lane;
          int pl = plane, rw = t0 + r + shift;
          uint32_t bytes = 16;
          if (rw < 0) {  // x index u = (t0 + r) * s + q < 0
            const int u = (t0 + r) * p.s + q;
            if (p.pad_mode == 0) { pl = (-u) % p.s; rw = (-u) / p.s; }   // reflect
            else if (p.pad_mode == 2) { pl = 0; rw = 0; }                 // replicate
            else { pl = 0; rw = 0; bytes = 0; }                           // constant zero
          }
          src_row[it] = ((size_t)pl * rows_in + rw) * 8;
          src_bytes[it] = bytes;
        }
        for (int kk = 0; kk < ksteps; ++kk, ++k) {
          if ((k & 1) != pid) {  // the other producer's unit
            if (++stage == STAGES) { stage = 0; phase ^= 1u; }
            continue;
          }
          mbar_wait(&empty[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
#pragma unroll
          for (int part = 0; part < 2; ++part)
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
              const int c = part * nch + 2 * kk + cc;
              const __nv_bfloat16* plane0 = xb + (size_t)c * p.s * (size_t)rows_in * 8;
              uint8_t* dst = sa + (part * 2 + cc) * (TILE_M * 16);
#pragma unroll
              for (int it = 0; it < TILE_M / 32; ++it) {
                const int r = it * 32 + lane;
                if (r < nrows) cp_async_16(dst + r * 16, plane0 + src_row[it], src_bytes[it]);
              }
            }
          cp_async_commit();
          if (lane == 0) {
            mbar_arrive_expect_tx(&full[stage], Cfg::W_BYTES);
            bulk_copy_g2s(sa + Cfg::A_BYTES, p.w + (((size_t)nt * p.K + j) * ksteps + kk) * (size_t)(Cfg::W_BYTES / 2),
                          Cfg::W_BYTES, &full[stage]);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
          if (++pending > LA) {
            cp_async_wait<LA>();
            publish_oldest();
          }
        }
      }
    }
    cp_async_wait<0>();
    while (pending > 0) publish_oldest();
    return;
  }

  // ===================== consumer warpgroups =====================
  const int cw = (warp >> 2) - 1;
  const int rl = cw * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment rows rl, rl + 8 of the tile
  const int c_lane = 2 * (lane & 3);
  const int nch_out = p.Cout / 8;
  int stage = 0;
  uint32_t phase = 0;
  // descriptors built once; per stage only the start-address field moves
  const uint64_t a0 = wgmma_desc_nosw(smem_u32(smem) + cw * 64 * 16, 128, TILE_M * 16);
  const uint64_t b0 = wgmma_desc_nosw(smem_u32(smem) + Cfg::A_BYTES, 128, BN * 16);
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
    int b, mt, nt;
    decode(tile, b, mt, nt);
    int prev = -1;
    for (int u = 0; u < units; ++u) {
      mbar_wait(&full[stage], phase);
      const uint64_t off = (uint64_t)(stage * (Cfg::STAGE_BYTES / 16));
      const uint64_t a_hi = a0 + off, a_lo = a_hi + 2 * TILE_M;
      const uint64_t b_hi = b0 + off, b_lo = b_hi + 2 * BN;
      wgmma_fence();
      wgmma_ss<BN>(acc, a_hi, b_hi, u > 0 ? 1u : 0u);
      wgmma_ss<BN>(acc, a_lo, b_hi, 1u);
      wgmma_ss<BN>(acc, a_hi, b_lo, 1u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);

    const int n0 = nt * BN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int t = mt * TILE_M + rl + 8 * h;
      if (t >= p.n_out) continue;
      const RowAddr ya = c8s_row(b, t, 2 * nch_out, p.out_fp32 ? 1 : p.out_phases, p.n_out);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int ch = n0 + 8 * j + c_lane;  // this thread's channels ch, ch + 1 of the 8-channel chunk n0 / 8 + j
        const float v0 = acc[4 * j + 2 * h] + (p.bias ? __ldg(p.bias + ch) : 0.f);
        const float v1 = acc[4 * j + 2 * h + 1] + (p.bias ? __ldg(p.bias + ch + 1) : 0.f);
        if (p.out_fp32) {
          float* dst = reinterpret_cast<float*>(p.y) + ((size_t)b * p.n_out + t) * p.Cout + ch;
          *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
          continue;
        }
        uint32_t oh, ol;
        split_bf16x2(v0, v1, oh, ol);
        __nv_bfloat16* yb = reinterpret_cast<__nv_bfloat16*>(p.y);
        if (p.up > 1) {
          // CausalConvTranspose1d as a 2-tap conv with up * C' output columns: column block r is output time t * up + r
          const int ch0 = ch - c_lane;
          const int creal = p.Cout / p.up, r_ = ch0 / creal, cbase = ch0 - r_ * creal;
          const size_t t_out = (size_t)t * p.up + r_, T_out = (size_t)p.n_out * p.up;
          const int nchr = creal / 8;
          const int chunk = cbase / 8;
          *reinterpret_cast<uint32_t*>(yb + (((size_t)b * 2 * nchr + chunk) * T_out + t_out) * 8 + c_lane) = oh;
          *reinterpret_cast<uint32_t*>(yb + (((size_t)b * 2 * nchr + nchr + chunk) * T_out + t_out) * 8 + c_lane) = ol;
        } else {
          const int chunk = (n0 >> 3) + j;
          *reinterpret_cast<uint32_t*>(yb + ya.off + (size_t)chunk * ya.chunk_stride + c_lane) = oh;
          *reinterpret_cast<uint32_t*>(yb + ya.off + (size_t)(nch_out + chunk) * ya.chunk_stride + c_lane) = ol;
        }
      }
    }
  }
}

template <int BN>
static int launch_conv(const ConvParams& p, cudaStream_t stream) {
  using Cfg = ConvCfg<BN>;
  auto kfn = conv_tc_kernel<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    ALM_CUDA_OK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int grid = min(p.total_tiles, num_sms());
  kfn<<<grid, CTA_THREADS, Cfg::SMEM_BYTES, stream>>>(p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

}  // namespace ctc
}  // namespace alm

extern "C" int alm_codec_first_conv(const float* x, const float* w, const float* bias, void* y, int B, int T, int Cout,
                                    int K, int pad_mode, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && w && y && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(K >= 1 && K <= 8 && pad_mode >= 0 && pad_mode <= 2, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(T > K - 1, ALM_ERR_ARG);
  dim3 grid(ceil_div(T, 128), min(B, 65535));
  __nv_bfloat16* yy = reinterpret_cast<__nv_bfloat16*>(y);
  if (Cout == 32) ctc::first_conv_kernel<32><<<grid, 128, 0, stream>>>(x, w, bias, yy, B, T, K, pad_mode);
  else if (Cout == 64) ctc::first_conv_kernel<64><<<grid, 128, 0, stream>>>(x, w, bias, yy, B, T, K, pad_mode);
  else return ALM_ERR_UNSUPPORTED;
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_codec_ru_tc(const void* x, void* y, const void* w_units, const float* b7, const float* b1, int B,
                               int C, int T, int dilation, int pad_mode, int out_phases, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && y && w_units && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(dilation >= 1 && 6 * dilation <= ctc::MAX_HALO && pad_mode >= 0 && pad_mode <= 2, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(T > 6 * dilation, ALM_ERR_ARG);
  ALM_REQUIRE(out_phases >= 1 && T % out_phases == 0, ALM_ERR_ARG);
  ctc::RuParams p;
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.w = reinterpret_cast<const __nv_bfloat16*>(w_units);
  p.b7 = b7;
  p.b1 = b1;
  p.B = B; p.T = T; p.d = dilation; p.pad_mode = pad_mode; p.out_phases = out_phases;
  p.tiles_per_clip = ceil_div(T, ctc::RU_TILE_M);
  p.total_tiles = p.tiles_per_clip * B;
  switch (C) {
    case 32: return ctc::launch_ru<32>(p, stream);
    case 64: return ctc::launch_ru<64>(p, stream);
    case 128: return ctc::launch_ru<128>(p, stream);
    case 256: return ctc::launch_ru<256>(p, stream);
    default: return ALM_ERR_UNSUPPORTED;
  }
}

extern "C" int alm_codec_ru_se_tc(const void* x, void* y, const void* w_units, const float* b7, const float* b1,
                                  const float* se_b1, const float* se_b2, int B, int C, int se_ci, int T, int dilation,
                                  int pad_mode, int out_phases, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && y && w_units && se_b1 && se_b2 && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(dilation >= 1 && 6 * dilation <= ctc::MAX_HALO && pad_mode >= 0 && pad_mode <= 2, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(T > 6 * dilation, ALM_ERR_ARG);
  ALM_REQUIRE(out_phases >= 1 && T % out_phases == 0, ALM_ERR_ARG);
  ctc::RuParams p;
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.w = reinterpret_cast<const __nv_bfloat16*>(w_units);
  p.b7 = b7;
  p.b1 = b1;
  p.se_b1 = se_b1;
  p.se_b2 = se_b2;
  p.se_ci = se_ci;
  p.B = B; p.T = T; p.d = dilation; p.pad_mode = pad_mode; p.out_phases = out_phases;
  p.tiles_per_clip = ceil_div(T, ctc::RU_TILE_M);
  p.total_tiles = p.tiles_per_clip * B;
  auto inner_ok = [&](int ns) { return se_ci >= 1 && se_ci <= ns; };
  switch (C) {
    case 32: return inner_ok(ctc::RuCfg<32, true>::NS) ? ctc::launch_ru<32, true>(p, stream) : ALM_ERR_UNSUPPORTED;
    case 64: return inner_ok(ctc::RuCfg<64, true>::NS) ? ctc::launch_ru<64, true>(p, stream) : ALM_ERR_UNSUPPORTED;
    case 128: return inner_ok(ctc::RuCfg<128, true>::NS) ? ctc::launch_ru<128, true>(p, stream) : ALM_ERR_UNSUPPORTED;
    case 256: return inner_ok(ctc::RuCfg<256, true>::NS) ? ctc::launch_ru<256, true>(p, stream) : ALM_ERR_UNSUPPORTED;
    default: return ALM_ERR_UNSUPPORTED;
  }
}

extern "C" int alm_codec_conv_tc(const void* x, void* y, const void* w_units, const float* bias, int B, int Cin,
                                 int Cout, int Tin, int K, int stride, int pad_mode, int out_phases, int out_fp32,
                                 int upsample, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && y && w_units && B > 0 && Tin > 0, ALM_ERR_ARG);
  ALM_REQUIRE(Cin % 16 == 0 && K >= stride && stride >= 1 && Tin % stride == 0, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(pad_mode >= 0 && pad_mode <= 2, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(Tin > K, ALM_ERR_ARG);
  const int BN = Cout % 256 == 0 ? 256 : (Cout % 128 == 0 ? 128 : 64);
  ALM_REQUIRE(Cout % BN == 0, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(upsample >= 1 && Cout % upsample == 0 && (upsample == 1 || ((Cout / upsample) % 16 == 0 && !out_fp32)),
              ALM_ERR_UNSUPPORTED);
  ctc::ConvParams p;
  p.up = upsample;
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.y = y;
  p.w = reinterpret_cast<const __nv_bfloat16*>(w_units);
  p.bias = bias;
  p.B = B; p.Cin = Cin; p.Cout = Cout; p.Tin = Tin; p.K = K; p.s = stride; p.pad_mode = pad_mode;
  p.n_out = Tin / stride;  // causal padding K - s keeps exactly Tin / s outputs
  p.out_phases = out_phases; p.out_fp32 = out_fp32;
  ALM_REQUIRE(out_fp32 || (out_phases >= 1 && p.n_out % out_phases == 0), ALM_ERR_ARG);
  p.m_tiles = ceil_div(p.n_out, ctc::TILE_M);
  p.n_tiles = Cout / BN;
  p.total_tiles = B * p.m_tiles * p.n_tiles;
  if (BN == 256) return ctc::launch_conv<256>(p, stream);
  if (BN == 128) return ctc::launch_conv<128>(p, stream);
  return ctc::launch_conv<64>(p, stream);
}

extern "C" int alm_encodec_resblock_tc(const void* x, void* y, const void* w_units, const float* b3, const float* b_out,
                                       int B, int C, int T, int elu_out, int out_phases, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && y && w_units && b3 && b_out && B > 0, ALM_ERR_ARG);
  ALM_REQUIRE(T > 2, ALM_ERR_ARG);  // the reflect halo of the k3 conv
  ALM_REQUIRE(out_phases >= 1 && T % out_phases == 0, ALM_ERR_ARG);
  ctc::RuParams p;
  p.x = reinterpret_cast<const __nv_bfloat16*>(x);
  p.y = reinterpret_cast<__nv_bfloat16*>(y);
  p.w = reinterpret_cast<const __nv_bfloat16*>(w_units);
  p.b7 = b3;
  p.b1 = b_out;
  p.B = B; p.T = T; p.d = 1; p.pad_mode = 0; p.out_phases = out_phases; p.elu_out = elu_out;
  p.tiles_per_clip = ceil_div(T, ctc::RU_TILE_M);
  p.total_tiles = p.tiles_per_clip * B;
  switch (C) {
    case 32: return ctc::launch_ru<32, false, true>(p, stream);
    case 64: return ctc::launch_ru<64, false, true>(p, stream);
    case 128: return ctc::launch_ru<128, false, true>(p, stream);
    case 256: return ctc::launch_ru<256, false, true>(p, stream);
    default: return ALM_ERR_UNSUPPORTED;
  }
}

extern "C" int alm_codec_pack_c8s(const float* x, void* y, int B, int n, int C, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && y && B > 0 && n > 0 && C > 0 && C % 8 == 0, ALM_ERR_ARG);
  const long long total = (long long)B * n * (C / 8);
  const long long want_blocks = (total + 255) / 256;
  const int grid = (int)(want_blocks < num_sms() * 16 ? want_blocks : num_sms() * 16);
  ctc::pack_c8s_kernel<<<grid, 256, 0, stream>>>(x, reinterpret_cast<__nv_bfloat16*>(y), B, n, C);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_codec_last_conv(const void* x, const float* w, const float* bias, float* y, int B, int T, int Cin,
                                   int K, int pad_mode, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(x && w && y && B > 0 && T > 0, ALM_ERR_ARG);
  ALM_REQUIRE(K >= 1 && K <= 8 && pad_mode >= 0 && pad_mode <= 2 && T > K - 1, ALM_ERR_UNSUPPORTED);
  dim3 grid(ceil_div(T, 128), min(B, 65535));
  const __nv_bfloat16* xx = reinterpret_cast<const __nv_bfloat16*>(x);
  if (Cin == 32) ctc::last_conv_kernel<32><<<grid, 128, 0, stream>>>(xx, w, bias, y, B, T, K, pad_mode);
  else if (Cin == 64) ctc::last_conv_kernel<64><<<grid, 128, 0, stream>>>(xx, w, bias, y, B, T, K, pad_mode);
  else return ALM_ERR_UNSUPPORTED;
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
