// Multi-query causal attention backward for sm_90a (autograd of attend.py:69-146), two kernels:
//
//  dKV kernel: one CTA = (batch, 128 keys).  It walks every (head, query block) that can see these keys
//      S^T = K Q^T,  dP^T = V dO^T                       (wgmma, both operands in smem)
//      P^T = exp(S^T*scale - lse),  dS^T = scale * P^T (dP^T - delta)   (on the accumulator fragments)
//      dV += P^T dO,  dK += dS^T Q                       (wgmma with P^T / dS^T as register A operands; accumulated
//                                                          in registers over all heads: MQA shares k/v, so no atomics)
//  dQ kernel: one CTA = (batch, head, 128 queries), walks the key tiles:
//      S = Q K^T, dP = dO V^T, dS = scale * P (dP - delta), dQ += dS K.
//
// Q/K/V/dO tiles arrive by TMA (SWIZZLE_128B); the SAME smem tile serves as a K-major operand
// (contraction over the 64-wide head dim) and as an MN-major operand (contraction over its 128 rows).
// Warps 0-3 / 4-7 are the two consumer warpgroups (tile rows [0, 64) / [64, 128)).  There is no producer warp: a
// separate one would cap every thread at 168 registers, and the dQ / dK / dV products need more.  Warp 0 refills a
// pipeline slot as soon as both warpgroups have released it; STAGES - 1 loads stay in flight.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {

constexpr int AB_T = 128;                     // tile edge (queries or keys)
constexpr int AB_D = 64;
constexpr int AB_TILE = AB_T * AB_D * 2;      // 16 KB
constexpr int AB_THREADS = 256;               // two consumer warpgroups; warp 0 also issues the TMA loads
constexpr int AB_STAGES = 3;
constexpr float LOG2E = 1.4426950408889634f;

struct AttnBwdParams {
  const float* lse;      // [b, h, n_q_pad]  log2-domain LSE (m + log2 l) as written by the forward
  const float* delta;    // [b, h, n_q_pad]
  const uint32_t* kmask;  // packed key mask bits (alm_pack_key_mask) or null
  int kb_stride;          // words per batch row
  const float* bias;     // [h, n_q, bias_rs] additive score bias (as given to the forward) or null
  float* dbias;          // same layout, fp32: d(bias) is ACCUMULATED (red.add) over batches / calls; or null
  long long bias_hs, bias_rs;
  __nv_bfloat16* dq;     // [b, n_q, h*64], row stride lddq
  __nv_bfloat16* dk;     // [b, n_k, 64], row stride lddk
  __nv_bfloat16* dv;
  long long lddq, lddk, lddv;
  int b, h, n_q, n_k, n_q_pad;
  int causal;
  float scale, scale_log2;
};

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// fp32 accumulator fragment of an m64n128 product -> the 8 bf16 A fragments (k16 steps) of the next product
__device__ __forceinline__ void pack_a_frags(const float (&v)[64], uint32_t (&a)[8][4]) {
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    a[kk][0] = pack_bf16x2(v[8 * kk + 0], v[8 * kk + 1]);
    a[kk][1] = pack_bf16x2(v[8 * kk + 2], v[8 * kk + 3]);
    a[kk][2] = pack_bf16x2(v[8 * kk + 4], v[8 * kk + 5]);
    a[kk][3] = pack_bf16x2(v[8 * kk + 6], v[8 * kk + 7]);
  }
}

// store rows r_base + 8 h of an m64n64 fp32 fragment as bf16 (row -> dst row pointer, or null to skip)
__device__ __forceinline__ void store_d64(const float (&acc)[32], __nv_bfloat16* row0, __nv_bfloat16* row1, int c_lane) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    __nv_bfloat16* dst = h == 0 ? row0 : row1;
    if (dst == nullptr) continue;
#pragma unroll
    for (int g = 0; g < 8; ++g)
      *reinterpret_cast<uint32_t*>(dst + 8 * g + c_lane) = pack_bf16x2(acc[4 * g + 2 * h], acc[4 * g + 2 * h + 1]);
  }
}

// ================================================================================================
// dK / dV
// ================================================================================================
constexpr int DKV_SMEM = AB_TILE * (2 + 2 * AB_STAGES) + AB_STAGES * 2 * 512 + 256;

template <bool HAS_BIAS>
__global__ void __launch_bounds__(AB_THREADS, 1)
mqa_attn_bwd_dkv_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                        const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                        const AttnBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sK = smem;
  uint8_t* sV = sK + AB_TILE;
  uint8_t* sQ = sV + AB_TILE;                    // [stages]
  uint8_t* sdO = sQ + AB_STAGES * AB_TILE;       // [stages]
  float* sLse = reinterpret_cast<float*>(sdO + AB_STAGES * AB_TILE);  // [stages][128]
  float* sDelta = sLse + AB_STAGES * AB_T;                            // [stages][128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sDelta + AB_STAGES * AB_T);
  uint64_t* kv_full = bars;
  uint64_t* qdo_full = bars + 1;              // [stages]
  uint64_t* qdo_empty = qdo_full + AB_STAGES; // [stages]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // heaviest key blocks first across ALL batches (LPT order): CTA x -> (kb = x / b, batch = x % b)
  const int kb = blockIdx.x / p.b, batch = blockIdx.x % p.b;
  const int k0 = kb * AB_T;
  const int off = p.n_k - p.n_q;
  const int n_qblocks = (p.n_q + AB_T - 1) / AB_T;
  int qb_min = 0;
  if (p.causal && k0 - off > 0) qb_min = (k0 - off) / AB_T;
  const int q_per_head = n_qblocks - qb_min;
  const int n_iter = q_per_head > 0 ? q_per_head * p.h : 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmdO);
    mbar_init(kv_full, 1);
    for (int i = 0; i < AB_STAGES; ++i) { mbar_init(&qdo_full[i], 1); mbar_init(&qdo_empty[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  // TMA issue (warp 0, one elected lane): K / V once, then Q / dO / lse / delta of iteration `it` into slot it % STAGES
  auto issue_qdo = [&](int it) {
    const int st = it % AB_STAGES;
    const int head = it / q_per_head, qb = qb_min + it % q_per_head;
    const size_t roff = ((size_t)batch * p.h + head) * p.n_q_pad + (size_t)qb * AB_T;
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(&qdo_full[st], 2 * AB_TILE + 2 * AB_T * 4);
      tma_load_3d(sQ + st * AB_TILE, &tmQ, &qdo_full[st], head * AB_D, qb * AB_T, batch);
      tma_load_3d(sdO + st * AB_TILE, &tmdO, &qdo_full[st], head * AB_D, qb * AB_T, batch);
      bulk_copy_g2s(sLse + st * AB_T, p.lse + roff, AB_T * 4, &qdo_full[st]);
      bulk_copy_g2s(sDelta + st * AB_T, p.delta + roff, AB_T * 4, &qdo_full[st]);
    }
    __syncwarp();
  };
  if (warp == 0 && n_iter > 0) {
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(kv_full, 2 * AB_TILE);
      tma_load_3d(sK, &tmK, kv_full, 0, k0, batch);
      tma_load_3d(sV, &tmV, kv_full, 0, k0, batch);
    }
    __syncwarp();
    for (int it = 0; it < min(n_iter, AB_STAGES); ++it) issue_qdo(it);
  }

  // consumers: warpgroup cw owns key rows [64 cw, 64 cw + 64); fragment rows r_base + 8 h, columns 8 g + c_lane + c
  const int cw = warp >> 2;
  const int r_base = cw * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c_lane = 2 * (lane & 3);
  int kj[2];
  bool key_ok[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    kj[h] = k0 + r_base + 8 * h;
    key_ok[h] = kj[h] < p.n_k;
    if (key_ok[h] && p.kmask != nullptr)
      key_ok[h] = (p.kmask[(size_t)batch * p.kb_stride + (kj[h] >> 5)] >> (kj[h] & 31)) & 1u;
  }
  float dv[32], dk[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) { dv[e] = 0.f; dk[e] = 0.f; }
  const uint32_t k_addr = smem_u32(sK) + cw * 8192, v_addr = smem_u32(sV) + cw * 8192;
  if (n_iter > 0) mbar_wait(kv_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < n_iter; ++it) {
    const int qb = qb_min + it % q_per_head;
    const int q0 = qb * AB_T;
    [[maybe_unused]] const long long bias_head = HAS_BIAS ? (long long)(it / q_per_head) * p.bias_hs : 0;
    mbar_wait(&qdo_full[stage], phase);
    const uint32_t q_addr = smem_u32(sQ + stage * AB_TILE), do_addr = smem_u32(sdO + stage * AB_TILE);
    float st[64], dpt[64];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AB_D / 16; ++k)
      wgmma_ss<AB_T>(st, wgmma_desc_sw128(k_addr + k * 32, 1024, 16), wgmma_desc_sw128(q_addr + k * 32, 1024, 16),
                     k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < AB_D / 16; ++k)
      wgmma_ss<AB_T>(dpt, wgmma_desc_sw128(v_addr + k * 32, 1024, 16), wgmma_desc_sw128(do_addr + k * 32, 1024, 16),
                     k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(st);
    wgmma_fence_acc(dpt);
    const float* lse_s = sLse + stage * AB_T;
    const float* del_s = sDelta + stage * AB_T;
    // whole tile below the causal diagonal and inside n_q: only the per-row key flag matters
    const bool tile_full = (q0 + AB_T <= p.n_q) && (!p.causal || k0 + AB_T - 1 <= q0 + off);
#pragma unroll
    for (int g = 0; g < AB_T / 8; ++g)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = 8 * g + c_lane + c;
        const int qi = q0 + col;
        const float lv = lse_s[col], dl = del_s[col];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int e = 4 * g + 2 * h + c;
          const bool ok = key_ok[h] && (tile_full || (qi < p.n_q && (!p.causal || kj[h] <= qi + off)));
          float shift = -lv;
          [[maybe_unused]] long long bidx = 0;
          if constexpr (HAS_BIAS) {
            bidx = bias_head + (long long)min(qi, p.n_q - 1) * p.bias_rs + min(kj[h], p.n_k - 1);
            shift = fmaf(__ldg(p.bias + bidx), LOG2E, shift);
          }
          const float pe = ok ? ex2_approx(fmaf(st[e], p.scale_log2, shift)) : 0.f;
          const float ds = ok ? pe * (dpt[e] - dl) : 0.f;
          if constexpr (HAS_BIAS) {
            if (ok && p.dbias != nullptr) atomicAdd(p.dbias + bidx, ds);
          }
          st[e] = pe;
          dpt[e] = ds * p.scale;
        }
      }
    uint32_t pa[8][4], da[8][4];
    pack_a_frags(st, pa);
    pack_a_frags(dpt, da);
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_T / 16; ++kk)
      wgmma_rs<AB_D, 1>(dv, pa[kk], wgmma_desc_sw128(do_addr + kk * 2048, 1024, 8192), 1u);
#pragma unroll
    for (int kk = 0; kk < AB_T / 16; ++kk)
      wgmma_rs<AB_D, 1>(dk, da[kk], wgmma_desc_sw128(q_addr + kk * 2048, 1024, 8192), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    if (lane == 0) mbar_arrive(&qdo_empty[stage]);
    if (warp == 0 && it + AB_STAGES < n_iter) {  // refill this slot once both warpgroups are done with it
      mbar_wait(&qdo_empty[stage], phase);
      issue_qdo(it + AB_STAGES);
    }
    if (++stage == AB_STAGES) { stage = 0; phase ^= 1u; }
  }
  // epilogue: dV, dK from registers
  __nv_bfloat16* rv[2];
  __nv_bfloat16* rk[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const bool in = kj[h] < p.n_k;
    rv[h] = in ? p.dv + ((size_t)batch * p.n_k + kj[h]) * p.lddv : nullptr;
    rk[h] = in ? p.dk + ((size_t)batch * p.n_k + kj[h]) * p.lddk : nullptr;
  }
  store_d64(dv, rv[0], rv[1], c_lane);
  store_d64(dk, rk[0], rk[1], c_lane);
}

// ================================================================================================
// dQ
// ================================================================================================
constexpr int DQ_STAGES = 4;
constexpr int DQ_SMEM = AB_TILE * (2 + 2 * DQ_STAGES) + 256;

template <bool HAS_BIAS>
__global__ void __launch_bounds__(AB_THREADS, 1)
mqa_attn_bwd_dq_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                       const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                       const AttnBwdParams p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sQ = smem;
  uint8_t* sdO = sQ + AB_TILE;
  uint8_t* sK = sdO + AB_TILE;                 // [stages]
  uint8_t* sV = sK + DQ_STAGES * AB_TILE;      // [stages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + DQ_STAGES * AB_TILE);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;
  uint64_t* kv_empty = kv_full + DQ_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_qblocks = (p.n_q + AB_T - 1) / AB_T;
  const int qb = n_qblocks - 1 - (int)blockIdx.x;
  const int head = blockIdx.y, batch = blockIdx.z;
  const int q0 = qb * AB_T;
  const int off = p.n_k - p.n_q;
  int kv_end = p.n_k;
  if (p.causal) kv_end = min(p.n_k, q0 + AB_T + off);
  const int n_tiles = kv_end > 0 ? (kv_end + AB_T - 1) / AB_T : 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV); tma_prefetch_desc(&tmdO);
    mbar_init(q_full, 1);
    for (int i = 0; i < DQ_STAGES; ++i) { mbar_init(&kv_full[i], 1); mbar_init(&kv_empty[i], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  // TMA issue (warp 0, one elected lane): Q / dO once, then the K / V tile j into slot j % STAGES
  auto issue_kv = [&](int j) {
    const int st = j % DQ_STAGES;
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(&kv_full[st], 2 * AB_TILE);
      tma_load_3d(sK + st * AB_TILE, &tmK, &kv_full[st], 0, j * AB_T, batch);
      tma_load_3d(sV + st * AB_TILE, &tmV, &kv_full[st], 0, j * AB_T, batch);
    }
    __syncwarp();
  };
  if (warp == 0 && n_tiles > 0) {
    if (elect_one_sync()) {
      mbar_arrive_expect_tx(q_full, 2 * AB_TILE);
      tma_load_3d(sQ, &tmQ, q_full, head * AB_D, q0, batch);
      tma_load_3d(sdO, &tmdO, q_full, head * AB_D, q0, batch);
    }
    __syncwarp();
    for (int j = 0; j < min(n_tiles, DQ_STAGES); ++j) issue_kv(j);
  }

  // consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64)
  const int cw = warp >> 2;
  const int r_base = cw * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c_lane = 2 * (lane & 3);
  int qi[2], q_limit[2];
  float lse[2], delta[2];
  [[maybe_unused]] const float* brow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    qi[h] = q0 + r_base + 8 * h;
    const size_t roff = ((size_t)batch * p.h + head) * p.n_q_pad + qi[h];
    lse[h] = p.lse[roff];          // log2-domain; n_q_pad >= n_qblocks*128: always in bounds
    delta[h] = p.delta[roff];
    q_limit[h] = p.causal ? qi[h] + off : p.n_k - 1;
    if constexpr (HAS_BIAS) brow[h] = p.bias + (long long)head * p.bias_hs + (long long)min(qi[h], p.n_q - 1) * p.bias_rs;
  }
  const uint32_t* mrow = p.kmask ? p.kmask + (size_t)batch * p.kb_stride : nullptr;
  const uint32_t q_addr = smem_u32(sQ) + cw * 8192, do_addr = smem_u32(sdO) + cw * 8192;
  float dq[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) dq[e] = 0.f;
  if (n_tiles > 0) mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < n_tiles; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t k_addr = smem_u32(sK + stage * AB_TILE), v_addr = smem_u32(sV + stage * AB_TILE);
    float sc[64], dp[64];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AB_D / 16; ++k)
      wgmma_ss<AB_T>(sc, wgmma_desc_sw128(q_addr + k * 32, 1024, 16), wgmma_desc_sw128(k_addr + k * 32, 1024, 16),
                     k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < AB_D / 16; ++k)
      wgmma_ss<AB_T>(dp, wgmma_desc_sw128(do_addr + k * 32, 1024, 16), wgmma_desc_sw128(v_addr + k * 32, 1024, 16),
                     k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(sc);
    wgmma_fence_acc(dp);
    const int kbase = j * AB_T;
    const bool tile_full = mrow == nullptr && (q0 + AB_T <= p.n_q) && (kbase + AB_T <= p.n_k) &&
                           (!p.causal || kbase + AB_T - 1 <= q0 + off);
    uint32_t mbits[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
    if (mrow != nullptr) {
      const uint4 mv = __ldg(reinterpret_cast<const uint4*>(mrow + j * 4));
      mbits[0] = mv.x; mbits[1] = mv.y; mbits[2] = mv.z; mbits[3] = mv.w;
    }
#pragma unroll
    for (int g = 0; g < AB_T / 8; ++g)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = 8 * g + c_lane + c;
        const int kj = kbase + col;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int e = 4 * g + 2 * h + c;
          bool ok = tile_full;
          if (!tile_full) ok = qi[h] < p.n_q && kj < p.n_k && kj <= q_limit[h] && ((mbits[col >> 5] >> (col & 31)) & 1u);
          float shift = -lse[h];
          if constexpr (HAS_BIAS) {
            // bias_rs is a multiple of 4 and >= n_k: columns past the padded row read 0
            if (kj < p.bias_rs) shift = fmaf(__ldg(brow[h] + kj), LOG2E, shift);
          }
          const float pe = ok ? ex2_approx(fmaf(sc[e], p.scale_log2, shift)) : 0.f;
          sc[e] = ok ? pe * (dp[e] - delta[h]) * p.scale : 0.f;
        }
      }
    uint32_t da[8][4];
    pack_a_frags(sc, da);
    wgmma_fence_acc(dq);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_T / 16; ++kk)
      wgmma_rs<AB_D, 1>(dq, da[kk], wgmma_desc_sw128(k_addr + kk * 2048, 1024, 8192), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dq);
    if (lane == 0) mbar_arrive(&kv_empty[stage]);
    if (warp == 0 && j + DQ_STAGES < n_tiles) {  // refill this slot once both warpgroups are done with it
      mbar_wait(&kv_empty[stage], phase);
      issue_kv(j + DQ_STAGES);
    }
    if (++stage == DQ_STAGES) { stage = 0; phase ^= 1u; }
  }
  __nv_bfloat16* rq[2];
#pragma unroll
  for (int h = 0; h < 2; ++h)
    rq[h] = qi[h] < p.n_q ? p.dq + ((size_t)batch * p.n_q + qi[h]) * p.lddq + head * AB_D : nullptr;
  store_d64(dq, rq[0], rq[1], c_lane);
}

}  // namespace alm

extern "C" int alm_mqa_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, int64_t k_bstride,
                                const void* v, int64_t ldv, int64_t v_bstride, const void* d_o, int64_t lddo,
                                const void* key_mask, const float* lse, const float* delta, int n_q_pad, void* dq,
                                int64_t lddq, void* dk, int64_t lddk, void* dv, int64_t lddv, const float* bias,
                                float* dbias, int64_t bias_hstride, int64_t bias_rstride, int b, int h, int n_q,
                                int n_k, int causal, float scale, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(q && k && v && d_o && lse && delta && dq && dk && dv, ALM_ERR_ARG);
  ALM_REQUIRE(b > 0 && h > 0 && n_q > 0 && n_k >= n_q, ALM_ERR_ARG);
  ALM_REQUIRE(n_q_pad % AB_T == 0 && n_q_pad >= n_q, ALM_ERR_ARG);
  if (bias != nullptr) {
    ALM_REQUIRE(bias_rstride >= n_k && bias_rstride % 4 == 0 && bias_hstride % 4 == 0, ALM_ERR_ALIGN);
    ALM_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15u) == 0, ALM_ERR_ALIGN);
  } else {
    ALM_REQUIRE(dbias == nullptr, ALM_ERR_ARG);
  }
  ALM_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && lddo % 8 == 0 && lddq % 8 == 0 && lddk % 8 == 0 &&
                  lddv % 8 == 0 && k_bstride % 8 == 0 && v_bstride % 8 == 0,
              ALM_ERR_ALIGN);
  CUtensorMap tmQ, tmK, tmV, tmdO;
  {
    uint64_t dims[3] = {(uint64_t)h * AB_D, (uint64_t)n_q, (uint64_t)b};
    uint64_t strides[3] = {2, (uint64_t)ldq * 2, (uint64_t)n_q * ldq * 2};
    uint32_t box[3] = {AB_D, AB_T, 1};
    int rc = make_tensor_map(&tmQ, q, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
    strides[1] = (uint64_t)lddo * 2;
    strides[2] = (uint64_t)n_q * lddo * 2;
    rc = make_tensor_map(&tmdO, d_o, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)AB_D, (uint64_t)n_k, (uint64_t)b};
    uint64_t strides[3] = {2, (uint64_t)ldk * 2, (uint64_t)k_bstride * 2};
    uint32_t box[3] = {AB_D, AB_T, 1};
    int rc = make_tensor_map(&tmK, k, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
    strides[1] = (uint64_t)ldv * 2;
    strides[2] = (uint64_t)v_bstride * 2;
    rc = make_tensor_map(&tmV, v, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
  }
  AttnBwdParams p;
  p.lse = lse; p.delta = delta;
  p.kmask = reinterpret_cast<const uint32_t*>(key_mask);
  p.kb_stride = (n_k + 127) / 128 * 4;
  p.dq = (__nv_bfloat16*)dq; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  p.lddq = lddq; p.lddk = lddk; p.lddv = lddv;
  p.bias = bias; p.dbias = dbias; p.bias_hs = bias_hstride; p.bias_rs = bias_rstride;
  p.b = b; p.h = h; p.n_q = n_q; p.n_k = n_k; p.n_q_pad = n_q_pad;
  p.causal = causal;
  p.scale = scale;
  p.scale_log2 = scale * LOG2E;
  static bool attr_set = false;
  if (!attr_set) {
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_dkv_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DKV_SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_dq_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_dkv_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DKV_SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_dq_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, DQ_SMEM));
    attr_set = true;
  }
  dim3 grid_kv(((n_k + AB_T - 1) / AB_T) * b);
  if (bias != nullptr)
    mqa_attn_bwd_dkv_kernel<true><<<grid_kv, AB_THREADS, DKV_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, p);
  else
    mqa_attn_bwd_dkv_kernel<false><<<grid_kv, AB_THREADS, DKV_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, p);
  ALM_CHECK_LAUNCH();
  dim3 grid_q((n_q + AB_T - 1) / AB_T, h, b);
  if (bias != nullptr)
    mqa_attn_bwd_dq_kernel<true><<<grid_q, AB_THREADS, DQ_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, p);
  else
    mqa_attn_bwd_dq_kernel<false><<<grid_q, AB_THREADS, DQ_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(2);
  return ALM_OK;
}
