// Multi-query causal attention backward for sm_90a (autograd of attend.py:69-146), one kernel.
//
// One CTA = (batch, 128 keys).  It walks every (head, query block) that can see these keys and computes, once each,
//     S^T = K Q^T,  dP^T = V dO^T                                      (wgmma, both operands in smem)
//     P^T = exp(S^T*scale - lse),  dS^T = scale * P^T (dP^T - delta)   (on the accumulator fragments)
//     dV += P^T dO   (P^T as register A operand)
//     dK += dS^T Q,  dQ_partial = dS K   (dS^T stored as bf16 in smem, read K-major for dK and MN-major for dQ)
// dV / dK accumulate in registers over all heads (MQA shares k/v: no atomics).  The partial dQ of each tile is
// staged in shared memory and reduce-added into an fp32 workspace [b, n_q, h*64] by TMA
// (cp.reduce.async.bulk.tensor, two boxes per warpgroup and tile); the host zeroes it beforehand (alm_attn_delta) and
// converts it to bf16 dq afterwards.  The elementwise phases (P^T, dS^T) are branch-free: masked, causal and tail
// elements enter the exponential as -inf, so a key mask that differs between the rows of a warp costs no divergence.
//
// Q/K/V/dO tiles arrive by TMA (SWIZZLE_128B); the SAME smem tile serves as a K-major operand
// (contraction over the 64-wide head dim) and as an MN-major operand (contraction over its 128 rows).
// Warps 0-3 / 4-7 are the two consumer warpgroups (key rows [0, 64) / [64, 128) and dQ query rows [0, 64) /
// [64, 128)); each thread needs ~250 registers.  A separate producer warpgroup with a setmaxnreg hand-off does not
// help: ptxas allocates for the 384-thread launch bound (168 registers) and spills ~850 B.  Warp 0 issues the loads
// instead.  Inside a warpgroup S^T and dP^T are separate commit groups, so the exponentials overlap dP^T and dV
// overlaps the dS arithmetic.  The two warpgroups meet once per iteration, on a named barrier, when both halves of
// dS^T are in shared memory; dS^T is double-buffered so that barrier also orders its reuse.  Past that barrier both
// have released the previous iteration's slot, so warp 0 refills it without waiting: STAGES - 1 loads stay ahead.
// The same barrier frees a warpgroup's own key rows of the other dS^T slot (16 KB) until it writes its next dS^T
// there, and that is where its dQ partial is staged: no extra shared memory.
// With DROPOUT (keep mask Z from alm_common.cuh: dropout_keep, regenerated here, never stored):
//     dV += (P^T o Z / (1-p)) dO,   dP^T <- dP^T o Z / (1-p),   dS^T = P^T (dP^T - delta)
// delta = rowsum(dO o O) needs no change because O is the dropped output.  One thread's two key rows by its query
// columns {2c, 2c+1} mod 8 are exactly whole 8-element groups of the generator, so 8 draws per tile cover its 64
// elements; they run while S^T and dP^T are computed.
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
  float* dq_acc;         // [b, n_q, h*64] fp32, zeroed; partial dQ products are reduced into it
  __nv_bfloat16* dk;     // [b, n_k, 64], row stride lddk
  __nv_bfloat16* dv;
  long long lddk, lddv;
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

// keep bits of one (128 keys x 128 queries) tile for this thread: key rows key0, key0 + 8, query columns
// qrow0 + 8 g + c (qrow0 = counter row of column 0 of this thread); bit 4 g + 2 h + c, the index of st / dpt
__device__ __forceinline__ uint64_t attn_bwd_keep_bits(const DropoutArgs& d, uint32_t qrow0, uint32_t key0) {
  uint64_t bits = 0;
#pragma unroll
  for (int cc = 0; cc < AB_T / 16; ++cc) {
    const uint32_t i0 = qrow0 + 16 * cc;
    const uint4 dr = dropout_draw(d, i0, key0);
#pragma unroll
    for (int gh = 0; gh < 2; ++gh)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (dropout_pick(d, dr, i0 + 8 * gh + c, key0 + 8 * h)) bits |= 1ull << (8 * cc + 4 * gh + 2 * h + c);
  }
  return bits;
}

// ================================================================================================
// fused dK / dV / dQ
// ================================================================================================
constexpr int AB_DS_TILE = AB_T * AB_T * 2;   // dS^T tile [128 keys][128 queries] bf16 = 32 KB
constexpr int AB_SMEM = AB_TILE * (2 + 2 * AB_STAGES) + 2 * AB_DS_TILE + AB_STAGES * 2 * 512 + 256;
constexpr uint32_t AB_DS_BAR = 1;             // named barrier of the two consumer warpgroups (0 is __syncthreads)
constexpr uint32_t AB_WG_BAR = 2;             // + cw: named barrier of consumer warpgroup cw alone

// Diagnostic build (-DALM_ATTN_BWD_TRACE, tools/attn_bwd_probe.py): warp 0 of each consumer warpgroup of CTA 0 writes
// clock64() at the phase boundaries of its first AB_TRACE_ITERS iterations; alm_attn_bwd_trace_read copies them out.
constexpr int AB_TRACE_ITERS = 128, AB_TRACE_STAMPS = 8;
#ifdef ALM_ATTN_BWD_TRACE
__device__ long long g_attn_bwd_trace[2][AB_TRACE_ITERS][AB_TRACE_STAMPS];
#define AB_STAMP(i)                                                                                   \
  do {                                                                                                \
    if (blockIdx.x == 0 && (threadIdx.x & 127) == 0 && it < AB_TRACE_ITERS)                           \
      g_attn_bwd_trace[threadIdx.x >> 7][it][i] = clock64();                                          \
  } while (0)
#else
#define AB_STAMP(i)
#endif

template <bool HAS_BIAS, bool DROPOUT>
__global__ void __launch_bounds__(AB_THREADS, 1)
mqa_attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const __grid_constant__ CUtensorMap tmdO,
                    const __grid_constant__ CUtensorMap tmdQ, const AttnBwdParams p, const DropoutArgs drop) {
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0) __trap();
  uint8_t* sK = smem;
  uint8_t* sV = sK + AB_TILE;
  uint8_t* sQ = sV + AB_TILE;                    // [stages]
  uint8_t* sdO = sQ + AB_STAGES * AB_TILE;       // [stages]
  uint8_t* sDS = sdO + AB_STAGES * AB_TILE;      // [2] dS^T, double-buffered across iterations
  float* sLse = reinterpret_cast<float*>(sDS + 2 * AB_DS_TILE);  // [stages][128]
  float* sDelta = sLse + AB_STAGES * AB_T;                       // [stages][128]
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
    tma_prefetch_desc(&tmdQ);
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

  // consumers: warpgroup cw owns key rows [64 cw, 64 cw + 64) of S^T / dP^T / dK / dV and query rows
  // [64 cw, 64 cw + 64) of dQ; fragment rows r_base + 8 h, columns 8 g + c_lane + c
  const int cw = warp >> 2;
  const int wl = warp & 3;
  const int r_base = cw * 64 + wl * 16 + (lane >> 2);
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
  const uint32_t k_all = smem_u32(sK);
  const uint32_t k_addr = k_all + cw * 8192, v_addr = smem_u32(sV) + cw * 8192;
  const bool wg_leader = (threadIdx.x & 127) == 0;   // issues this warpgroup's dQ reduce-adds
  if (n_iter > 0) mbar_wait(kv_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int it = 0; it < n_iter; ++it) {
    const int head = it / q_per_head;
    const int q0 = (qb_min + it % q_per_head) * AB_T;
    [[maybe_unused]] const long long bias_head = HAS_BIAS ? (long long)head * p.bias_hs : 0;
    AB_STAMP(0);
    mbar_wait(&qdo_full[stage], phase);
    AB_STAMP(1);
    const uint32_t q_addr = smem_u32(sQ + stage * AB_TILE), do_addr = smem_u32(sdO + stage * AB_TILE);
    const uint32_t ds_addr = smem_u32(sDS + (it & 1) * AB_DS_TILE);
    // S^T = K Q^T and dP^T = V dO^T as two commit groups: the exponentials run while dP^T is computed
    float st[64], dpt[64];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < AB_D / 16; ++k)
      wgmma_ss<AB_T>(st, wgmma_desc_sw128(k_addr + k * 32, 1024, 16), wgmma_desc_sw128(q_addr + k * 32, 1024, 16),
                     k > 0 ? 1u : 0u);
    wgmma_commit();
#pragma unroll
    for (int k = 0; k < AB_D / 16; ++k)
      wgmma_ss<AB_T>(dpt, wgmma_desc_sw128(v_addr + k * 32, 1024, 16), wgmma_desc_sw128(do_addr + k * 32, 1024, 16),
                     k > 0 ? 1u : 0u);
    wgmma_commit();
    AB_STAMP(2);
    [[maybe_unused]] uint64_t keep = 0;
    if constexpr (DROPOUT)
      keep = attn_bwd_keep_bits(drop, ((uint32_t)batch * p.h + head) * (uint32_t)p.n_q_pad + q0 + c_lane, kj[0]);
    const float* lse_s = sLse + stage * AB_T;
    const float* del_s = sDelta + stage * AB_T;
    // key row kj[h] sees query qi iff key_ok[h] and q_lo[h] <= qi < q_end; a whole tile below the causal diagonal
    // and inside n_q needs no range test.  Every per-element decision below is a select, never a branch: a branch
    // around the exponential diverges wherever the key mask differs between the rows of a warp.
    const bool tile_full = (q0 + AB_T <= p.n_q) && (!p.causal || k0 + AB_T - 1 <= q0 + off);
    const int q_end = tile_full ? INT_MAX : p.n_q;
    int q_lo[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) q_lo[h] = tile_full || !p.causal ? INT_MIN : kj[h] - off;
    auto visible = [&](int h, int qi) { return key_ok[h] & (qi >= q_lo[h]) & (qi < q_end); };
    auto bias_index = [&](int h, int qi) {
      return bias_head + (long long)min(qi, p.n_q - 1) * p.bias_rs + min(kj[h], p.n_k - 1);
    };
    wgmma_wait<1>();
    wgmma_fence_acc(st);
    // P^T = exp(S^T * scale - lse), kept in fp32 for dS; invisible elements get ex2(-inf) = 0
#pragma unroll
    for (int g = 0; g < AB_T / 8; ++g)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = 8 * g + c_lane + c;
        const int qi = q0 + col;
        const float lv = lse_s[col];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int e = 4 * g + 2 * h + c;
          float shift = -lv;
          if constexpr (HAS_BIAS) shift = fmaf(__ldg(p.bias + bias_index(h, qi)), LOG2E, shift);
          const float x = fmaf(st[e], p.scale_log2, shift);
          st[e] = ex2_approx(visible(h, qi) ? x : -INFINITY);
        }
      }
    AB_STAMP(3);
    // dV += P^T dO runs under the dS arithmetic
    uint32_t pa[8][4];
    if constexpr (DROPOUT) {
      float pz[64];
#pragma unroll
      for (int e = 0; e < 64; ++e) pz[e] = ((keep >> e) & 1u) ? st[e] * drop.scale : 0.f;
      pack_a_frags(pz, pa);
    } else {
      pack_a_frags(st, pa);
    }
    wgmma_fence_acc(dv);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_T / 16; ++kk)
      wgmma_rs<AB_D, 1>(dv, pa[kk], wgmma_desc_sw128(do_addr + kk * 2048, 1024, 8192), 1u);
    wgmma_commit();
    wgmma_wait<1>();
    wgmma_fence_acc(dpt);
    // this warpgroup's rows of the dS^T slot staged the previous tile's dQ partial: its reduce must have read them
    if (it > 0) {
      if (wg_leader) bulk_wait_group_read<0>();
      named_bar_sync(AB_WG_BAR + cw, 128);
    }
    // dS^T = scale * P^T (dP^T - delta), stored as bf16 into the 128-B-swizzled dS^T tile: two 16-KB halves of
    // [128 keys][64 queries]; one half is the K-major A operand of dK (contraction over queries) and, read MN-major,
    // the A operand of dQ (contraction over keys)
#pragma unroll
    for (int g = 0; g < AB_T / 8; ++g) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = 8 * g + c_lane + c;
        const int qi = q0 + col;
        const float dl = del_s[col];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int e = 4 * g + 2 * h + c;
          const bool ok = visible(h, qi);
          float ds;
          if constexpr (DROPOUT)
            ds = ok ? st[e] * ((((keep >> e) & 1u) ? dpt[e] * drop.scale : 0.f) - dl) : 0.f;
          else
            ds = ok ? st[e] * (dpt[e] - dl) : 0.f;
          if constexpr (HAS_BIAS) {
            if (ok && p.dbias != nullptr) atomicAdd(p.dbias + bias_index(h, qi), ds);
          }
          dpt[e] = ds * p.scale;
        }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r_base + 8 * h;
        const uint32_t a = ds_addr + (g >> 3) * (AB_DS_TILE / 2) + row * 128 + (((g & 7) ^ (row & 7)) << 4) + 2 * c_lane;
        st_shared_u32(a, pack_bf16x2(dpt[4 * g + 2 * h], dpt[4 * g + 2 * h + 1]));
      }
    }
    AB_STAMP(4);
    fence_proxy_async_smem();
    named_bar_sync(AB_DS_BAR, 2 * 128);  // both halves of dS^T written before either warpgroup reads them for dQ
    AB_STAMP(5);
    // both warpgroups are past iteration it - 1 and have released its slot, so this wait does not block: refill it
    if (warp == 0 && it >= 1 && it - 1 + AB_STAGES < n_iter) {
      const int prev = stage == 0 ? AB_STAGES - 1 : stage - 1;
      mbar_wait(&qdo_empty[prev], stage == 0 ? phase ^ 1u : phase);
      issue_qdo(it - 1 + AB_STAGES);
    }
    // dK += dS^T Q (own 64 keys x all queries) and dQ = dS K (own 64 queries x all keys), both from shared memory
    float dq[32];
    wgmma_fence_acc(dk);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < AB_T / 16; ++kk)
      wgmma_ss<AB_D, 0, 1>(dk, wgmma_desc_sw128(ds_addr + (kk >> 2) * (AB_DS_TILE / 2) + cw * 8192 + (kk & 3) * 32, 1024, 16),
                           wgmma_desc_sw128(q_addr + kk * 2048, 1024, 8192), 1u);
#pragma unroll
    for (int kk = 0; kk < AB_T / 16; ++kk)
      wgmma_ss<AB_D, 1, 1>(dq, wgmma_desc_sw128(ds_addr + cw * (AB_DS_TILE / 2) + kk * 2048, 1024, 8192),
                           wgmma_desc_sw128(k_all + kk * 2048, 1024, 8192), kk > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(dv);
    wgmma_fence_acc(dk);
    wgmma_fence_acc(dq);
    AB_STAMP(6);
    if (lane == 0) mbar_arrive(&qdo_empty[stage]);
    // partial dQ -> fp32 workspace: staged in this warpgroup's own key rows of the OTHER dS^T slot (16 KB: rows
    // [64 cw, 64 cw + 64) of both query halves), which nobody reads until this warpgroup rewrites them with dS^T of
    // the next tile (the other warpgroup finished its dQ of tile it - 1 before the barrier above).  Each 8-KB half
    // is a [64 queries][32 fp32] 128-B-swizzled box; one thread reduce-adds both into dq_acc by TMA, which clips
    // the n_q tail.
    const uint32_t stg = smem_u32(sDS + ((it + 1) & 1) * AB_DS_TILE) + cw * 8192;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = wl * 16 + (lane >> 2) + 8 * h;
#pragma unroll
      for (int g = 0; g < AB_D / 8; ++g) {
        const int byte = 32 * (g & 3) + 4 * c_lane;
        st_shared_f32x2(stg + (g >> 2) * (AB_DS_TILE / 2) + row * 128 + ((((byte >> 4) ^ (row & 7)) << 4) | (byte & 15)),
                        dq[4 * g + 2 * h], dq[4 * g + 2 * h + 1]);
      }
    }
    fence_proxy_async_smem();
    named_bar_sync(AB_WG_BAR + cw, 128);
    if (wg_leader) {
      tma_reduce_add_3d(&tmdQ, stg, head * AB_D, q0 + cw * 64, batch);
      tma_reduce_add_3d(&tmdQ, stg + AB_DS_TILE / 2, head * AB_D + 32, q0 + cw * 64, batch);
      bulk_commit_group();
    }
    AB_STAMP(7);
    if (++stage == AB_STAGES) { stage = 0; phase ^= 1u; }
  }
  if (wg_leader) bulk_wait_group<0>();
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

// dq [b, n_q, h*64] bf16 (row stride lddq) <- the fp32 workspace [b, n_q, h*64] (contiguous); 4 columns per thread
__global__ void attn_dq_convert_kernel(const float4* __restrict__ acc, __nv_bfloat16* __restrict__ dq, long long lddq,
                                       long long rows, int cols4) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols4) return;
  const long long r = i / cols4;
  const int c = (int)(i - r * cols4);
  const float4 v = acc[i];
  *reinterpret_cast<uint2*>(dq + r * lddq + 4 * c) = make_uint2(pack_bf16x2(v.x, v.y), pack_bf16x2(v.z, v.w));
}

}  // namespace alm

extern "C" int alm_mqa_attn_bwd(const void* q, int64_t ldq, const void* k, int64_t ldk, int64_t k_bstride,
                                const void* v, int64_t ldv, int64_t v_bstride, const void* d_o, int64_t lddo,
                                const void* key_mask, const float* lse, const float* delta, int n_q_pad, void* dq,
                                int64_t lddq, float* dq_acc, void* dk, int64_t lddk, void* dv, int64_t lddv, const float* bias,
                                float* dbias, int64_t bias_hstride, int64_t bias_rstride, int b, int h, int n_q,
                                int n_k, int causal, float scale, float dropout_p, uint64_t seed, uint32_t site,
                                alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(q && k && v && d_o && lse && delta && dq && dq_acc && dk && dv, ALM_ERR_ARG);
  ALM_REQUIRE(b > 0 && h > 0 && n_q > 0 && n_k >= n_q, ALM_ERR_ARG);
  ALM_REQUIRE(n_q_pad % AB_T == 0 && n_q_pad >= n_q, ALM_ERR_ARG);
  ALM_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, ALM_ERR_ARG);
  // the dropout counter rows are (b*h + head) * (n_q rounded up to 128) + i, as in the forward
  ALM_REQUIRE(dropout_p == 0.f || n_q_pad == (n_q + AB_T - 1) / AB_T * AB_T, ALM_ERR_ARG);
  ALM_REQUIRE((long long)b * h * n_q_pad < (1ll << 32), ALM_ERR_UNSUPPORTED);
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
  CUtensorMap tmdQ;  // fp32 dq_acc [b, n_q, h*64] in [64 queries][32 columns] boxes (128-B rows, swizzled)
  {
    uint64_t dims[3] = {(uint64_t)h * AB_D, (uint64_t)n_q, (uint64_t)b};
    uint64_t strides[3] = {4, (uint64_t)h * AB_D * 4, (uint64_t)n_q * h * AB_D * 4};
    uint32_t box[3] = {32, 64, 1};
    int rc = make_tensor_map(&tmdQ, dq_acc, 4, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
  }
  AttnBwdParams p;
  p.lse = lse; p.delta = delta;
  p.kmask = reinterpret_cast<const uint32_t*>(key_mask);
  p.kb_stride = (n_k + 127) / 128 * 4;
  p.dq_acc = dq_acc; p.dk = (__nv_bfloat16*)dk; p.dv = (__nv_bfloat16*)dv;
  p.lddk = lddk; p.lddv = lddv;
  p.bias = bias; p.dbias = dbias; p.bias_hs = bias_hstride; p.bias_rs = bias_rstride;
  p.b = b; p.h = h; p.n_q = n_q; p.n_k = n_k; p.n_q_pad = n_q_pad;
  p.causal = causal;
  p.scale = scale;
  p.scale_log2 = scale * LOG2E;
  // counter rows (b*h + head) * n_q_pad + i, columns = key index
  const DropoutArgs dargs = make_dropout_args(dropout_p, seed, site);
  static bool attr_set = false;
  if (!attr_set) {
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_bwd_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, AB_SMEM));
    attr_set = true;
  }
  dim3 grid(((n_k + AB_T - 1) / AB_T) * b);
  const bool drop = dropout_p > 0.f;
  if (bias != nullptr && drop)
    mqa_attn_bwd_kernel<true, true><<<grid, AB_THREADS, AB_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, tmdQ, p, dargs);
  else if (bias != nullptr)
    mqa_attn_bwd_kernel<true, false><<<grid, AB_THREADS, AB_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, tmdQ, p, dargs);
  else if (drop)
    mqa_attn_bwd_kernel<false, true><<<grid, AB_THREADS, AB_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, tmdQ, p, dargs);
  else
    mqa_attn_bwd_kernel<false, false><<<grid, AB_THREADS, AB_SMEM, stream>>>(tmQ, tmK, tmV, tmdO, tmdQ, p, dargs);
  ALM_CHECK_LAUNCH();
  const long long rows = (long long)b * n_q;
  const int cols4 = h * AB_D / 4;
  attn_dq_convert_kernel<<<(unsigned)ceil_div(rows * cols4, 256LL), 256, 0, stream>>>(
      reinterpret_cast<const float4*>(dq_acc), (__nv_bfloat16*)dq, lddq, rows, cols4);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(2);
  return ALM_OK;
}

#ifdef ALM_ATTN_BWD_TRACE
// [2 warpgroups][AB_TRACE_ITERS][AB_TRACE_STAMPS] clock64 stamps of the last launch's CTA 0 -> host (synchronous)
extern "C" int alm_attn_bwd_trace_read(long long* dst) {
  ALM_CUDA_OK(cudaMemcpyFromSymbol(dst, alm::g_attn_bwd_trace, sizeof(alm::g_attn_bwd_trace)));
  return ALM_OK;
}
#endif
