// Multi-query causal attention forward for sm_90a (replaces attend.py:69-146 as called from
// audiolm_pytorch.py:390): softmax(q k^T * d^-1/2, masked by key-padding mask and right-aligned causal
// mask) v, with ONE shared k/v head of width D = 32, 64 or 128 (a template parameter) for all query heads.
//
// One CTA = (batch b, head h, 128 queries).  Q/K/V tiles arrive by TMA into swizzled smem (SwizzledTile<D>: one
// 128-B-swizzled [128 x 64] tile at D = 64, two of them side by side at D = 128, one 64-B-swizzled [128 x 32] tile at
// D = 32); each of the two
// consumer warpgroups owns 64 query rows: S = Q K^T is a wgmma with both operands in smem, the online (flash)
// softmax runs on the S accumulator fragment in registers, and P V is a wgmma whose A operand (P, bf16) is taken
// straight from those registers, accumulating O in registers.
//   warpgroup 0 : TMA producer (warp 0)      warpgroups 1, 2 : softmax + MMA, query rows [0, 64) / [64, 128)
// An optional additive score bias [h, n_q, n_k] (flash_attn=False path, attend.py:122-124) is added to the scores;
// tiles that lie fully below the causal diagonal take a predicate-free path.
// With DROPOUT, P is multiplied by the keep mask (alm_common.cuh: dropout_keep) times 1/(1-p) when it is packed into
// the A operand of P V; the row max, the row sum and the stored LSE use the un-dropped P.
// D = 128 holds 64 O accumulators beside the 64 scores of a tile, more than the 168 registers a 384-thread CTA gives
// every thread: there the producer warpgroup hands registers to the consumers (setmaxnreg 40 / 232), and the K/V ring
// has 3 stages instead of 4 (Q + 3 x (K + V) = 224 KB).
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {

constexpr int ATT_BM = 128;     // queries per CTA
constexpr int ATT_BN = 128;     // keys per tile
constexpr int ATT_THREADS = 384;
template <int D>                // D = head width (dim_head)
struct AttFwdCfg {
  static constexpr int KV_STAGES = D == 128 ? 3 : 4;
  static constexpr int HALF_BYTES = 128 * SwizzledTile<D>::ROW_BYTES;  // one swizzled [128 x min(D, 64)] half
  static constexpr int TILE_BYTES = 128 * D * 2;                       // 16 KB at D = 64
  static constexpr int SMEM_BYTES = TILE_BYTES * (1 + 2 * KV_STAGES) + 256;
};

struct AttnFwdParams {
  __nv_bfloat16* o;       // [b, n_q, h*D] row stride ldo
  float* lse;             // [b, h, lse_stride] log2-domain LSE of the scaled scores (for backward); may be null
  const uint32_t* kmask;  // packed key mask (alm_pack_key_mask): bit i of word w of row b = key 32 w + i may be attended; may be null
  int kb_stride;          // words per batch row: 4 * ceil(n_k / 128)
  const float* bias;      // [h, n_q, bias_rs] additive score bias (natural-log domain, added after the scale); may be null
  long long bias_hs, bias_rs;  // element strides between heads / query rows (bias_rs % 4 == 0, >= n_k)
  long long ldo, lse_stride;
  int b, h, n_q, n_k;
  int causal;
  float scale_log2;       // d^-1/2 * log2(e)
  int n_q_pad;            // n_q rounded up to 128: query rows of the dropout counter are (b*h + head) * n_q_pad + i
  uint32_t drop_row0;     // dropout counter row of this launch's batch 0 (the host launches batch chunks, see below)
  DropoutArgs drop;
};

__device__ __forceinline__ float att_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Dropout keep bits of one 128-key tile for this thread's fragment: rows qrow, qrow + 8 (counter rows), columns
// kbase + 8 g + c_lane + c; bit 4 g + 2 h + c. The lane pair (lane, lane ^ 4) holds rows (qrow, qrow ^ 1): for each
// 16-key step each of the two draws the group of its own c and hands the partner the words of the partner's rows.
__device__ __forceinline__ uint64_t attn_fwd_keep_bits(const DropoutArgs& d, uint32_t qrow, uint32_t kbase, int c_lane) {
  const uint32_t odd = qrow & 1u;
  uint64_t bits = 0;
#pragma unroll
  for (int kk = 0; kk < ATT_BN / 16; ++kk) {
    const uint32_t j0 = kbase + 16 * kk + c_lane;
    const uint4 own = dropout_draw(d, qrow, j0 + odd);
    const uint32_t ra = __shfl_xor_sync(0xffffffffu, odd ? own.x : own.y, 4);
    const uint32_t rb = __shfl_xor_sync(0xffffffffu, odd ? own.z : own.w, 4);
    const uint4 other = odd ? make_uint4(0u, ra, 0u, rb) : make_uint4(ra, 0u, rb, 0u);
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const uint4 dr = (uint32_t)c == odd ? own : other;
#pragma unroll
      for (int half = 0; half < 2; ++half)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (dropout_pick(d, dr, qrow + 8 * h, j0 + 8 * half + c)) bits |= 1ull << (8 * kk + 4 * half + 2 * h + c);
    }
  }
  return bits;
}

template <int ATT_D, bool HAS_BIAS, bool DROPOUT>
__global__ void __launch_bounds__(ATT_THREADS, 1)
mqa_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
  using Tile = SwizzledTile<ATT_D>;
  using Cfg = AttFwdCfg<ATT_D>;
  constexpr int ATT_KV_STAGES = Cfg::KV_STAGES, ATT_TILE_BYTES = Cfg::TILE_BYTES, HALF = Cfg::HALF_BYTES;
  constexpr bool REG_HANDOFF = ATT_D == 128;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw;
  if ((smem_u32(smem) & 1023u) != 0) __trap();  // SW128 tiles need 1024-B alignment
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + ATT_TILE_BYTES;                   // [stages]
  uint8_t* sV = sK + ATT_KV_STAGES * ATT_TILE_BYTES;   // [stages]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + ATT_KV_STAGES * ATT_TILE_BYTES);
  uint64_t* q_full = bars;
  uint64_t* kv_full = bars + 1;                        // [stages]
  uint64_t* kv_empty = kv_full + ATT_KV_STAGES;        // [stages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int n_qblocks = (p.n_q + ATT_BM - 1) / ATT_BM;
  const int qb = n_qblocks - 1 - (int)blockIdx.x;  // heavy (late) query blocks first
  const int head = blockIdx.y;
  const int batch = blockIdx.z;
  const int q0 = qb * ATT_BM;
  const int off = p.n_k - p.n_q;  // right alignment of queries against keys (KV cache)
  int kv_end = p.n_k;
  if (p.causal) kv_end = min(p.n_k, q0 + ATT_BM + off);
  const int n_tiles = kv_end > 0 ? (kv_end + ATT_BN - 1) / ATT_BN : 0;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    for (int i = 0; i < ATT_KV_STAGES; ++i) {
      mbar_init(&kv_full[i], 1);
      mbar_init(&kv_empty[i], 8);  // one arrive per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (wg == 0) {
    if constexpr (REG_HANDOFF) setmaxnreg_dec<40>();
    if (warp == 0 && n_tiles > 0) {
      // ---------------- TMA producer (whole warp runs the loop, one elected lane issues) -------
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(q_full, ATT_TILE_BYTES);
#pragma unroll
        for (int hf = 0; hf < Tile::HALVES; ++hf)
          tma_load_3d(sQ + hf * HALF, &tmQ, q_full, head * ATT_D + hf * Tile::HW, q0, batch);
      }
      __syncwarp();
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_tiles; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1u);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&kv_full[stage], 2 * ATT_TILE_BYTES);
#pragma unroll
          for (int hf = 0; hf < Tile::HALVES; ++hf) {
            tma_load_3d(sK + stage * ATT_TILE_BYTES + hf * HALF, &tmK, &kv_full[stage], hf * Tile::HW, j * ATT_BN, batch);
            tma_load_3d(sV + stage * ATT_TILE_BYTES + hf * HALF, &tmV, &kv_full[stage], hf * Tile::HW, j * ATT_BN, batch);
          }
        }
        __syncwarp();
        if (++stage == ATT_KV_STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ---------------- consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64) ----------------
  // fragment: this thread holds rows r_base + 8 h (h = 0, 1) and, of every 8-column group j, columns 8 j + c_lane + {0, 1}
  if constexpr (REG_HANDOFF) setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int r_base = cw * 64 + (warp & 3) * 16 + (lane >> 2);
  const int c_lane = 2 * (lane & 3);
  constexpr float kLog2e = 1.4426950408889634f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  float o_acc[ATT_D / 2];
#pragma unroll
  for (int d = 0; d < ATT_D / 2; ++d) o_acc[d] = 0.f;
  int q_limit[2];
  [[maybe_unused]] const float* brow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int qi = q0 + r_base + 8 * h;
    q_limit[h] = min(p.causal ? qi + off : p.n_k - 1, p.n_k - 1);  // last key index this query may see
    // bias row (rows past n_q are clamped: their output is dropped)
    if constexpr (HAS_BIAS) brow[h] = p.bias + (long long)head * p.bias_hs + (long long)min(qi, p.n_q - 1) * p.bias_rs;
  }
  const uint32_t* mrow = p.kmask ? p.kmask + (long long)batch * p.kb_stride : nullptr;
  const uint32_t q_addr = smem_u32(sQ) + cw * 64 * Tile::ROW_BYTES;
  [[maybe_unused]] const uint32_t drop_row =
      p.drop_row0 + ((uint32_t)batch * p.h + head) * (uint32_t)p.n_q_pad + q0 + r_base;

  if (n_tiles > 0) mbar_wait(q_full, 0);
  int stage = 0;
  uint32_t phase = 0;
  for (int j = 0; j < n_tiles; ++j) {
    mbar_wait(&kv_full[stage], phase);
    const uint32_t k_addr = smem_u32(sK + stage * ATT_TILE_BYTES);
    const uint32_t v_addr = smem_u32(sV + stage * ATT_TILE_BYTES);
    float s[ATT_BN / 2];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < ATT_D / 16; ++k)
      wgmma_ss<ATT_BN>(s, Tile::kmajor(q_addr, k, HALF), Tile::kmajor(k_addr, k, HALF), k > 0 ? 1u : 0u);
    wgmma_commit();
    [[maybe_unused]] uint64_t keep = 0;  // drawn while S = Q K^T runs
    if constexpr (DROPOUT) keep = attn_fwd_keep_bits(p.drop, drop_row, j * ATT_BN, c_lane);
    wgmma_wait<0>();
    wgmma_fence_acc(s);

    const int kbase = j * ATT_BN;
    // CTA-uniform: every row of the block sees every key of this tile (no key mask, fully below the diagonal)
    const bool tile_full = mrow == nullptr && kbase + ATT_BN <= p.n_k && (!p.causal || kbase + ATT_BN - 1 <= q0 + off);
    uint32_t valid[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};  // key bits of the tile (mask only)
    if (!tile_full && mrow != nullptr) {
      const uint4 mv = __ldg(reinterpret_cast<const uint4*>(mrow + j * 4));
      valid[0] = mv.x; valid[1] = mv.y; valid[2] = mv.z; valid[3] = mv.w;
    }
    uint32_t pa[ATT_BN / 16][4];  // P as bf16 A fragments, one per 16-key k step
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      // scores -> log2 domain (scale, bias), invalid entries -> -inf
#pragma unroll
      for (int g = 0; g < ATT_BN / 8; ++g)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int col = 8 * g + c_lane + c;
          float v = s[4 * g + 2 * h + c] * p.scale_log2;
          if constexpr (HAS_BIAS) {
            if (kbase + col < p.bias_rs) v = fmaf(__ldg(brow[h] + kbase + col), kLog2e, v);
          }
          if (!tile_full) {
            const bool ok = kbase + col <= q_limit[h] && ((valid[col >> 5] >> (col & 31)) & 1u);
            if (!ok) v = -INFINITY;
          }
          s[4 * g + 2 * h + c] = v;
        }
      float m_tile = -INFINITY;
#pragma unroll
      for (int g = 0; g < ATT_BN / 8; ++g) m_tile = fmaxf(m_tile, fmaxf(s[4 * g + 2 * h], s[4 * g + 2 * h + 1]));
      m_tile = fmaxf(m_tile, __shfl_xor_sync(0xffffffffu, m_tile, 1));
      m_tile = fmaxf(m_tile, __shfl_xor_sync(0xffffffffu, m_tile, 2));
      const float m_new = fmaxf(m_run[h], m_tile);
      const float m_use = (m_new == -INFINITY) ? 0.f : m_new;
      const float alpha = att_ex2(m_run[h] - m_use);  // m_run == -inf -> 0
      float l_tile = 0.f;
#pragma unroll
      for (int g = 0; g < ATT_BN / 8; ++g)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const float pv = att_ex2(s[4 * g + 2 * h + c] - m_use);  // -inf -> 0
          s[4 * g + 2 * h + c] = pv;
          l_tile += pv;
        }
      l_run[h] = fmaf(l_run[h], alpha, l_tile);  // partial over this thread's columns; the quad is summed at the end
      m_run[h] = m_new;
#pragma unroll
      for (int g = 0; g < ATT_D / 8; ++g) {
        o_acc[4 * g + 2 * h] *= alpha;
        o_acc[4 * g + 2 * h + 1] *= alpha;
      }
    }
    if constexpr (DROPOUT) {
#pragma unroll
      for (int e = 0; e < ATT_BN / 2; ++e) s[e] = ((keep >> e) & 1u) ? s[e] * p.drop.scale : 0.f;
    }
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {
      pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
    // O += P V (V is the MN-major B operand: [keys][D dims])
    wgmma_fence_acc(o_acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      wgmma_rs<ATT_D, 1>(o_acc, pa[kk], Tile::mnmajor(v_addr, kk, HALF), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(o_acc);
    if (lane == 0) mbar_arrive(&kv_empty[stage]);
    if (++stage == ATT_KV_STAGES) { stage = 0; phase ^= 1u; }
  }

#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l_tot = l_run[h];
    l_tot += __shfl_xor_sync(0xffffffffu, l_tot, 1);
    l_tot += __shfl_xor_sync(0xffffffffu, l_tot, 2);
    const int qi = q0 + r_base + 8 * h;
    if (qi < p.n_q) {
      const float inv = l_tot > 0.f ? 1.f / l_tot : 0.f;
      __nv_bfloat16* dst = p.o + ((long long)batch * p.n_q + qi) * p.ldo + head * ATT_D + c_lane;
#pragma unroll
      for (int g = 0; g < ATT_D / 8; ++g)
        *reinterpret_cast<uint32_t*>(dst + 8 * g) = pack_bf16x2(o_acc[4 * g + 2 * h] * inv, o_acc[4 * g + 2 * h + 1] * inv);
      if (p.lse != nullptr && (lane & 3) == 0) {
        const float lse = l_tot > 0.f ? (m_run[h] + log2f(l_tot)) : INFINITY;  // log2 domain (x ln2 = natural)
        p.lse[((long long)batch * p.h + head) * p.lse_stride + qi] = lse;
      }
    }
  }
}

}  // namespace alm

namespace alm {
// key mask bytes [b, n_k] (non-zero = attend) -> bits [b, 4 * ceil(n_k / 128)] (keys past n_k: 0); one warp per word
// of the flattened [b * words] output on a 1-D grid, so the batch is not bound by the 65535 limit of grid.y
__global__ void pack_key_mask_kernel(const uint8_t* __restrict__ mask, uint32_t* __restrict__ bits, int n_k, int words,
                                     long long total) {
  const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= total) return;
  const long long b = i / words;
  const int k = (int)(i - b * words) * 32 + (threadIdx.x & 31);
  const bool on = k < n_k && mask[b * n_k + k] != 0;
  const uint32_t v = __ballot_sync(0xffffffffu, on);
  if ((threadIdx.x & 31) == 0) bits[i] = v;
}
}  // namespace alm

extern "C" int alm_pack_key_mask(const void* key_mask, void* bits, int b, int n_k, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(key_mask && bits && b > 0 && n_k > 0, ALM_ERR_ARG);
  const int words = (n_k + 127) / 128 * 4;
  const long long total = (long long)b * words;
  const long long blocks = ceil_div(total, 8LL);
  ALM_REQUIRE(blocks <= INT_MAX, ALM_ERR_UNSUPPORTED);
  pack_key_mask_kernel<<<(unsigned)blocks, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(key_mask),
                                                            reinterpret_cast<uint32_t*>(bits), n_k, words, total);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

namespace alm {
// the four instantiations of one head width: attribute set-up once, then the launch over batch chunks
template <int D>
static int attn_fwd_launch(const void* q, int64_t ldq, const void* k, int64_t ldk, int64_t k_bstride, const void* v,
                           int64_t ldv, int64_t v_bstride, const void* key_mask, void* o, int64_t ldo, float* lse,
                           const float* bias, int b, bool drop, AttnFwdParams p, cudaStream_t stream) {
  using Tile = SwizzledTile<D>;
  constexpr int SMEM = AttFwdCfg<D>::SMEM_BYTES;
  const int h = p.h, n_q = p.n_q, n_k = p.n_k;
  static bool attr_set = false;
  if (!attr_set) {
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_fwd_kernel<D, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_fwd_kernel<D, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_fwd_kernel<D, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_fwd_kernel<D, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_set = true;
  }
  // Batch is grid.z, which stops at 65535, so larger batches (the local attention passes batch x heads x windows)
  // run as consecutive launches over chunks of batch rows: operands, outputs and the key mask are offset here, the
  // dropout counter rows by p.drop_row0.  The (qblock, head, batch) order of each launch is unchanged.
  constexpr int kMaxGridZ = 65535;
  const int n_launch = ceil_div(b, kMaxGridZ);
  for (int b0 = 0; b0 < b; b0 += kMaxGridZ) {
    const int nb = min(b - b0, kMaxGridZ);
    CUtensorMap tmQ, tmK, tmV;
    {
      uint64_t dims[3] = {(uint64_t)h * D, (uint64_t)n_q, (uint64_t)nb};
      uint64_t strides[3] = {2, (uint64_t)ldq * 2, (uint64_t)n_q * ldq * 2};
      uint32_t box[3] = {Tile::HW, ATT_BM, 1};
      int rc = make_tensor_map(&tmQ, reinterpret_cast<const __nv_bfloat16*>(q) + (long long)b0 * n_q * ldq, 2, 3, dims,
                               strides, box, Tile::SWIZZLE);
      if (rc != ALM_OK) return rc;
    }
    {
      uint64_t dims[3] = {(uint64_t)D, (uint64_t)n_k, (uint64_t)nb};
      uint64_t strides[3] = {2, (uint64_t)ldk * 2, (uint64_t)k_bstride * 2};
      uint32_t box[3] = {Tile::HW, ATT_BN, 1};
      int rc = make_tensor_map(&tmK, reinterpret_cast<const __nv_bfloat16*>(k) + (long long)b0 * k_bstride, 2, 3, dims,
                               strides, box, Tile::SWIZZLE);
      if (rc != ALM_OK) return rc;
      strides[1] = (uint64_t)ldv * 2;
      strides[2] = (uint64_t)v_bstride * 2;
      rc = make_tensor_map(&tmV, reinterpret_cast<const __nv_bfloat16*>(v) + (long long)b0 * v_bstride, 2, 3, dims,
                           strides, box, Tile::SWIZZLE);
      if (rc != ALM_OK) return rc;
    }
    p.o = reinterpret_cast<__nv_bfloat16*>(o) + (long long)b0 * n_q * ldo;
    p.lse = lse != nullptr ? lse + (long long)b0 * h * p.lse_stride : nullptr;
    p.kmask = key_mask != nullptr ? reinterpret_cast<const uint32_t*>(key_mask) + (long long)b0 * p.kb_stride : nullptr;
    p.b = nb;
    p.drop_row0 = (uint32_t)((long long)b0 * h * p.n_q_pad);
    const dim3 grid((n_q + ATT_BM - 1) / ATT_BM, h, nb);
    if (bias != nullptr && drop)
      mqa_attn_fwd_kernel<D, true, true><<<grid, ATT_THREADS, SMEM, stream>>>(tmQ, tmK, tmV, p);
    else if (bias != nullptr)
      mqa_attn_fwd_kernel<D, true, false><<<grid, ATT_THREADS, SMEM, stream>>>(tmQ, tmK, tmV, p);
    else if (drop)
      mqa_attn_fwd_kernel<D, false, true><<<grid, ATT_THREADS, SMEM, stream>>>(tmQ, tmK, tmV, p);
    else
      mqa_attn_fwd_kernel<D, false, false><<<grid, ATT_THREADS, SMEM, stream>>>(tmQ, tmK, tmV, p);
    ALM_CHECK_LAUNCH();
  }
  ALM_LAUNCHED(n_launch);
  return ALM_OK;
}
}  // namespace alm

extern "C" int alm_mqa_attn_fwd_dh(const void* q, int64_t ldq, const void* k, int64_t ldk, int64_t k_bstride,
                                   const void* v, int64_t ldv, int64_t v_bstride, const void* key_mask, void* o,
                                   int64_t ldo, float* lse, int64_t lse_stride, const float* bias,
                                   int64_t bias_hstride, int64_t bias_rstride, int b, int h, int n_q, int n_k,
                                   int causal, float scale, float dropout_p, uint64_t seed, uint32_t site,
                                   int dim_head, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(dim_head == 32 || dim_head == 64 || dim_head == 128, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(q && k && v && o, ALM_ERR_ARG);
  ALM_REQUIRE(b > 0 && h > 0 && n_q > 0 && n_k > 0 && n_k >= n_q, ALM_ERR_ARG);
  ALM_REQUIRE(dropout_p >= 0.f && dropout_p < 1.f, ALM_ERR_ARG);
  ALM_REQUIRE((long long)b * h * ((n_q + 127) / 128 * 128) < (1ll << 32), ALM_ERR_UNSUPPORTED);  // 32-bit counter rows
  ALM_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, ALM_ERR_ALIGN);
  ALM_REQUIRE(k_bstride % 8 == 0 && v_bstride % 8 == 0, ALM_ERR_ALIGN);
  ALM_REQUIRE((reinterpret_cast<uintptr_t>(o) & 15u) == 0, ALM_ERR_ALIGN);
  if (bias != nullptr) {
    ALM_REQUIRE(bias_rstride >= n_k && bias_rstride % 4 == 0 && bias_hstride % 4 == 0, ALM_ERR_ALIGN);
    ALM_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15u) == 0, ALM_ERR_ALIGN);
  }

  AttnFwdParams p;
  p.kb_stride = (n_k + 127) / 128 * 4;
  p.bias = bias;
  p.bias_hs = bias_hstride;
  p.bias_rs = bias_rstride;
  p.ldo = ldo;
  p.lse_stride = lse_stride;
  p.h = h; p.n_q = n_q; p.n_k = n_k;
  p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  p.n_q_pad = (n_q + 127) / 128 * 128;
  p.drop = make_dropout_args(dropout_p, seed, site);
  const bool drop = dropout_p > 0.f;
#define ALM_ATT_FWD(DD) \
  attn_fwd_launch<DD>(q, ldq, k, ldk, k_bstride, v, ldv, v_bstride, key_mask, o, ldo, lse, bias, b, drop, p, stream)
  if (dim_head == 32) return ALM_ATT_FWD(32);
  if (dim_head == 64) return ALM_ATT_FWD(64);
  return ALM_ATT_FWD(128);
#undef ALM_ATT_FWD
}

extern "C" int alm_mqa_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, int64_t k_bstride,
                                const void* v, int64_t ldv, int64_t v_bstride, const void* key_mask, void* o,
                                int64_t ldo, float* lse, int64_t lse_stride, const float* bias, int64_t bias_hstride,
                                int64_t bias_rstride, int b, int h, int n_q, int n_k, int causal, float scale,
                                float dropout_p, uint64_t seed, uint32_t site, alm_stream_t stream_) {
  return alm_mqa_attn_fwd_dh(q, ldq, k, ldk, k_bstride, v, ldv, v_bstride, key_mask, o, ldo, lse, lse_stride, bias,
                             bias_hstride, bias_rstride, b, h, n_q, n_k, causal, scale, dropout_p, seed, site, 64,
                             stream_);
}
