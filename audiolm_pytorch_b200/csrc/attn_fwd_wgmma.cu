// Multi-query causal attention forward for sm_90a (replaces attend.py:69-146 as called from
// audiolm_pytorch.py:390): softmax(q k^T * d^-1/2, masked by key-padding mask and right-aligned causal
// mask) v, with ONE shared k/v head of width 64 for all query heads.
//
// One CTA = (batch b, head h, 128 queries).  Q/K/V tiles arrive by TMA into 128-B-swizzled smem; each of the two
// consumer warpgroups owns 64 query rows: S = Q K^T is a wgmma with both operands in smem, the online (flash)
// softmax runs on the S accumulator fragment in registers, and P V is a wgmma whose A operand (P, bf16) is taken
// straight from those registers, accumulating O in registers.
//   warpgroup 0 : TMA producer (warp 0)      warpgroups 1, 2 : softmax + MMA, query rows [0, 64) / [64, 128)
// An optional additive score bias [h, n_q, n_k] (flash_attn=False path, attend.py:122-124) is added to the scores;
// tiles that lie fully below the causal diagonal take a predicate-free path.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {

constexpr int ATT_BM = 128;     // queries per CTA
constexpr int ATT_BN = 128;     // keys per tile
constexpr int ATT_D = 64;       // head width (dim_head)
constexpr int ATT_KV_STAGES = 4;
constexpr int ATT_THREADS = 384;
constexpr int ATT_TILE_BYTES = 128 * 64 * 2;  // 16 KB: one [128 x 64] bf16 SW128 tile
constexpr int ATT_SMEM_BYTES = ATT_TILE_BYTES * (1 + 2 * ATT_KV_STAGES) + 256;

struct AttnFwdParams {
  __nv_bfloat16* o;       // [b, n_q, h*64] row stride ldo
  float* lse;             // [b, h, lse_stride] log2-domain LSE of the scaled scores (for backward); may be null
  const uint32_t* kmask;  // packed key mask (alm_pack_key_mask): bit i of word w of row b = key 32 w + i may be attended; may be null
  int kb_stride;          // words per batch row: 4 * ceil(n_k / 128)
  const float* bias;      // [h, n_q, bias_rs] additive score bias (natural-log domain, added after the scale); may be null
  long long bias_hs, bias_rs;  // element strides between heads / query rows (bias_rs % 4 == 0, >= n_k)
  long long ldo, lse_stride;
  int b, h, n_q, n_k;
  int causal;
  float scale_log2;       // d^-1/2 * log2(e)
};

__device__ __forceinline__ float att_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <bool HAS_BIAS>
__global__ void __launch_bounds__(ATT_THREADS, 1)
mqa_attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                    const __grid_constant__ CUtensorMap tmV, const AttnFwdParams p) {
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
    if (warp == 0 && n_tiles > 0) {
      // ---------------- TMA producer (whole warp runs the loop, one elected lane issues) -------
      if (elect_one_sync()) {
        mbar_arrive_expect_tx(q_full, ATT_TILE_BYTES);
        tma_load_3d(sQ, &tmQ, q_full, head * ATT_D, q0, batch);
      }
      __syncwarp();
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_tiles; ++j) {
        mbar_wait(&kv_empty[stage], phase ^ 1u);
        if (elect_one_sync()) {
          mbar_arrive_expect_tx(&kv_full[stage], 2 * ATT_TILE_BYTES);
          tma_load_3d(sK + stage * ATT_TILE_BYTES, &tmK, &kv_full[stage], 0, j * ATT_BN, batch);
          tma_load_3d(sV + stage * ATT_TILE_BYTES, &tmV, &kv_full[stage], 0, j * ATT_BN, batch);
        }
        __syncwarp();
        if (++stage == ATT_KV_STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ---------------- consumers: warpgroup cw owns query rows [64 cw, 64 cw + 64) ----------------
  // fragment: this thread holds rows r_base + 8 h (h = 0, 1) and, of every 8-column group j, columns 8 j + c_lane + {0, 1}
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
  const uint32_t q_addr = smem_u32(sQ) + cw * 8192;

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
      wgmma_ss<ATT_BN>(s, wgmma_desc_sw128(q_addr + k * 32, 1024, 16), wgmma_desc_sw128(k_addr + k * 32, 1024, 16),
                       k > 0 ? 1u : 0u);
    wgmma_commit();
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
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk) {
      pa[kk][0] = pack_bf16x2(s[8 * kk + 0], s[8 * kk + 1]);
      pa[kk][1] = pack_bf16x2(s[8 * kk + 2], s[8 * kk + 3]);
      pa[kk][2] = pack_bf16x2(s[8 * kk + 4], s[8 * kk + 5]);
      pa[kk][3] = pack_bf16x2(s[8 * kk + 6], s[8 * kk + 7]);
    }
    // O += P V (V is the MN-major B operand: [keys][64 dims])
    wgmma_fence_acc(o_acc);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < ATT_BN / 16; ++kk)
      wgmma_rs<ATT_D, 1>(o_acc, pa[kk], wgmma_desc_sw128(v_addr + kk * 2048, 1024, 8192), 1u);
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
// key mask bytes [b, n_k] (non-zero = attend) -> bits [b, 4 * ceil(n_k / 128)] (keys past n_k: 0)
__global__ void pack_key_mask_kernel(const uint8_t* __restrict__ mask, uint32_t* __restrict__ bits, int n_k, int words) {
  const int b = blockIdx.y;
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= words) return;
  const int k = w * 32 + (threadIdx.x & 31);
  const bool on = k < n_k && mask[(long long)b * n_k + k] != 0;
  const uint32_t v = __ballot_sync(0xffffffffu, on);
  if ((threadIdx.x & 31) == 0) bits[(long long)b * words + w] = v;
}
}  // namespace alm

extern "C" int alm_pack_key_mask(const void* key_mask, void* bits, int b, int n_k, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(key_mask && bits && b > 0 && n_k > 0, ALM_ERR_ARG);
  const int words = (n_k + 127) / 128 * 4;
  dim3 grid(ceil_div(words, 8), b);
  pack_key_mask_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const uint8_t*>(key_mask),
                                                 reinterpret_cast<uint32_t*>(bits), n_k, words);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_mqa_attn_fwd(const void* q, int64_t ldq, const void* k, int64_t ldk, int64_t k_bstride,
                                const void* v, int64_t ldv, int64_t v_bstride, const void* key_mask, void* o,
                                int64_t ldo, float* lse, int64_t lse_stride, const float* bias, int64_t bias_hstride,
                                int64_t bias_rstride, int b, int h, int n_q, int n_k, int causal, float scale,
                                alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(q && k && v && o, ALM_ERR_ARG);
  ALM_REQUIRE(b > 0 && h > 0 && n_q > 0 && n_k > 0 && n_k >= n_q, ALM_ERR_ARG);
  ALM_REQUIRE(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, ALM_ERR_ALIGN);
  ALM_REQUIRE(k_bstride % 8 == 0 && v_bstride % 8 == 0, ALM_ERR_ALIGN);
  ALM_REQUIRE((reinterpret_cast<uintptr_t>(o) & 15u) == 0, ALM_ERR_ALIGN);
  if (bias != nullptr) {
    ALM_REQUIRE(bias_rstride >= n_k && bias_rstride % 4 == 0 && bias_hstride % 4 == 0, ALM_ERR_ALIGN);
    ALM_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15u) == 0, ALM_ERR_ALIGN);
  }

  CUtensorMap tmQ, tmK, tmV;
  {
    uint64_t dims[3] = {(uint64_t)h * ATT_D, (uint64_t)n_q, (uint64_t)b};
    uint64_t strides[3] = {2, (uint64_t)ldq * 2, (uint64_t)n_q * ldq * 2};
    uint32_t box[3] = {ATT_D, ATT_BM, 1};
    int rc = make_tensor_map(&tmQ, q, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
  }
  {
    uint64_t dims[3] = {(uint64_t)ATT_D, (uint64_t)n_k, (uint64_t)b};
    uint64_t strides[3] = {2, (uint64_t)ldk * 2, (uint64_t)k_bstride * 2};
    uint32_t box[3] = {ATT_D, ATT_BN, 1};
    int rc = make_tensor_map(&tmK, k, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
    strides[1] = (uint64_t)ldv * 2;
    strides[2] = (uint64_t)v_bstride * 2;
    rc = make_tensor_map(&tmV, v, 2, 3, dims, strides, box, true);
    if (rc != ALM_OK) return rc;
  }
  AttnFwdParams p;
  p.o = reinterpret_cast<__nv_bfloat16*>(o);
  p.lse = lse;
  p.kmask = reinterpret_cast<const uint32_t*>(key_mask);
  p.kb_stride = (n_k + 127) / 128 * 4;
  p.bias = bias;
  p.bias_hs = bias_hstride;
  p.bias_rs = bias_rstride;
  p.ldo = ldo;
  p.lse_stride = lse_stride;
  p.b = b; p.h = h; p.n_q = n_q; p.n_k = n_k;
  p.causal = causal;
  p.scale_log2 = scale * 1.4426950408889634f;
  static bool attr_set = false;
  if (!attr_set) {
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_fwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     ATT_SMEM_BYTES));
    ALM_CUDA_OK(cudaFuncSetAttribute(mqa_attn_fwd_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     ATT_SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((n_q + ATT_BM - 1) / ATT_BM, h, b);
  if (bias != nullptr)
    mqa_attn_fwd_kernel<true><<<grid, ATT_THREADS, ATT_SMEM_BYTES, stream>>>(tmQ, tmK, tmV, p);
  else
    mqa_attn_fwd_kernel<false><<<grid, ATT_THREADS, ATT_SMEM_BYTES, stream>>>(tmQ, tmK, tmV, p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
