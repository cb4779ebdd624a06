// Persistent, warp-specialised bf16 GEMM for sm_90a (H100).
//   warpgroup 0 : TMA producer (one elected lane of warp 0) — cp.async.bulk.tensor into a STAGES-deep SW128 smem ring
//   warpgroups 1, 2 : consumers — wgmma m64nBNk16 on rows [0, 64) / [64, 128) of the 128-row tile, fp32 accumulators
//                     in registers, then the epilogue: bf16 outputs that TMA can address go through a swizzled smem
//                     staging buffer and a TMA tensor store (the warpgroup goes on to the next tile while it drains),
//                     everything else (fp32 / accumulating / CE / misaligned C) is stored straight from the registers
// Operands may be K-major or MN-major (wgmma transpose bits), which covers forward (x W^T), dgrad (dy W) and
// wgrad (dy^T x) without materialising any transpose.
#include "alm_common.cuh"
#include "ptx_sm90.cuh"

namespace alm {

struct GemmParams {
  void* C;
  const float* bias;
  long long ldc, strideC;
  int M, N, K, batch;
  int m_blocks, n_blocks, k_blocks, split_k;
  int c_fp32, acc_mode;
  int tma_store;  // bf16 C, acc_mode 0, 16-B aligned base and pitches: epilogue through smem + tmC
  float alpha;
  // fused logit head + cross entropy (CE kernel variant only; alm_gemm_head_ce):
  //   ce_mode 1: nothing is stored; every (row, n tile) emits its soft-max partial {max, sum 2^(t - max)} of
  //              t = logit * log2(e) into ce_part [M][n_blocks][2], and the tile that holds the label its logit into ce_lab
  //   ce_mode 2: C (bf16) = (softmax - onehot) * (*ce_num / *ce_den), zero rows where label == ce_ignore
  int ce_mode;
  const long long* ce_labels;
  long long ce_ignore;
  float* ce_part;
  float* ce_lab;
  const float* ce_lse;   // natural-log LSE per row (mode 2)
  const float* ce_num;
  const float* ce_den;
};

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;
constexpr int GEMM_THREADS = 384;

template <int BLOCK_N>
struct GemmCfg {
  static constexpr int STAGES = BLOCK_N == 256 ? 4 : (BLOCK_N == 128 ? 6 : 8);
  static constexpr int A_BYTES = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;
  static constexpr int B_BYTES = BLOCK_N * GEMM_BLOCK_K * 2;
  // epilogue staging: 2 consumer warpgroups x 2 buffers x [64 rows][64 bf16] (SW128, one TMA store box each)
  static constexpr int C_SUB_BYTES = 64 * 64 * 2;
  static constexpr int C_STAGE_BYTES = 4 * C_SUB_BYTES;
  static constexpr int SMEM_BYTES =
      STAGES * (A_BYTES + B_BYTES) + C_STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(SMEM_BYTES <= 227 * 1024, "exceeds the sm_90 dynamic shared memory limit");
};

template <int BLOCK_N, bool A_MN, bool B_MN, bool CE = false>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmC, const GemmParams p) {
  using Cfg = GemmCfg<BLOCK_N>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + STAGES * Cfg::A_BYTES;
  uint8_t* stage_c = smem + STAGES * (Cfg::A_BYTES + Cfg::B_BYTES);  // 1024-B aligned (SW128 TMA box)
  uint64_t* bars = reinterpret_cast<uint64_t*>(stage_c + Cfg::C_STAGE_BYTES);
  uint64_t* full_bar = bars;                  // [STAGES]  TMA -> MMA
  uint64_t* empty_bar = bars + STAGES;        // [STAGES]  consumers -> TMA (one arrive per consumer warp)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (p.tma_store) tma_prefetch_desc(&tmC);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int tiles_per_batch = p.m_blocks * p.n_blocks * p.split_k;
  const int total_tiles = tiles_per_batch * p.batch;
  const int kb_per_split = (p.k_blocks + p.split_k - 1) / p.split_k;

  // tile -> (batch, split, m block, n block); n fastest so consecutive CTAs share the A panel
  auto decode = [&](int t, int& b, int& s, int& mb, int& nb) {
    b = t / tiles_per_batch;
    int r = t - b * tiles_per_batch;
    s = r / (p.m_blocks * p.n_blocks);
    r -= s * (p.m_blocks * p.n_blocks);
    mb = r / p.n_blocks;
    nb = r - mb * p.n_blocks;
  };
  auto k_range = [&](int s, int& kb0, int& kb1) {
    kb0 = s * kb_per_split;
    kb1 = min(p.k_blocks, kb0 + kb_per_split);
  };

  if (wg == 0) {
    setmaxnreg_dec<40>();
    if (warp == 0) {
      // ===================== TMA producer (whole warp runs the uniform loop, one elected lane issues) ============
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        int b, s, mb, nb, kb0, kb1;
        decode(t, b, s, mb, nb);
        k_range(s, kb0, kb1);
        const int m0 = mb * GEMM_BLOCK_M, n0 = nb * BLOCK_N;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem_a + stage * Cfg::A_BYTES;
          uint8_t* sb = smem_b + stage * Cfg::B_BYTES;
          const int k0 = kb * GEMM_BLOCK_K;
          if (elect_one_sync()) {
            mbar_arrive_expect_tx(&full_bar[stage], Cfg::A_BYTES + Cfg::B_BYTES);
            if constexpr (!A_MN) {
              tma_load_3d(sa, &tmA, &full_bar[stage], k0, m0, b);
            } else {
#pragma unroll
              for (int i = 0; i < GEMM_BLOCK_M / 64; ++i)
                tma_load_3d(sa + i * (GEMM_BLOCK_K * 128), &tmA, &full_bar[stage], m0 + i * 64, k0, b);
            }
            if constexpr (!B_MN) {
              tma_load_3d(sb, &tmB, &full_bar[stage], k0, n0, b);
            } else {
#pragma unroll
              for (int i = 0; i < BLOCK_N / 64; ++i)
                tma_load_3d(sb + i * (GEMM_BLOCK_K * 128), &tmB, &full_bar[stage], n0 + i * 64, k0, b);
            }
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================== consumers: warpgroup cw owns rows [64 cw, 64 cw + 64) of every tile =====================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;
  const int wq = warp & 3;
  const int r_base = cw * 64 + wq * 16 + (lane >> 2);  // accumulator rows r_base and r_base + 8
  const int c_lane = 2 * (lane & 3);                    // accumulator columns 8 j + c_lane, + 1
  int stage = 0;
  uint32_t phase = 0;
  float acc[BLOCK_N / 2];
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    int b, s, mb, nb, kb0, kb1;
    decode(t, b, s, mb, nb);
    k_range(s, kb0, kb1);
    int prev_stage = -1;
    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a_addr = smem_u32(smem_a + stage * Cfg::A_BYTES) + cw * 8192;
      const uint32_t b_addr = smem_u32(smem_b + stage * Cfg::B_BYTES);
      wgmma_fence_acc(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) {
        const uint64_t da = A_MN ? wgmma_desc_sw128(a_addr + k * 2048, 1024, GEMM_BLOCK_K * 128)
                                 : wgmma_desc_sw128(a_addr + k * 32, 1024, 16);
        const uint64_t db = B_MN ? wgmma_desc_sw128(b_addr + k * 2048, 1024, GEMM_BLOCK_K * 128)
                                 : wgmma_desc_sw128(b_addr + k * 32, 1024, 16);
        wgmma_ss<BLOCK_N, A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, (kb > kb0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();  // the previous k block's MMAs are done: its smem slot may be refilled
      wgmma_fence_acc(acc);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    const int n0 = nb * BLOCK_N;
    if constexpr (!CE) {
      if (p.tma_store) {
        // ============ epilogue through smem: 64-column sub-tiles of this warpgroup's 64 rows, one TMA store each ====
        // same values and bf16 rounding as the register path; TMA clips rows >= M and columns >= N
        // (thread 0 of the warpgroup issues and waits for its stores; an even sub-tile count alternates the two
        // buffers, a single sub-tile (BLOCK_N 64) reuses one)
        constexpr int SUBS = BLOCK_N / 64, NBUF = SUBS % 2 == 0 ? 2 : 1;
        // this thread's staging rows: wq * 16 + lane / 4 and + 8, whose (row & 7) = lane / 4 picks the swizzle
        const uint32_t st_base =
            smem_u32(stage_c) + cw * 2 * Cfg::C_SUB_BYTES + (wq * 16 + (lane >> 2)) * 128 + (lane & 3) * 4;
#pragma unroll
        for (int sub = 0; sub < SUBS; ++sub) {
          uint8_t* buf = stage_c + (cw * 2 + sub % NBUF) * Cfg::C_SUB_BYTES;
          if ((threadIdx.x & 127) == 0) bulk_wait_group_read<NBUF - 1>();  // last store from this buffer read it
          named_bar_sync(1 + cw, 128);
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = sub * 8 + jj;
              const int col = n0 + 8 * j + c_lane;
              float v0 = acc[4 * j + 2 * h] * p.alpha, v1 = acc[4 * j + 2 * h + 1] * p.alpha;
              if (p.bias != nullptr) {
                if (col < p.N) v0 += __ldg(p.bias + col);
                if (col + 1 < p.N) v1 += __ldg(p.bias + col + 1);
              }
              // 128-B swizzle: 16-B chunk jj of row r sits at chunk jj ^ (r & 7) -> conflict-free 4-B stores
              st_shared_u32(st_base + (sub % NBUF) * Cfg::C_SUB_BYTES + h * 1024 + ((jj ^ (lane >> 2)) << 4),
                            pack_bf16x2(v0, v1));
            }
          fence_proxy_async_smem();
          named_bar_sync(1 + cw, 128);
          if ((threadIdx.x & 127) == 0) {
            tma_store_3d(&tmC, buf, n0 + sub * 64, mb * GEMM_BLOCK_M + cw * 64, b);
            bulk_commit_group();
          }
        }
        continue;
      }
    }

    // ===================== epilogue from the accumulator fragment =====================
    // split-K: the bias is added once, by the split that owns k block 0
    const float* bias = s == 0 ? p.bias : nullptr;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gm = mb * GEMM_BLOCK_M + r_base + 8 * h;
      const bool row_ok = gm < p.M;
      const long long row_off = (long long)b * p.strideC + (long long)gm * p.ldc;
      // fused head + cross entropy: this row's state for the tile
      [[maybe_unused]] float ce_lse2 = 0.f, ce_scale = 0.f;
      [[maybe_unused]] long long ce_label = -1;  // the label's column, -1 when the label is not a column
      if constexpr (CE) {
        bool bad_label = false;  // outside [0, N) and not ignore_index: its loss and gradient row are NaN
        if (row_ok) {
          const long long label = p.ce_labels[gm];
          const bool in_range = label >= 0 && label < p.N;
          ce_label = in_range ? label : -1;
          bad_label = !in_range && label != p.ce_ignore;
          if (p.ce_mode == 2) {
            ce_lse2 = p.ce_lse[gm] * 1.4426950408889634f;
            ce_scale = label == p.ce_ignore ? 0.f
                       : bad_label      ? __int_as_float(0x7fc00000)
                                        : __ldg(p.ce_num) / __ldg(p.ce_den);
          }
        }
        if (p.ce_mode == 1) {
          // no tile holds a bad label's column: the first tile writes its NaN, so every row keeps exactly one writer
          if (bad_label && nb == 0 && (lane & 3) == 0) p.ce_lab[gm] = __int_as_float(0x7fc00000);
          // row max / sum over the tile: each thread covers 2 columns per 8-column group, the 4 lanes of a quad the row
          float cm = -INFINITY;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int col = n0 + 8 * j + c_lane + c;
              float v = acc[4 * j + 2 * h + c] * p.alpha;
              if (bias != nullptr && col < p.N) v += __ldg(bias + col);
              if (row_ok && col == ce_label) p.ce_lab[gm] = v;
              v = col < p.N ? v * 1.4426950408889634f : -INFINITY;
              acc[4 * j + 2 * h + c] = v;
              cm = fmaxf(cm, v);
            }
          cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 1));
          cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 2));  // finite: the tile has at least one valid column
          float cs = 0.f;
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) cs += exp2f(acc[4 * j + 2 * h + c] - cm);
          cs += __shfl_xor_sync(0xffffffffu, cs, 1);
          cs += __shfl_xor_sync(0xffffffffu, cs, 2);
          if (row_ok && (lane & 3) == 0) {
            float* pp = p.ce_part + ((size_t)gm * p.n_blocks + nb) * 2;
            pp[0] = cm;
            pp[1] = cs;
          }
          continue;  // nothing is stored in this mode
        }
      }
      if (!row_ok) continue;
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = n0 + 8 * j + c_lane;
        if (col >= p.N) break;
        float v0 = acc[4 * j + 2 * h] * p.alpha, v1 = acc[4 * j + 2 * h + 1] * p.alpha;
        const bool pair = col + 1 < p.N;
        if (bias != nullptr) {
          v0 += __ldg(bias + col);
          if (pair) v1 += __ldg(bias + col + 1);
        }
        if constexpr (CE) {
          v0 = (exp2f(v0 * 1.4426950408889634f - ce_lse2) - (col == ce_label ? 1.f : 0.f)) * ce_scale;
          v1 = (exp2f(v1 * 1.4426950408889634f - ce_lse2) - (col + 1 == ce_label ? 1.f : 0.f)) * ce_scale;
        }
        if (p.c_fp32) {
          float* dst = reinterpret_cast<float*>(p.C) + row_off + col;
          const bool vec = pair && ((reinterpret_cast<uintptr_t>(dst) & 7u) == 0);
          if (p.acc_mode == 2) {
            if (vec) {
              asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(dst), "f"(v0), "f"(v1) : "memory");
            } else {
              atomicAdd(dst, v0);
              if (pair) atomicAdd(dst + 1, v1);
            }
          } else if (vec) {
            float2 o = make_float2(v0, v1);
            if (p.acc_mode == 1) {
              const float2 old = *reinterpret_cast<float2*>(dst);
              o.x += old.x; o.y += old.y;
            }
            *reinterpret_cast<float2*>(dst) = o;
          } else {
            dst[0] = (p.acc_mode == 1 ? dst[0] : 0.f) + v0;
            if (pair) dst[1] = (p.acc_mode == 1 ? dst[1] : 0.f) + v1;
          }
        } else {
          __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(p.C) + row_off + col;
          if (p.acc_mode != 0) {
            v0 += __bfloat162float(dst[0]);
            if (pair) v1 += __bfloat162float(dst[1]);
          }
          if (pair && ((reinterpret_cast<uintptr_t>(dst) & 3u) == 0)) {
            *reinterpret_cast<uint32_t*>(dst) = pack_bf16x2(v0, v1);
          } else {
            dst[0] = __float2bfloat16_rn(v0);
            if (pair) dst[1] = __float2bfloat16_rn(v1);
          }
        }
      }
    }
  }
  if ((threadIdx.x & 127) == 0) bulk_wait_group<0>();  // the CTA's smem must outlive its pending TMA stores
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool CE = false>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const CUtensorMap& tmC, const GemmParams& p,
                       cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N>;
  auto kfn = gemm_bf16_wgmma_kernel<BLOCK_N, A_MN, B_MN, CE>;
  static bool attr_set = false;
  if (!attr_set) {
    ALM_CUDA_OK(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::SMEM_BYTES));
    attr_set = true;
  }
  const int total = p.m_blocks * p.n_blocks * p.split_k * p.batch;
  const int grid = total < num_sms() ? total : num_sms();
  kfn<<<grid, GEMM_THREADS, Cfg::SMEM_BYTES, stream>>>(tmA, tmB, tmC, p);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

// (transformer.gemm_block_n keeps a host copy for best_split_k; tests/test_gemm_ce_envelope_gpu.py checks they agree)
static int pick_block_n(int N) {
  if (N <= 64) return 64;
  if (N <= 128) return 128;
  // 128x256 tiles have 33 % more FLOP per operand byte than 128x128 (85 vs 64 FLOP/B of smem fill), which is what
  // decides throughput for K ~ 1024; accept up to ~10 % padded columns before falling back to 128-wide tiles
  const int pad256 = ceil_div(N, 256) * 256, pad128 = ceil_div(N, 128) * 128;
  return (pad128 * 10 < pad256 * 9) ? 128 : 256;
}

}  // namespace alm

namespace alm {
struct CeEpilogue {
  int mode;
  const long long* labels;
  long long ignore;
  float* part;
  float* lab;
  const float* lse;
  const float* num;
  const float* den;
};
}  // namespace alm

static int gemm_common(const void* A, int a_mn, int64_t lda, int64_t strideA, const void* B, int b_mn, int64_t ldb,
                       int64_t strideB, void* C, int c_fp32, int64_t ldc, int64_t strideC, int M, int N, int K, int batch,
                       float alpha, const float* bias, int acc_mode, int split_k, cudaStream_t stream,
                       const alm::CeEpilogue* ce) {
  using namespace alm;
  ALM_REQUIRE(A && B && (C || (ce && ce->mode == 1)), ALM_ERR_ARG);
  ALM_REQUIRE(M > 0 && N > 0 && K > 0 && batch > 0, ALM_ERR_ARG);
  ALM_REQUIRE(acc_mode >= 0 && acc_mode <= 2 && split_k >= 1, ALM_ERR_ARG);
  ALM_REQUIRE(split_k == 1 || (acc_mode == 2 && c_fp32), ALM_ERR_ARG);
  ALM_REQUIRE(!(a_mn && !b_mn), ALM_ERR_UNSUPPORTED);  // (MN,K) is never needed on this path
  ALM_REQUIRE(lda % 8 == 0 && ldb % 8 == 0 && strideA % 8 == 0 && strideB % 8 == 0, ALM_ERR_ALIGN);

  const int BN = pick_block_n(N);
  GemmParams p;
  p.C = C;
  p.bias = bias;
  p.ldc = ldc;
  p.strideC = strideC;
  p.M = M; p.N = N; p.K = K; p.batch = batch;
  p.m_blocks = ceil_div(M, GEMM_BLOCK_M);
  p.n_blocks = ceil_div(N, BN);
  p.k_blocks = ceil_div(K, GEMM_BLOCK_K);
  if (split_k > p.k_blocks) split_k = p.k_blocks;
  // every split must own at least one k block
  while (split_k > 1 && (split_k - 1) * ceil_div(p.k_blocks, split_k) >= p.k_blocks) --split_k;
  p.split_k = split_k;
  p.c_fp32 = c_fp32;
  p.acc_mode = acc_mode;
  p.alpha = alpha;
  p.ce_mode = 0;
  if (ce != nullptr) {
    p.ce_mode = ce->mode;
    p.ce_labels = ce->labels;
    p.ce_ignore = ce->ignore;
    p.ce_part = ce->part;
    p.ce_lab = ce->lab;
    p.ce_lse = ce->lse;
    p.ce_num = ce->num;
    p.ce_den = ce->den;
  }

  CUtensorMap tmA, tmB;
  {
    uint64_t dims[3], strides[3];
    uint32_t box[3];
    if (!a_mn) {
      dims[0] = (uint64_t)K; dims[1] = (uint64_t)M;
      box[0] = GEMM_BLOCK_K; box[1] = GEMM_BLOCK_M;
    } else {
      dims[0] = (uint64_t)M; dims[1] = (uint64_t)K;
      box[0] = 64; box[1] = GEMM_BLOCK_K;
    }
    dims[2] = (uint64_t)batch; box[2] = 1;
    strides[0] = 2; strides[1] = (uint64_t)lda * 2;
    strides[2] = batch > 1 ? (uint64_t)strideA * 2 : dims[1] * strides[1];
    int rc = make_tensor_map(&tmA, A, 2, 3, dims, strides, box, 128);
    if (rc != ALM_OK) return rc;
  }
  {
    uint64_t dims[3], strides[3];
    uint32_t box[3];
    if (!b_mn) {
      dims[0] = (uint64_t)K; dims[1] = (uint64_t)N;
      box[0] = GEMM_BLOCK_K; box[1] = (uint32_t)BN;
    } else {
      dims[0] = (uint64_t)N; dims[1] = (uint64_t)K;
      box[0] = 64; box[1] = GEMM_BLOCK_K;
    }
    dims[2] = (uint64_t)batch; box[2] = 1;
    strides[0] = 2; strides[1] = (uint64_t)ldb * 2;
    strides[2] = batch > 1 ? (uint64_t)strideB * 2 : dims[1] * strides[1];
    int rc = make_tensor_map(&tmB, B, 2, 3, dims, strides, box, 128);
    if (rc != ALM_OK) return rc;
  }

  // bf16 stores through TMA where a tensor map can describe C (16-B aligned base and pitches); the rest keeps the
  // register epilogue (fp32 C, read-modify-write accumulation, the CE variant, e.g. a pitch of 10,920 B)
  CUtensorMap tmC = {};
  p.tma_store = ce == nullptr && !c_fp32 && acc_mode == 0 && (reinterpret_cast<uintptr_t>(C) & 15u) == 0 &&
                (ldc * 2) % 16 == 0 && (batch == 1 || (strideC * 2) % 16 == 0);
  if (p.tma_store) {
    const uint64_t dims[3] = {(uint64_t)N, (uint64_t)M, (uint64_t)batch};
    const uint64_t strides[3] = {2, (uint64_t)ldc * 2, batch > 1 ? (uint64_t)strideC * 2 : (uint64_t)M * ldc * 2};
    const uint32_t box[3] = {64, 64, 1};
    int rc = make_tensor_map(&tmC, C, 2, 3, dims, strides, box, 128);
    if (rc != ALM_OK) return rc;
  }

  if (ce != nullptr) {   // (row-major x, row-major head weight: the only layout the fused head needs)
    if (BN == 256) return launch_gemm<256, false, false, true>(tmA, tmB, tmC, p, stream);
    if (BN == 128) return launch_gemm<128, false, false, true>(tmA, tmB, tmC, p, stream);
    return launch_gemm<64, false, false, true>(tmA, tmB, tmC, p, stream);
  }
#define ALM_GEMM_DISPATCH(BN_)                                                             \
  if (!a_mn && !b_mn) return launch_gemm<BN_, false, false>(tmA, tmB, tmC, p, stream);     \
  if (!a_mn && b_mn) return launch_gemm<BN_, false, true>(tmA, tmB, tmC, p, stream);       \
  return launch_gemm<BN_, true, true>(tmA, tmB, tmC, p, stream);
  if (BN == 256) { ALM_GEMM_DISPATCH(256) }
  if (BN == 128) { ALM_GEMM_DISPATCH(128) }
  { ALM_GEMM_DISPATCH(64) }
#undef ALM_GEMM_DISPATCH
}

extern "C" int alm_gemm_bf16(const void* A, int a_mn, int64_t lda, int64_t strideA, const void* B, int b_mn,
                             int64_t ldb, int64_t strideB, void* C, int c_fp32, int64_t ldc, int64_t strideC, int M,
                             int N, int K, int batch, float alpha, const float* bias, int acc_mode, int split_k,
                             alm_stream_t stream_) {
  return gemm_common(A, a_mn, lda, strideA, B, b_mn, ldb, strideB, C, c_fp32, ldc, strideC, M, N, K, batch, alpha, bias,
                     acc_mode, split_k, reinterpret_cast<cudaStream_t>(stream_), nullptr);
}

// number of n tiles of the head GEMM for a vocabulary of V (= the second dimension of `part` below)
extern "C" int alm_gemm_head_ce_tiles(int V) { return alm::ceil_div(V, alm::pick_block_n(V)); }

// Fused logit head + cross entropy (audiolm_pytorch.py:621, 798, 965-983, 1325-1361 heads; :1561-1565, 1836-1854,
// 2119-2137 F.cross_entropy): the [M, V] fp32 logits never reach HBM.
//   mode 1: logits = X W^T (+ bias) are reduced in the GEMM epilogue to per-(row, n tile) soft-max partials
//           part [M, tiles, 2] = {max, sum 2^(t - max)} of t = logit * log2(e), and lab_logit [M] = logit[label];
//           alm_ce_finish turns them into the row LSE and loss
//   mode 2: the GEMM is recomputed and its epilogue writes d(loss)/d(logits) = (softmax - onehot) * (*scale_num /
//           *scale_den) as bf16 [M, ldd] (rows with label == ignore_index are zero; columns >= V are not written)
extern "C" int alm_gemm_head_ce(const void* X, int64_t ldx, const void* W, int64_t ldw, const float* bias,
                                const int64_t* labels, int64_t ignore_index, int mode, float* part, float* lab_logit,
                                const float* lse, const float* scale_num, const float* scale_den, void* dlogits,
                                int64_t ldd, int M, int V, int K, alm_stream_t stream_) {
  ALM_REQUIRE(mode == 1 || mode == 2, ALM_ERR_ARG);
  ALM_REQUIRE(labels != nullptr, ALM_ERR_ARG);
  if (mode == 1) ALM_REQUIRE(part && lab_logit, ALM_ERR_ARG);
  else ALM_REQUIRE(lse && scale_num && scale_den && dlogits && ldd >= V, ALM_ERR_ARG);
  alm::CeEpilogue ce{mode, reinterpret_cast<const long long*>(labels), (long long)ignore_index, part, lab_logit, lse,
                     scale_num, scale_den};
  return gemm_common(X, 0, ldx, 0, W, 0, ldw, 0, dlogits, 0, ldd, 0, M, V, K, 1, 1.f, bias, 0, 1,
                     reinterpret_cast<cudaStream_t>(stream_), &ce);
}
