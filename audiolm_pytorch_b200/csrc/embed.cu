// Token embedding gather / scatter for the three transformers (SURVEY K4).
//
// Reference: audiolm_pytorch.py:686-699 (semantic), :896-918 (coarse), :1188-1223 (fine): every input position is the
// sum of up to two rows taken from a handful of parameter tables (a start token, nn.Embedding rows offset by the
// quantizer, the quantizer-position embedding), concatenated along the sequence.  The reference issues
// `nn.Embedding` + `repeat` + `torch.cat` + adds, and autograd answers with a sort-based `embedding_dense_backward`
// per table (16 radix-sort launches per step in the round-1 launch list).  Here: ONE gather launch and ONE scatter
// launch driven by a per-position source list.
//
//   src [M][2] int32: (table_id << 24) | row, or -1 for "no contribution" (padding ids, positions with one source)
//   out [M][d] fp32 = sum of the selected rows                      (forward)
//   grad_tables[table_id][row][:] += dout[m][:]                     (backward, 16-byte vector reductions)
#include "alm_common.cuh"

namespace alm {

constexpr int EMB_MAX_TABLES = 8;
struct EmbTables {
  const float* t[EMB_MAX_TABLES];
};
struct EmbGradTables {
  float* t[EMB_MAX_TABLES];
};

__global__ void __launch_bounds__(256) embed_gather_kernel(EmbTables tabs, const int* __restrict__ src,
                                                           float* __restrict__ out, int M, int d) {
  const int vec = d / 4;  // float4 per row
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)M * vec;
       i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec), v = (int)(i - (long long)m * vec);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int s = __ldg(src + 2 * m + k);
      if (s >= 0) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(tabs.t[s >> 24] + (size_t)(s & 0xFFFFFF) * d) + v);
        acc.x += r.x; acc.y += r.y; acc.z += r.z; acc.w += r.w;
      }
    }
    reinterpret_cast<float4*>(out)[i] = acc;
  }
}

__global__ void __launch_bounds__(256) embed_scatter_kernel(EmbGradTables tabs, const int* __restrict__ src,
                                                            const float* __restrict__ dout, int M, int d) {
  const int vec = d / 4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < (long long)M * vec;
       i += (long long)gridDim.x * blockDim.x) {
    const int m = (int)(i / vec), v = (int)(i - (long long)m * vec);
    const float4 g = __ldg(reinterpret_cast<const float4*>(dout) + i);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int s = __ldg(src + 2 * m + k);
      if (s >= 0) {
        float* dst = tabs.t[s >> 24] + (size_t)(s & 0xFFFFFF) * d + 4 * v;
        asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "f"(g.x), "f"(g.y), "f"(g.z), "f"(g.w)
                     : "memory");
      }
    }
  }
}

}  // namespace alm

extern "C" int alm_embed_gather(const float* const* tables, int n_tables, const int32_t* src, float* out, int M, int d,
                                alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(tables && src && out && M > 0 && d > 0 && d % 4 == 0, ALM_ERR_ARG);
  ALM_REQUIRE(n_tables >= 1 && n_tables <= EMB_MAX_TABLES, ALM_ERR_UNSUPPORTED);
  EmbTables t{};
  for (int i = 0; i < n_tables; ++i) {
    ALM_REQUIRE((reinterpret_cast<uintptr_t>(tables[i]) & 15u) == 0, ALM_ERR_ALIGN);
    t.t[i] = tables[i];
  }
  const long long work = (long long)M * (d / 4);
  const int grid = (int)((work + 255) / 256 < num_sms() * 16 ? (work + 255) / 256 : num_sms() * 16);
  embed_gather_kernel<<<grid, 256, 0, stream>>>(t, src, out, M, d);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}

extern "C" int alm_embed_scatter(float* const* grad_tables, int n_tables, const int32_t* src, const float* dout, int M,
                                 int d, alm_stream_t stream_) {
  using namespace alm;
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(grad_tables && src && dout && M > 0 && d > 0 && d % 4 == 0, ALM_ERR_ARG);
  ALM_REQUIRE(n_tables >= 1 && n_tables <= EMB_MAX_TABLES, ALM_ERR_UNSUPPORTED);
  EmbGradTables t{};
  for (int i = 0; i < n_tables; ++i) {
    ALM_REQUIRE((reinterpret_cast<uintptr_t>(grad_tables[i]) & 15u) == 0, ALM_ERR_ALIGN);
    t.t[i] = grad_tables[i];
  }
  const long long work = (long long)M * (d / 4);
  const int grid = (int)((work + 255) / 256 < num_sms() * 16 ? (work + 255) / 256 : num_sms() * 16);
  embed_scatter_kernel<<<grid, 256, 0, stream>>>(t, src, dout, M, d);
  ALM_CHECK_LAUNCH();
  ALM_LAUNCHED(1);
  return ALM_OK;
}
