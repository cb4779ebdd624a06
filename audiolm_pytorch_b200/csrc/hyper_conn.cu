// C ABI of the Hyper-Connections kernels (hyper_conn.cuh): argument checks, then a dispatch on the stream count to
// the launchers instantiated in hyper_conn_s*.cu.
#include "hyper_conn.cuh"

namespace alm {
ALM_HC_INSTANTIATE(extern template, 2)
ALM_HC_INSTANTIATE(extern template, 3)
ALM_HC_INSTANTIATE(extern template, 4)
ALM_HC_INSTANTIATE(extern template, 5)
ALM_HC_INSTANTIATE(extern template, 6)
ALM_HC_INSTANTIATE(extern template, 7)
ALM_HC_INSTANTIATE(extern template, 8)
}  // namespace alm

using namespace alm;

// call F<S>(args...) for the runtime stream count
#define HC_BY_STREAMS(F, ...)                  \
  switch (streams) {                           \
    case 2: return F<2>(__VA_ARGS__);          \
    case 3: return F<3>(__VA_ARGS__);          \
    case 4: return F<4>(__VA_ARGS__);          \
    case 5: return F<5>(__VA_ARGS__);          \
    case 6: return F<6>(__VA_ARGS__);          \
    case 7: return F<7>(__VA_ARGS__);          \
    case 8: return F<8>(__VA_ARGS__);          \
    default: return ALM_ERR_UNSUPPORTED;       \
  }

extern "C" int alm_hc_pre_fwd(const void* R_in, const void* Y, const float* beta_prev, const float* x_expand,
                              const float* gamma_hc, const float* dyn_alpha, const float* dyn_beta,
                              const float* static_alpha, const float* static_beta, const float* alpha_scale,
                              const float* beta_scale, const float* ln_gamma, void* R_out, void* bin, void* xn,
                              float* beta_out, float* aux, int M, int d, int streams, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(streams >= HC_MIN_S && streams <= HC_MAX_S, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(d % 8 == 0 && d >= 8 && d <= 8192 && M > 0, ALM_ERR_ARG);
  ALM_REQUIRE((x_expand != nullptr) != (R_in != nullptr), ALM_ERR_ARG);
  HC_BY_STREAMS(hc_pre_fwd_s, R_in, Y, beta_prev, x_expand, gamma_hc, dyn_alpha, dyn_beta, static_alpha, static_beta,
                alpha_scale, beta_scale, ln_gamma, R_out, bin, xn, beta_out, aux, M, d, stream)
}

extern "C" int alm_hc_pre_bwd(const void* R_in, const void* Y, const float* beta_prev, const float* x_expand,
                              const float* gamma_hc, const float* dyn_alpha, const float* dyn_beta,
                              const float* static_alpha, const float* static_beta, const float* alpha_scale,
                              const float* beta_scale, const float* ln_gamma, const float* aux, const void* dR_out,
                              const void* dxn, const void* dbin_extra, const float* dbeta, void* dR_in, void* dY,
                              float* dbeta_prev, float* dx_expand, float dx_scale, float* g_gamma_hc,
                              float* g_dyn_alpha, float* g_dyn_beta, float* g_static_alpha, float* g_static_beta,
                              float* g_alpha_scale, float* g_beta_scale, float* g_ln_gamma, int M, int d,
                              int streams, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(streams >= HC_MIN_S && streams <= HC_MAX_S, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(d % 8 == 0 && d >= 8 && d <= 8192 && M > 0, ALM_ERR_ARG);
  HC_BY_STREAMS(hc_pre_bwd_s, R_in, Y, beta_prev, x_expand, gamma_hc, dyn_alpha, dyn_beta, static_alpha, static_beta,
                alpha_scale, beta_scale, ln_gamma, aux, dR_out, dxn, dbin_extra, dbeta, dR_in, dY, dbeta_prev,
                dx_expand, dx_scale, g_gamma_hc, g_dyn_alpha, g_dyn_beta, g_static_alpha, g_static_beta,
                g_alpha_scale, g_beta_scale, g_ln_gamma, M, d, stream)
}

extern "C" int alm_hc_post_fwd(const void* R_in, const void* Y, const float* beta_prev, const float* ln_gamma,
                               void* out, float* stats, int M, int d, int streams, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(streams >= HC_MIN_S && streams <= HC_MAX_S, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(d % 8 == 0 && d >= 8 && d <= 8192 && M > 0, ALM_ERR_ARG);
  HC_BY_STREAMS(hc_post_fwd_s, R_in, Y, beta_prev, ln_gamma, out, stats, M, d, stream)
}

extern "C" int alm_hc_post_bwd(const void* R_in, const void* Y, const float* beta_prev, const float* ln_gamma,
                               const float* stats, const void* dout, void* dR_in, void* dY, float* dbeta_prev,
                               float* g_ln_gamma, int M, int d, int streams, alm_stream_t stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ALM_REQUIRE(streams >= HC_MIN_S && streams <= HC_MAX_S, ALM_ERR_UNSUPPORTED);
  ALM_REQUIRE(d % 8 == 0 && d >= 8 && d <= 8192 && M > 0, ALM_ERR_ARG);
  HC_BY_STREAMS(hc_post_bwd_s, R_in, Y, beta_prev, ln_gamma, stats, dout, dR_in, dY, dbeta_prev, g_ln_gamma, M, d,
                stream)
}
