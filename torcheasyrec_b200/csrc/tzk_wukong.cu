// tzk_wukong.cu — C entry points of the WuKong layer's fused interaction (tzk_wukong.cuh).  A translation unit of its
// own, so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#include "tzk_wukong.cuh"

using namespace tzk;

#define WUKONG_SHAPES(what)                                                                                          \
  TZK_REQUIRE(B >= 0 && grid >= 1, what ": need B >= 0 and grid >= 1");                                               \
  TZK_REQUIRE(tzk_wukong::usable(n, d, k, f, l),                                                                      \
              what ": shape outside the kernels' cover (n <= 64, d in {4, 8, 16, 32}, k <= 32, f, l >= 1, f + l <= 64)")

extern "C" int tzk_wukong_mix_fwd(const float* x, const float* w_fmb, const float* gamma, const float* beta,
                                  const float* w_lcb, const float* w_res, int64_t B, int32_t n, int32_t d, int32_t k,
                                  int32_t f, int32_t l, int32_t grid, float* ln_f, float* stats, float* base,
                                  tzk_stream_t stream) {
  WUKONG_SHAPES("wukong_mix_fwd");
  TZK_REQUIRE(w_res != nullptr || n == f + l, "wukong_mix_fwd: the identity residual needs n == f + l");
  tzk_wukong::mix_fwd(x, w_fmb, gamma, beta, w_lcb, w_res, B, n, d, k, f, l, grid, ln_f, stats, base,
                      as_stream(stream));
  TZK_CHECK_LAUNCH("wukong_mix_fwd_kernel");
  return 0;
}

extern "C" int tzk_wukong_mix_bwd(const float* x, const float* w_fmb, const float* gamma, const float* w_lcb,
                                  const float* w_res, const float* stats, const float* d_ln_f, const float* d_base,
                                  int64_t B, int32_t n, int32_t d, int32_t k, int32_t f, int32_t l, int32_t grid,
                                  float* dx, float* partials, float* dparams, tzk_stream_t stream) {
  WUKONG_SHAPES("wukong_mix_bwd");
  TZK_REQUIRE(w_res != nullptr || n == f + l, "wukong_mix_bwd: the identity residual needs n == f + l");
  tzk_wukong::mix_bwd(x, w_fmb, gamma, w_lcb, w_res, stats, d_ln_f, d_base, B, n, d, k, f, l, grid, dx, partials,
                      dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("wukong_mix_bwd_kernel");
  return 0;
}

extern "C" int tzk_wukong_out_fwd(const float* fmb_out, const float* base, const float* gamma, const float* beta,
                                  int64_t B, int32_t d, int32_t f, int32_t l, int32_t grid, float* y, float* stats,
                                  tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && grid >= 1, "wukong_out_fwd: need B >= 0 and grid >= 1");
  TZK_REQUIRE(tzk_wukong::out_fwd(fmb_out, base, gamma, beta, B, d, f, l, grid, y, stats, as_stream(stream)) == 0,
              "wukong_out_fwd: need d in {4, 8, 16, 32} and f, l >= 1");
  TZK_CHECK_LAUNCH("wukong_out_fwd_kernel");
  return 0;
}

extern "C" int tzk_wukong_out_bwd(const float* fmb_out, const float* base, const float* gamma, const float* stats,
                                  const float* dy, int64_t B, int32_t d, int32_t f, int32_t l, int32_t grid,
                                  float* d_fmb_out, float* d_base, float* partials, float* dparams,
                                  tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && grid >= 1, "wukong_out_bwd: need B >= 0 and grid >= 1");
  TZK_REQUIRE(tzk_wukong::out_bwd(fmb_out, base, gamma, stats, dy, B, d, f, l, grid, d_fmb_out, d_base, partials,
                                  dparams, as_stream(stream)) == 0,
              "wukong_out_bwd: need d in {4, 8, 16, 32} and f, l >= 1");
  TZK_CHECK_LAUNCH("wukong_out_bwd_kernel");
  return 0;
}
