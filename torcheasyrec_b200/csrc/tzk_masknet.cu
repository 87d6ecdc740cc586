// tzk_masknet.cu — C entry points of MaskNet's fused mask and FFN stages (tzk_masknet.cuh).  A translation unit of its
// own, so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#include "tzk_masknet.cuh"

using namespace tzk;

#define MASKNET_SHAPES(what, E, H)                                                                                    \
  TZK_REQUIRE(B >= 0 && grid >= 1, what ": need B >= 0 and grid >= 1");                                               \
  TZK_REQUIRE(tzk_masknet::usable(E, H, nb),                                                                          \
              what ": shape outside the kernels' cover (pad4(E) <= 1024, 4 <= H <= 1024 with H % 4 == 0, "            \
                   "1 <= n_mask_blocks <= 8)")

extern "C" int tzk_masknet_mask_fwd(const float* e, int32_t lde, const float* m, const float* b2, const float* gamma,
                                    const float* beta, int64_t B, int32_t E, int32_t nb, int32_t grid, float* v,
                                    float* stats, tzk_stream_t stream) {
  MASKNET_SHAPES("masknet_mask_fwd", E, 4);
  TZK_REQUIRE(lde >= E, "masknet_mask_fwd: need lde >= E");
  tzk_masknet::mask_fwd(e, lde, m, b2, gamma, beta, B, E, nb, grid, v, stats, as_stream(stream));
  TZK_CHECK_LAUNCH("masknet_mask_fwd_kernel");
  return 0;
}

extern "C" int tzk_masknet_mask_bwd(const float* e, int32_t lde, const float* m, const float* b2, const float* gamma,
                                    const float* beta, const float* stats, const float* dv, int64_t B, int32_t E,
                                    int32_t nb, int32_t grid, float* dm, float* de, float* partials, float* dparams,
                                    tzk_stream_t stream) {
  MASKNET_SHAPES("masknet_mask_bwd", E, 4);
  TZK_REQUIRE(lde >= E, "masknet_mask_bwd: need lde >= E");
  tzk_masknet::mask_bwd(e, lde, m, b2, gamma, beta, stats, dv, B, E, nb, grid, dm, de, partials, dparams,
                        as_stream(stream));
  TZK_CHECK_LAUNCH("masknet_mask_bwd_kernel");
  return 0;
}

extern "C" int tzk_masknet_ffn_fwd(const float* z, const float* b3, const float* gamma, const float* beta, int64_t B,
                                   int32_t H, int32_t nb, int32_t grid, float* y, float* stats, tzk_stream_t stream) {
  MASKNET_SHAPES("masknet_ffn_fwd", 1, H);
  tzk_masknet::ffn_fwd(z, b3, gamma, beta, B, H, nb, grid, y, stats, as_stream(stream));
  TZK_CHECK_LAUNCH("masknet_ffn_fwd_kernel");
  return 0;
}

extern "C" int tzk_masknet_ffn_bwd(const float* z, const float* b3, const float* gamma, const float* beta,
                                   const float* stats, const float* dy, int64_t B, int32_t H, int32_t nb, int32_t grid,
                                   float* dz, float* partials, float* dparams, tzk_stream_t stream) {
  MASKNET_SHAPES("masknet_ffn_bwd", 1, H);
  tzk_masknet::ffn_bwd(z, b3, gamma, beta, stats, dy, B, H, nb, grid, dz, partials, dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("masknet_ffn_bwd_kernel");
  return 0;
}
