// tzk_rocket.cu — C entry points of RocketLaunching's fused booster / light head (tzk_rocket.cuh).  A translation unit
// of its own, so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#include "tzk_rocket.cuh"

using namespace tzk;

#define ROCKET_COVER                                                                                                  \
  "head description outside the kernels' cover (2 <= C <= 8, hidden and pair widths 4..1024 and multiples of 4, "   \
  "16-B aligned rows, at most 8 pairs, pairs only with the booster head and labels)"

extern "C" int tzk_rocket_head_fwd(const tzk_rocket_args* args_host, int32_t grid, float* partials, float* losses,
                                   tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_rocket::check(*args_host, false) == 0, "rocket_head_fwd: " ROCKET_COVER);
  TZK_REQUIRE(grid >= 1 && (losses == nullptr || partials != nullptr) &&
                  (args_host->B == 0 || (args_host->labels == nullptr) == (losses == nullptr)),
              "rocket_head_fwd: need grid >= 1 and, with labels, the partials / losses buffers");
  tzk_rocket::head_fwd(*args_host, grid, partials, losses, as_stream(stream));
  TZK_CHECK_LAUNCH("rocket_head_fwd_kernel");
  return 0;
}

extern "C" int tzk_rocket_head_bwd(const tzk_rocket_args* args_host, const float* dlosses, const float* losses,
                                   int32_t grid, float* partials, float* dparams, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_rocket::check(*args_host, true) == 0, "rocket_head_bwd: " ROCKET_COVER);
  TZK_REQUIRE(grid >= 1 && dlosses != nullptr && losses != nullptr && partials != nullptr && dparams != nullptr,
              "rocket_head_bwd: need grid >= 1 and the dlosses / losses / partials / dparams buffers");
  tzk_rocket::head_bwd(*args_host, dlosses, losses, grid, partials, dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("rocket_head_bwd_kernel");
  return 0;
}
