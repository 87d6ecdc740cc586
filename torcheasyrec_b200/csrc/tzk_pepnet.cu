// tzk_pepnet.cu — C entry points of PEPNet's fused gate-neural-unit product (tzk_pepnet.cuh).  A translation unit of
// its own, so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#define TZK_UNPAREN(...) __VA_ARGS__
#define TZK_LAUNCH(kernel, grid, block, smem, stream, ...) TZK_UNPAREN kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#include "tzk_pepnet.cuh"

using namespace tzk;

#define PEPNET_COVER                                                                                                  \
  "segments outside the kernels' cover (1 <= n_segs <= 8, 4 <= N <= 1024 with N % 4 == 0, pitches multiples of 4 "   \
  "floats, 16-B aligned pointers, act identity or ReLU)"

extern "C" int tzk_pepnet_gate_fwd(const tzk_pepnet_gate_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_pepnet::check(*args_host, false) == 0, "pepnet_gate_fwd: " PEPNET_COVER);
  TZK_REQUIRE(grid >= 1, "pepnet_gate_fwd: need grid >= 1");
  tzk_pepnet::gate_fwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("pepnet_gate_fwd_kernel");
  return 0;
}

extern "C" int tzk_pepnet_gate_bwd(const tzk_pepnet_gate_args* args_host, int32_t grid, float* partials,
                                   float* dparams, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_pepnet::check(*args_host, true) == 0, "pepnet_gate_bwd: " PEPNET_COVER);
  TZK_REQUIRE(grid >= 1 && partials != nullptr && dparams != nullptr,
              "pepnet_gate_bwd: need grid >= 1 and the partials / dparams buffers");
  tzk_pepnet::gate_bwd(*args_host, grid, partials, dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("pepnet_gate_bwd_kernel");
  return 0;
}
