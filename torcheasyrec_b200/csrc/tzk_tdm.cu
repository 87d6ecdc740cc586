// tzk_tdm.cu — C entry points of TDM's fused multi-window DIN attention (tzk_tdm.cuh).  A translation unit of its own,
// so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#include "tzk_tdm.cuh"

using namespace tzk;

#define TDM_COVER                                                                                                     \
  "description outside the kernels' cover (4 <= C <= 128 with C % 4 == 0, 1 <= Dq <= C, 1..3 attention layers of "  \
  "1..64 units, ReLU or PReLU, 1..32 windows of total length <= 256, shared memory within 227 KB, 16-B aligned rows)"

extern "C" int64_t tzk_tdm_smem_bytes(const tzk_tdm_args* args_host, int32_t backward) {
  if (args_host == nullptr) return 0;
  tzk_tdm_args a = *args_host;
  a.B = 0;                          // the shapes alone
  if (tzk_tdm::check(a, backward != 0) != 0) return 0;
  return (int64_t)tzk_tdm::smem_bytes(a, backward != 0);
}

extern "C" int tzk_tdm_fwd(const tzk_tdm_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_tdm::check(*args_host, false) == 0, "tdm_fwd: " TDM_COVER);
  TZK_REQUIRE(grid >= 1, "tdm_fwd: need grid >= 1");
  tzk_tdm::fwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("tdm_fwd_kernel");
  return 0;
}

extern "C" int tzk_tdm_bwd(const tzk_tdm_args* args_host, int32_t grid, float* partials, float* dparams,
                           tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_tdm::check(*args_host, true) == 0, "tdm_bwd: " TDM_COVER);
  TZK_REQUIRE(grid >= 1 && partials != nullptr && dparams != nullptr,
              "tdm_bwd: need grid >= 1 and the partials / dparams buffers");
  tzk_tdm::bwd(*args_host, grid, partials, dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("tdm_bwd_kernel");
  return 0;
}
