// tzk_dcn_v2.cu — C entry points of DCN-v2's fused cross network (tzk_dcn_v2.cuh).  A translation unit of its own, so
// no existing kernel is recompiled by it.
#include <cuda.h>
#include "tzk_common.cuh"

namespace {
#include "tzk_sm90_ptx.h"
}  // namespace

#include "tzk_dcn_v2.cuh"

using namespace tzk;

#define DCN_V2_COVER "description outside the kernels' cover (1 <= D <= 512, 1 <= L <= 8, 1 <= r <= 64, 16-B aligned work)"

extern "C" int64_t tzk_dcn_v2_smem_bytes(const tzk_dcn_v2_args* args_host, int32_t pass) {
  if (args_host == nullptr) return 0;
  tzk_dcn_v2_args a = *args_host;
  a.B = 0;                          // the shapes alone
  if (tzk_dcn_v2::check(a, pass) != 0) return 0;
  return (int64_t)tzk_dcn_v2::smem_bytes(a, pass);
}

extern "C" int tzk_dcn_v2_fwd(const tzk_dcn_v2_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_dcn_v2::check(*args_host, 0) == 0, "dcn_v2_fwd: " DCN_V2_COVER);
  TZK_REQUIRE(grid >= 1, "dcn_v2_fwd: need grid >= 1");
  tzk_dcn_v2::fwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("dcn_v2_fwd_kernel");
  return 0;
}

extern "C" int tzk_dcn_v2_bwd_data(const tzk_dcn_v2_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_dcn_v2::check(*args_host, 1) == 0, "dcn_v2_bwd_data: " DCN_V2_COVER);
  TZK_REQUIRE(grid >= 1, "dcn_v2_bwd_data: need grid >= 1");
  tzk_dcn_v2::bwd_data(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("dcn_v2_bwd_data_kernel");
  return 0;
}

extern "C" int tzk_dcn_v2_bwd_weight(const tzk_dcn_v2_args* args_host, int32_t chunks, float* partials, float* dparams,
                                     tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_dcn_v2::check(*args_host, 2) == 0, "dcn_v2_bwd_weight: " DCN_V2_COVER);
  TZK_REQUIRE(chunks >= 1 && partials != nullptr && dparams != nullptr,
              "dcn_v2_bwd_weight: need chunks >= 1 and the partials / dparams buffers");
  tzk_dcn_v2::bwd_weight(*args_host, chunks, partials, dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("dcn_v2_bwd_weight_kernel");
  return 0;
}
