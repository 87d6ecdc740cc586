// tzk_ple.cu — C entry points of the fused gates of a PLE extraction layer (tzk_ple.cuh).  A translation unit of its
// own, so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#include "tzk_ple.cuh"

using namespace tzk;

#define PLE_PREPARE(what, params)                                                                                     \
  TZK_REQUIRE(args_host != nullptr && tzk_ple::prepare(*args_host, params) == 0,                                      \
              what ": layer outside the kernels' cover (1 <= n_gates <= 9, n_experts <= 64, 1 <= E_g <= 32 distinct " \
                   "experts, 1 <= H <= 1024, 1 <= K <= 1024, sum E_g K_g <= 20480)")

extern "C" int64_t tzk_ple_gate_smem_bytes(const tzk_ple_gate_args* args_host, int32_t backward) {
  tzk_ple::Params a;
  if (args_host == nullptr || tzk_ple::prepare(*args_host, a) != 0) return 0;
  return (int64_t)(backward ? tzk_ple::bwd_smem(a) : tzk_ple::fwd_smem(a));
}

extern "C" int tzk_ple_gate_fwd(const tzk_ple_gate_args* args_host, int32_t grid, float* y, float* p,
                                tzk_stream_t stream) {
  tzk_ple::Params a;
  PLE_PREPARE("ple_gate_fwd", a);
  TZK_REQUIRE(grid >= 1, "ple_gate_fwd: need grid >= 1");
  tzk_ple::gate_fwd(a, grid, y, p, as_stream(stream));
  TZK_CHECK_LAUNCH("ple_gate_fwd_kernel");
  return 0;
}

extern "C" int tzk_ple_gate_bwd(const tzk_ple_gate_args* args_host, const float* p, const float* dy, int32_t grid,
                                float* d_experts, float* partials, float* dparams, tzk_stream_t stream) {
  tzk_ple::Params a;
  PLE_PREPARE("ple_gate_bwd", a);
  TZK_REQUIRE(grid >= 1, "ple_gate_bwd: need grid >= 1");
  tzk_ple::gate_bwd(a, p, dy, grid, d_experts, partials, dparams, as_stream(stream));
  TZK_CHECK_LAUNCH("ple_gate_bwd_kernel");
  return 0;
}
