// ple_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_ple.cuh (tests/test_ple_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <math.h>
#include <stdint.h>
#define TZK_SET_MAX_SMEM(kernel, bytes) (void)(bytes)
#include "../../torcheasyrec_b200/csrc/tzk_ple.cuh"

extern "C" int64_t ple_smem_bytes(const tzk_ple_gate_args* c, int backward) {
  tzk_ple::Params a;
  if (tzk_ple::prepare(*c, a) != 0) return 0;
  return (int64_t)(backward ? tzk_ple::bwd_smem(a) : tzk_ple::fwd_smem(a));
}
extern "C" int ple_gate_fwd(const tzk_ple_gate_args* c, int grid, float* y, float* p) {
  tzk_ple::Params a;
  if (tzk_ple::prepare(*c, a) != 0) return 1;
  return tzk_ple::gate_fwd(a, grid, y, p, nullptr);
}
extern "C" int ple_gate_bwd(const tzk_ple_gate_args* c, const float* p, const float* dy, int grid, float* d_experts,
                            float* partials, float* dparams) {
  tzk_ple::Params a;
  if (tzk_ple::prepare(*c, a) != 0) return 1;
  return tzk_ple::gate_bwd(a, p, dy, grid, d_experts, partials, dparams, nullptr);
}
