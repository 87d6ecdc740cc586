// pepnet_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_pepnet.cuh (tests/test_pepnet_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <math.h>
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_pepnet.cuh"

extern "C" int pepnet_check(const tzk_pepnet_gate_args* a, int backward) { return tzk_pepnet::check(*a, backward); }
extern "C" int pepnet_gate_fwd(const tzk_pepnet_gate_args* a, int grid) { return tzk_pepnet::gate_fwd(*a, grid, nullptr); }
extern "C" int pepnet_gate_bwd(const tzk_pepnet_gate_args* a, int grid, float* partials, float* dparams) {
  return tzk_pepnet::gate_bwd(*a, grid, partials, dparams, nullptr);
}
