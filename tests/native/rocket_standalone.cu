// rocket_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_rocket.cuh (tests/test_rocket_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <math.h>
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_rocket.cuh"

extern "C" int rocket_check(const tzk_rocket_args* a, int backward) { return tzk_rocket::check(*a, backward); }
extern "C" int rocket_head_fwd(const tzk_rocket_args* a, int grid, float* partials, float* losses) {
  return tzk_rocket::head_fwd(*a, grid, partials, losses, nullptr);
}
extern "C" int rocket_head_bwd(const tzk_rocket_args* a, const float* dlosses, const float* losses, int grid,
                               float* partials, float* dparams) {
  return tzk_rocket::head_bwd(*a, dlosses, losses, grid, partials, dparams, nullptr);
}
