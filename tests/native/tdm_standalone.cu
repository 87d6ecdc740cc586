// tdm_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_tdm.cuh (tests/test_tdm_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <math.h>
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_tdm.cuh"

extern "C" int tdm_check(const tzk_tdm_args* a, int backward) { return tzk_tdm::check(*a, backward != 0); }
extern "C" int64_t tdm_param_floats(const tzk_tdm_args* a) { return tzk_tdm::param_floats(*a); }
extern "C" int tdm_fwd(const tzk_tdm_args* a, int grid) { return tzk_tdm::fwd(*a, grid, nullptr); }
extern "C" int tdm_bwd(const tzk_tdm_args* a, int grid, float* partials, float* dparams) {
  return tzk_tdm::bwd(*a, grid, partials, dparams, nullptr);
}
