// dcn_v2_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_dcn_v2.cuh (tests/test_dcn_v2_cpu.py), with the
// mma.sync and cvt.rna.tf32 of sm90_cpu_emu.h.
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <stdint.h>
#include "sm90_cpu_emu.h"
#include "../../torcheasyrec_b200/csrc/tzk_dcn_v2.cuh"

extern "C" int dcn_v2_check(const tzk_dcn_v2_args* a, int pass) { return tzk_dcn_v2::check(*a, pass); }
extern "C" int64_t dcn_v2_work_floats(const tzk_dcn_v2_args* a) { return tzk_dcn_v2::work_floats(*a); }
extern "C" int64_t dcn_v2_param_floats(const tzk_dcn_v2_args* a) { return tzk_dcn_v2::param_floats(*a); }
extern "C" int dcn_v2_fwd(const tzk_dcn_v2_args* a, int grid) { return tzk_dcn_v2::fwd(*a, grid, nullptr); }
extern "C" int dcn_v2_bwd_data(const tzk_dcn_v2_args* a, int grid) { return tzk_dcn_v2::bwd_data(*a, grid, nullptr); }
extern "C" int dcn_v2_bwd_weight(const tzk_dcn_v2_args* a, int chunks, float* partials, float* dparams) {
  return tzk_dcn_v2::bwd_weight(*a, chunks, partials, dparams, nullptr);
}
