// interact_bf16_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_interact_bf16.cuh for
// tests/test_mixed_precision_cpu.py: the kernels' SOURCE runs on std::threads (cuda_cpu_shim.h) with the emulated
// mma.sync.m16n8k16 bf16 and round-to-nearest-even conversions of bf16_mma_emu.h.  Checks which lane owns what and the
// rounding points before the kernels meet a GPU; says nothing about speed.
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include "bf16_mma_emu.h"

#include "../../torcheasyrec_b200/csrc/tzk_interact_bf16.cuh"

extern "C" int tzk_ib16_fwd(const uint16_t* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t B,
                            uint16_t* out, int64_t ld_out, int grid) {
  TZK_LAUNCH((tzk_ib16::dot_interact27_fwd_bf16_kernel), grid, tzk_ib16::kWarps * 32, tzk_ib16::fwd_smem(), nullptr,
             dense, ld_dense, sparse, ld_sparse, B, out, ld_out);
  return 0;
}

extern "C" int tzk_ib16_bwd(const uint16_t* d_out, int64_t ld_dout, const uint16_t* dense, int64_t ld_dense,
                            const float* sparse, int64_t ld_sparse, int64_t B, uint16_t* d_dense, int64_t ld_ddense,
                            float* d_sparse, int64_t ld_dsparse, int grid) {
  TZK_LAUNCH((tzk_ib16::dot_interact27_bwd_bf16_kernel), grid, tzk_ib16::kWarps * 32, tzk_ib16::bwd_smem(), nullptr,
             dense, ld_dense, sparse, ld_sparse, d_out, ld_dout, B, d_dense, ld_ddense, d_sparse, ld_dsparse);
  return 0;
}
