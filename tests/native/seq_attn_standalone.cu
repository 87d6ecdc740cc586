// seq_attn_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_seq_attn.cuh (tests/test_seq_encoders_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <math.h>
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_seq_attn.cuh"

extern "C" int seq_attn_check(const tzk_seq_attn_args* a, int backward) {
  return tzk_seq_attn::check(*a, backward != 0);
}
extern "C" int self_attn_pool_fwd(const tzk_seq_attn_args* a, int grid) { return tzk_seq_attn::fwd(*a, grid, nullptr); }
extern "C" int self_attn_pool_bwd(const tzk_seq_attn_args* a, int grid) { return tzk_seq_attn::bwd(*a, grid, nullptr); }
extern "C" int jagged_pool_fwd(const tzk_jagged_pool_args* a, int grid) { return tzk_seq_attn::pool_fwd(*a, grid, nullptr); }
extern "C" int jagged_pool_bwd(const tzk_jagged_pool_args* a, int grid) { return tzk_seq_attn::pool_bwd(*a, grid, nullptr); }
