// tower_tail_masked_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_tower_tail.cuh in both modes, with the
// workspace layout exposed (tests/test_tower_tail_masked_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <stdint.h>
#include <math.h>     // expf, fabsf, fmaxf, fmaf, log1pf as the CUDA math library names them
#include "../../torcheasyrec_b200/csrc/tzk_tower_tail.cuh"

extern "C" size_t tzk_tail_ws(int64_t M, int32_t K, int32_t N) { return tzk_tail::workspace_bytes(M, K, N); }
extern "C" size_t tzk_tail_colsum_offset(int64_t M, int32_t K, int32_t N) { return tzk_tail::colsum_offset(M, K, N); }
extern "C" int tzk_tail_run_mode(const float* y1, int64_t ld_y, const float* w1, const float* b1, const float* w2,
                                 const float* b2, const float* labels, int64_t M, int32_t K, int32_t N, float* logits,
                                 float* dy1, int64_t ld_dy, float* out, void* ws, size_t ws_bytes, int32_t mask) {
  return tzk_tail::run(y1, ld_y, w1, b1, w2, b2, labels, M, K, N, logits, dy1, ld_dy, out, ws, ws_bytes, nullptr,
                       mask != 0);
}
