// tower_bwd2_standalone.cu — stand-alone build of torcheasyrec_b200/csrc/tzk_tower_bwd2.cuh (host shim tests, try script).
//
// Round-2 groundwork (DESIGN.md §9.3): the backward of the narrow tower layers (K, N <= 64) without shared-memory
// tiles and without barriers in the row loop.  Today's small_linear_bwd_kernel walks 128-row tiles through shared
// memory (load -> barrier -> dW/db -> dx -> barrier -> store -> barrier) and is latency-bound: 98 us for 64->32 at
// B = 65536 against ~10 us of HBM time and ~4 us of FFMA issue (profiles/README.md, "Narrow tower layers").
// Two kernels instead, both reading straight from global memory the way the forward small_linear_fwd_rows_kernel
// does (which is 2x faster than the library path):
//
//   small_linear_dx_rows_kernel   dx = (dy * [y > 0]) @ W         one thread per row, W broadcast from shared memory,
//                                                                 32 accumulators per pass, 16-B row stores
//   small_linear_dw_kernel        dW = dz^T @ x, db = colsum(dz)  a thread owns an NB x KB block of dW, loops over its
//                                                                 CTA's rows with U rows of independent 16-B loads in
//                                                                 flight; lanes of a warp share a dz row (broadcast)
//                                                                 and cover one x row (coalesced); row groups of a
//                                                                 CTA are folded in shared memory in a fixed order,
//                                                                 CTAs by small_linear_reduce2_kernel in CTA order.
// Same fp32 FFMA arithmetic as the library kernels; the dW summation order differs from tzk_small_linear_bwd's (rows
// interleaved over row groups), so the two agree to rounding, not bit for bit; both are run-to-run deterministic.
//
// GPU tests: tests/test_kernels_gpu.py::test_small_linear_fwd_bwd_vs_fp64_reference (both backward paths)
#ifdef TZK_CPU_SHIM
#include "cuda_cpu_shim.h"   // host execution for tests/test_tower_bwd2_cpu.py
#else
#include <cuda_runtime.h>
#include "../../torcheasyrec_b200/csrc/tzk_launch.cuh"
#endif
#include <stdint.h>

#include "../../torcheasyrec_b200/csrc/tzk_tower_bwd2.cuh"
using namespace tzk_bwd2;

extern "C" size_t tzk_small_linear_bwd2_workspace_bytes(int64_t M, int32_t K, int32_t N) {
  return workspace_bytes(M, K, N);
}

// Same contract as tzk_small_linear_bwd (include/tzk.h); 4 = shape not covered by the row-group mapping.
extern "C" int tzk_small_linear_bwd2(const float* x, int64_t ld_x, const float* w, const float* y, int64_t ld_y,
                                     const float* dy, int64_t ld_dy, int64_t M, int32_t K, int32_t N, int32_t relu,
                                     float* dx, int64_t ld_dx, float* dw, float* db, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  return run(x, ld_x, w, y, ld_y, dy, ld_dy, M, K, N, relu, dx, ld_dx, dw, db, workspace, workspace_bytes,
             reinterpret_cast<cudaStream_t>(stream));
}
