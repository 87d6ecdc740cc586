// binned_auc_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_metrics.cuh (tests/test_binned_auc_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_metrics.cuh"

extern "C" int tzk_auc_run(const void* pred, int pred_dtype, const void* label, int label_dtype, int64_t n,
                           const float* thr, int T, int64_t* counts, int64_t* invalid) {
  return tzk_auc::run(pred, pred_dtype, label, label_dtype, n, thr, T, counts, invalid, nullptr);
}
extern "C" int tzk_auc_fits_shared(int T) { return tzk_auc::fits_shared(T) ? 1 : 0; }
