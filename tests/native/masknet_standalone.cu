// masknet_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_masknet.cuh (tests/test_masknet_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_masknet.cuh"

extern "C" int mn_mask_fwd(const float* e, int lde, const float* m, const float* b2, const float* g, const float* b,
                           int64_t B, int E, int nb, int grid, float* v, float* stats) {
  return tzk_masknet::mask_fwd(e, lde, m, b2, g, b, B, E, nb, grid, v, stats, nullptr);
}
extern "C" int mn_mask_bwd(const float* e, int lde, const float* m, const float* b2, const float* g, const float* b,
                           const float* stats, const float* dv, int64_t B, int E, int nb, int grid, float* dm,
                           float* de, float* partials, float* dparams) {
  return tzk_masknet::mask_bwd(e, lde, m, b2, g, b, stats, dv, B, E, nb, grid, dm, de, partials, dparams, nullptr);
}
extern "C" int mn_ffn_fwd(const float* z, const float* b3, const float* g, const float* b, int64_t B, int H, int nb,
                          int grid, float* y, float* stats) {
  return tzk_masknet::ffn_fwd(z, b3, g, b, B, H, nb, grid, y, stats, nullptr);
}
extern "C" int mn_ffn_bwd(const float* z, const float* b3, const float* g, const float* b, const float* stats,
                          const float* dy, int64_t B, int H, int nb, int grid, float* dz, float* partials,
                          float* dparams) {
  return tzk_masknet::ffn_bwd(z, b3, g, b, stats, dy, B, H, nb, grid, dz, partials, dparams, nullptr);
}
