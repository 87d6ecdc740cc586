// wukong_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_wukong.cuh (tests/test_wukong_cpu.py).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <stdint.h>
#include "../../torcheasyrec_b200/csrc/tzk_wukong.cuh"

extern "C" int wk_mix_fwd(const float* x, const float* wf, const float* gf, const float* bf, const float* wl,
                          const float* wr, int64_t B, int n, int d, int k, int f, int l, int grid, float* ln_f,
                          float* stats, float* base) {
  return tzk_wukong::mix_fwd(x, wf, gf, bf, wl, wr, B, n, d, k, f, l, grid, ln_f, stats, base, nullptr);
}
extern "C" int wk_mix_bwd(const float* x, const float* wf, const float* gf, const float* wl, const float* wr,
                          const float* stats, const float* d_ln_f, const float* d_base, int64_t B, int n, int d, int k,
                          int f, int l, int grid, float* dx, float* partials, float* dparams) {
  return tzk_wukong::mix_bwd(x, wf, gf, wl, wr, stats, d_ln_f, d_base, B, n, d, k, f, l, grid, dx, partials, dparams,
                             nullptr);
}
extern "C" int wk_out_fwd(const float* fmb, const float* base, const float* g, const float* b, int64_t B, int d, int f,
                          int l, int grid, float* y, float* stats) {
  return tzk_wukong::out_fwd(fmb, base, g, b, B, d, f, l, grid, y, stats, nullptr);
}
extern "C" int wk_out_bwd(const float* fmb, const float* base, const float* g, const float* stats, const float* dy,
                          int64_t B, int d, int f, int l, int grid, float* d_fmb, float* d_base, float* partials,
                          float* dparams) {
  return tzk_wukong::out_bwd(fmb, base, g, stats, dy, B, d, f, l, grid, d_fmb, d_base, partials, dparams, nullptr);
}
