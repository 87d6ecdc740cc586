// wgmma_emu_standalone.cu — one warpgroup issuing one tzk_wgmma.cuh k8 step, compiled for the host with -DTZK_CPU_SHIM
// (cuda_cpu_shim.h + sm90_cpu_emu.h + sm90_wgmma_emu.h) for tests/test_wgmma_emu.py.  B is written into a SWIZZLE_128B box with tzk_tma.h's
// swz(), as a TMA load leaves it; A is gathered into mma.sync's fragment layout per warp.
//   a [64, 8], b [n, 32] (k-step ks of the box is used), c / out [64, n] row-major.
#include <stdint.h>

#include "cuda_cpu_shim.h"
#include "sm90_cpu_emu.h"
#include "sm90_wgmma_emu.h"

namespace {
#include "../../torcheasyrec_b200/csrc/tzk_tma.h"
#include "../../torcheasyrec_b200/csrc/tzk_wgmma.cuh"

template <int N>
__global__ void wgmma_emu_kernel(const float* a, const float* b, const float* c, int ks, int scale_d, float* out) {
  TZK_DYN_SMEM(uint8_t, smem);
  float* box = reinterpret_cast<float*>(smem);
  for (int i = threadIdx.x; i < N * 32; i += 128) box[swz(i / 32, i % 32)] = b[i];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, r = warp * 16 + g;
  const uint32_t af[4] = {__float_as_uint(a[r * 8 + t]), __float_as_uint(a[(r + 8) * 8 + t]),
                          __float_as_uint(a[r * 8 + t + 4]), __float_as_uint(a[(r + 8) * 8 + t + 4])};
  float d[N / 2];
  for (int i = 0; i < N / 8; ++i)
    for (int q = 0; q < 4; ++q) d[4 * i + q] = c[(r + 8 * (q >> 1)) * N + 8 * i + 2 * t + (q & 1)];
  wgmma_fence();
  wgmma_tf32<N>(d, af, wgmma_desc(box, ks), scale_d != 0);
  wgmma_commit();
  wgmma_wait<0>();
  for (int i = 0; i < N / 8; ++i)
    for (int q = 0; q < 4; ++q) out[(r + 8 * (q >> 1)) * N + 8 * i + 2 * t + (q & 1)] = d[4 * i + q];
}
}  // namespace

extern "C" int wgmma_emu(const float* a, const float* b, const float* c, int n, int ks, int scale_d, float* out) {
  const size_t smem = (size_t)n * 128;
  if (n == 8)
    TZK_LAUNCH((wgmma_emu_kernel<8>), 1, 128, smem, nullptr, a, b, c, ks, scale_d, out);
  else if (n == 32)
    TZK_LAUNCH((wgmma_emu_kernel<32>), 1, 128, smem, nullptr, a, b, c, ks, scale_d, out);
  else if (n == 64)
    TZK_LAUNCH((wgmma_emu_kernel<64>), 1, 128, smem, nullptr, a, b, c, ks, scale_d, out);
  else
    return 1;
  return 0;
}
