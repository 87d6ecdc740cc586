// wgmma_bits_n32.cu — wgmma_bits.cu's comparison at n = 32 (the m64n32k8 of interact_wide_bwd_kernel), for
// tests/test_wgmma_n32_bits_gpu.py: the same kernel, operand layouts and variants, instantiated for N = 32.
#include "wgmma_bits.cu"

extern "C" int wgmma_bits_n32(const float* a, const float* b, const float* c, int sets, float* out_wg, float* out_mma) {
  wgmma_bits_kernel<32><<<sets, 128, 2 * 32 * 128 + 1024>>>(a, b, c, out_wg, out_mma);
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
}
