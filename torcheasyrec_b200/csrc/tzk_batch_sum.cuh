// tzk_batch_sum.cuh — the batch sums of the dense models' fused kernels (tzk_wukong.cuh, tzk_masknet.cuh, tzk_ple.cuh,
// tzk_pepnet.cuh), and the block-level helpers they share.
//
// A weight, gamma, beta or bias gradient is a sum over the batch.  Every CTA of a backward kernel adds its own samples
// in a fixed order and writes its share as one row of a partials buffer [slices][G][P]; reduce() then adds the G rows
// of each slice in CTA order.  No float atomics: the sums depend only on the grid, which the host derives from B, the
// shapes and the SM count (kernels.CudaKernels._grid), so a replayed graph gives the eager step's bits.
//
// Plain CUDA (no PTX): compiles under nvcc and under tests/native/cuda_cpu_shim.h.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "tzk_launch.cuh"

namespace tzk_batch_sum {

// out[s, e] = sum over g = 0..G-1 of partials[s][g][e], accumulated from 0 in row order; blockIdx.y = s.
// static: every translation unit that includes this header gets its own copy of the kernel (no duplicate symbols).
static __global__ void __launch_bounds__(256) reduce_kernel(const float* __restrict__ partials, int G, int64_t P,
                                                            float* __restrict__ out) {
  const int64_t e = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (e >= P) return;
  const float* p = partials + (int64_t)blockIdx.y * G * P;
  float acc = 0.f;
  for (int g = 0; g < G; ++g) acc += p[(int64_t)g * P + e];
  out[(int64_t)blockIdx.y * P + e] = acc;
}

// out [slices][P] = the row-order sum of the G rows of each slice of partials [slices][G][P].  G = 0 (an empty batch,
// no backward launch before it) writes zeros and reads no partials.
static inline void reduce(const float* partials, int G, int64_t P, int slices, float* out, cudaStream_t stream) {
  TZK_LAUNCH((reduce_kernel), dim3((unsigned)((P + 255) / 256), (unsigned)slices), 256, 0, stream, partials, G, P, out);
}

// sums over the CTA of kWarps warps in a fixed order (xor butterfly in each warp, then the warps in order); every
// thread gets both totals.  s_red: 2 kWarps floats of shared memory.  Two barriers.
template <int kWarps>
__device__ __forceinline__ void block_sum2(float& a, float& b, float* s_red) {
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x / 32;
  if (threadIdx.x % 32 == 0) {
    s_red[w] = a;
    s_red[kWarps + w] = b;
  }
  __syncthreads();
  a = s_red[0];
  b = s_red[kWarps];
  for (int i = 1; i < kWarps; ++i) {
    a += s_red[i];
    b += s_red[kWarps + i];
  }
  __syncthreads();
}

// A launch with more than the default 48 KB of dynamic shared memory must opt the kernel in first.
template <class K>
inline void opt_in_smem(K kernel, size_t bytes) {
#ifndef TZK_CPU_SHIM
  if (bytes > 48 * 1024) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
#else
  (void)kernel;
  (void)bytes;
#endif
}
}  // namespace tzk_batch_sum
