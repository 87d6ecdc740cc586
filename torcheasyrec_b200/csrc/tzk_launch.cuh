// tzk_launch.cuh — the launch glue of the kernel sources: dynamic shared memory is declared with
// TZK_DYN_SMEM(type, name) and kernels are launched with TZK_LAUNCH((kernel<targs>), grid, block, smem, stream, args...).
// Under TZK_CPU_SHIM (tests/native/cuda_cpu_shim.h) the shim defines both to run the same source on the host, and this
// header stays out of the way.  A source whose kernels need a wider alignment of dynamic shared memory (the TMA
// swizzled tiles of tzk_interact_wide.cu and tzk_gemm3x.cu: 1024 B) defines TZK_DYN_SMEM before including this.
#pragma once
#ifndef TZK_CPU_SHIM
#ifndef TZK_DYN_SMEM
#define TZK_DYN_SMEM(type, name) extern __shared__ __align__(16) type name[]
#endif
#define TZK_UNPAREN(...) __VA_ARGS__
#define TZK_LAUNCH(kernel, grid, block, smem, stream, ...) TZK_UNPAREN kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif
