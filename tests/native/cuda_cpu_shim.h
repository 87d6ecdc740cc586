// cuda_cpu_shim.h — compile a plain CUDA kernel (no PTX, no warp intrinsics) with g++ and run it on the host, one
// std::thread per CUDA thread, one block at a time, __syncthreads() as a real barrier.
//
// TEST INFRASTRUCTURE (there is no GPU in the build container): it lets
// tests/test_tower_bwd2_cpu.py, tests/test_peer_exchange_model.py and tests/test_gemm3x_emu.py execute the kernels' actual source — index arithmetic, guards, reduction
// order — against numpy before their first contact with hardware.  It says nothing about performance, memory
// ordering or anything that needs PTX, and the product (libtzk.so) never sees it.
//
// A kernel source opts in with
//     #ifdef TZK_CPU_SHIM
//     #include "cuda_cpu_shim.h"
//     #else
//     #include <cuda_runtime.h>
//     #endif
// declares dynamic shared memory with TZK_DYN_SMEM(type, name) and launches with
//     TZK_LAUNCH((kernel<targs>), grid, block, smem_bytes, stream, args...);
#pragma once
#include <barrier>
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <thread>
#include <vector>

struct float4 { float x, y, z, w; };
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
struct float2 { float x, y; };
inline float2 make_float2(float x, float y) { return float2{x, y}; }
struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
typedef void* cudaStream_t;
typedef int cudaError_t;
constexpr int cudaSuccess = 0;
constexpr int cudaDevAttrMultiProcessorCount = 16;
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
inline cudaError_t cudaGetDevice(int* d) { *d = 0; return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int* v, int, int) { *v = 132; return cudaSuccess; }

namespace tzk_shim {
inline thread_local dim3 t_thread, t_block, t_bdim, t_gdim;
inline thread_local std::barrier<>* t_bar = nullptr;   // per emulated thread: launches may run concurrently
inline thread_local unsigned char* t_dyn = nullptr;
inline thread_local std::barrier<>* t_wbar = nullptr;  // the thread's warp (32 consecutive linear thread ids)
struct WarpSlots { unsigned long long v[32]; unsigned n; };
inline thread_local WarpSlots* t_wslots = nullptr;     // exchange area of the thread's warp (shuffles, ballots)
inline thread_local unsigned t_lane = 0;

template <class Body>
void launch(dim3 grid, dim3 block, size_t smem, Body body) {
  std::vector<unsigned char> dyn(smem + 128);
  unsigned char* base = dyn.data() + (128 - reinterpret_cast<uintptr_t>(dyn.data()) % 128) % 128;
  const unsigned n = block.x * block.y * block.z;
  for (unsigned bz = 0; bz < grid.z; ++bz)
    for (unsigned by = 0; by < grid.y; ++by)
      for (unsigned bx = 0; bx < grid.x; ++bx) {
        std::barrier<> bar(n);
        std::vector<std::unique_ptr<std::barrier<>>> warps;
        std::vector<WarpSlots> wslots((n + 31) / 32);
        for (unsigned w = 0; w * 32 < n; ++w) {
          warps.emplace_back(new std::barrier<>(n - w * 32 < 32 ? n - w * 32 : 32));
          wslots[w].n = n - w * 32 < 32 ? n - w * 32 : 32;
        }
        std::vector<std::thread> threads;
        threads.reserve(n);
        for (unsigned t = 0; t < n; ++t)
          threads.emplace_back([&, t] {
            t_thread = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
            t_block = dim3(bx, by, bz);
            t_bdim = block;
            t_gdim = grid;
            t_bar = &bar;
            t_dyn = base;
            t_wbar = warps[t / 32].get();
            t_wslots = &wslots[t / 32];
            t_lane = t % 32;
            body();
            bar.arrive_and_drop();   // a thread that returned early must not strand the others at a barrier
            t_wbar->arrive_and_drop();
          });
        for (auto& th : threads) th.join();
      }
}
}  // namespace tzk_shim

#define threadIdx tzk_shim::t_thread
#define blockIdx tzk_shim::t_block
#define blockDim tzk_shim::t_bdim
#define gridDim tzk_shim::t_gdim
#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __grid_constant__
#define __align__(n) alignas(n)
#define __shared__ static
#define __syncthreads() tzk_shim::t_bar->arrive_and_wait()
#define __syncwarp() tzk_shim::t_wbar->arrive_and_wait()
template <class T> inline T __ldg(const T* p) { return *p; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
// ---- warp intrinsics: every live lane of the warp must make the call (the kernels here use full-warp collectives) ----
namespace tzk_shim {
template <class T> inline T warp_exchange(T v, unsigned src_lane, bool take) {
  static_assert(sizeof(T) <= 8, "shuffle of a type wider than 64 bits");
  unsigned long long raw = 0;
  memcpy(&raw, &v, sizeof(T));
  t_wslots->v[t_lane] = raw;
  t_wbar->arrive_and_wait();
  T out = v;
  if (take && src_lane < t_wslots->n) memcpy(&out, &t_wslots->v[src_lane], sizeof(T));
  t_wbar->arrive_and_wait();
  return out;
}
}  // namespace tzk_shim
template <class T> inline T __shfl_sync(unsigned, T v, int src, int width = 32) {
  const unsigned base = tzk_shim::t_lane / width * width;
  return tzk_shim::warp_exchange(v, base + (unsigned)(src % width), true);
}
template <class T> inline T __shfl_up_sync(unsigned, T v, unsigned d, int width = 32) {
  const unsigned in = tzk_shim::t_lane % width;
  return tzk_shim::warp_exchange(v, tzk_shim::t_lane - d, in >= d);
}
template <class T> inline T __shfl_down_sync(unsigned, T v, unsigned d, int width = 32) {
  const unsigned in = tzk_shim::t_lane % width;
  return tzk_shim::warp_exchange(v, tzk_shim::t_lane + d, in + d < (unsigned)width);
}
template <class T> inline T __shfl_xor_sync(unsigned, T v, int m, int width = 32) {
  (void)width;
  return tzk_shim::warp_exchange(v, tzk_shim::t_lane ^ (unsigned)m, true);
}
inline unsigned __ballot_sync(unsigned, int pred) {
  tzk_shim::t_wslots->v[tzk_shim::t_lane] = pred ? 1ull : 0ull;
  tzk_shim::t_wbar->arrive_and_wait();
  unsigned m = 0;
  for (unsigned l = 0; l < tzk_shim::t_wslots->n; ++l) m |= (unsigned)tzk_shim::t_wslots->v[l] << l;
  tzk_shim::t_wbar->arrive_and_wait();
  return m;
}
inline int __popc(unsigned x) { return __builtin_popcount(x); }
namespace tzk_shim {
// every live lane of the warp contributes one 32-bit value and reads all of them (building block of the emulated mma)
inline void warp_allgather(unsigned v, unsigned (&out)[32]) {
  t_wslots->v[t_lane] = v;
  t_wbar->arrive_and_wait();
  for (unsigned l = 0; l < 32; ++l) out[l] = l < t_wslots->n ? (unsigned)t_wslots->v[l] : 0u;
  t_wbar->arrive_and_wait();
}
}  // namespace tzk_shim
template <class T> inline T atomicAdd(T* p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
template <class T> inline T atomicOr(T* p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }
template <class T> inline T atomicMax(T* p, T v) {
  T old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (old < v && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
  return old;
}
inline void __threadfence() {}
inline void __threadfence_system() {}
#define TZK_DYN_SMEM(type, name) type* name = reinterpret_cast<type*>(tzk_shim::t_dyn)
#define TZK_UNPAREN(...) __VA_ARGS__
#define TZK_LAUNCH(kernel, grid, block, smem, stream, ...) \
  tzk_shim::launch(dim3(grid), dim3(block), (smem), [&] { TZK_UNPAREN kernel(__VA_ARGS__); })
