// Shared helpers for the tzk kernels (sm_90a only).
#pragma once
#include <stdlib.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/tzk.h"

namespace tzk {

void set_error(const char* fmt, ...);

inline cudaStream_t as_stream(tzk_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

#define TZK_CHECK_LAUNCH(name)                                                      \
  do {                                                                              \
    cudaError_t e__ = cudaGetLastError();                                           \
    if (e__ != cudaSuccess) {                                                       \
      ::tzk::set_error("%s: launch failed: %s", name, cudaGetErrorString(e__));     \
      return 2;                                                                     \
    }                                                                               \
  } while (0)

#define TZK_REQUIRE(cond, ...)        \
  do {                                \
    if (!(cond)) {                    \
      ::tzk::set_error(__VA_ARGS__);  \
      return 1;                       \
    }                                 \
  } while (0)

constexpr int kSmCountH100 = 132;   // H100 SXM

// Switches of code paths that have not been through a GPU validation pass yet: `name`=0/1 decides; unset,
// TZK_EXPERIMENTAL=1 turns them all on; otherwise they stay off.
inline bool unvalidated_switch(const char* name) {
  const char* e = getenv(name);
  if (e && (e[0] == '0' || e[0] == '1')) return e[0] == '1';
  const char* x = getenv("TZK_EXPERIMENTAL");
  return x && x[0] == '1';
}

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
__host__ __device__ inline size_t align16(size_t x) { return (x + 15) / 16 * 16; }

// 128-bit streaming loads/stores.  Table rows are random-access and re-used only through L2, so they
// bypass L1 allocation; index lists / outputs are touched once.
// (not volatile: independent row loads must be free to issue back to back — the whole point is to keep many
// 64-B requests in flight per lane group)
__device__ __forceinline__ float4 ld_row_f4(const float* p) {
  float4 r;
  asm("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}
// rows another GPU of the NVSwitch domain published (peer memory): coherent, no L1 allocation, free to issue back to back
__device__ __forceinline__ float4 ld_coh_f4(const float* p) {
  float4 r;
  asm("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
// rows that the same kernel writes back (weights / optimizer state): coherent load
__device__ __forceinline__ float4 ld_rw_f4(const float* p) {
  float4 r;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
// ---- FP16 tables (feature.proto data_type = "FP16"): rows are stored as halfs, every kernel computes in fp32 ------------
__device__ __forceinline__ float4 ld_row_h4(const __half* p) {    // 4 consecutive halfs (8 B) -> float4
  unsigned int a, b;
  asm("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
  const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&a));
  const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&b));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
}
template <typename WT> __device__ __forceinline__ float4 ld_table_f4(const WT* p);
template <> __device__ __forceinline__ float4 ld_table_f4<float>(const float* p) { return ld_row_f4(p); }
template <> __device__ __forceinline__ float4 ld_table_f4<__half>(const __half* p) { return ld_row_h4(p); }
template <typename WT> __device__ __forceinline__ float ld_table_f1(const WT* p);
template <> __device__ __forceinline__ float ld_table_f1<float>(const float* p) { return __ldg(p); }
template <> __device__ __forceinline__ float ld_table_f1<__half>(const __half* p) { return __half2float(__ldg(p)); }

__device__ __forceinline__ void st_stream_f4(float* p, const float4& v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w)
               : "memory");
}
__device__ __forceinline__ float4 f4_add(const float4& a, const float4& b) {
  return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
}
__device__ __forceinline__ float4 f4_scale(const float4& a, float s) {
  return make_float4(a.x * s, a.y * s, a.z * s, a.w * s);
}

}  // namespace tzk
