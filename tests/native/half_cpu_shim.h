// half_cpu_shim.h — the IEEE binary16 type of cuda_fp16.h for kernel sources compiled for the host under TZK_CPU_SHIM
// (next to cuda_cpu_shim.h, which has no half type).
//
// TEST INFRASTRUCTURE: `__half` is the 16 stored bits; __half2float widens exactly (normals, subnormals, +-0, inf, NaN
// with its payload), as the FP16 table kernels do on the GPU before they compute in fp32.
#pragma once
#include <cstdint>
#include <cstring>

struct __half {
  uint16_t x;
};

inline float __half2float(__half h) {
  const uint32_t sign = (uint32_t)(h.x & 0x8000u) << 16;
  uint32_t exp = (h.x >> 10) & 0x1fu, man = h.x & 0x3ffu, bits;
  if (exp == 0x1fu) {
    bits = sign | 0x7f800000u | (man << 13);                   // inf / NaN
  } else if (exp == 0) {
    if (man == 0) {
      bits = sign;                                             // +-0
    } else {                                                   // subnormal: man * 2^-24, normalised
      int e = -1;
      do { man <<= 1; ++e; } while (!(man & 0x400u));
      bits = sign | ((uint32_t)(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
    }
  } else {
    bits = sign | ((exp + 127 - 15) << 23) | (man << 13);
  }
  float f;
  memcpy(&f, &bits, 4);
  return f;
}
