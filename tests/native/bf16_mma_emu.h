// bf16_mma_emu.h — host emulation of what tzk_interact_bf16.cuh takes from its includer, for the CPU tests only.  Goes
// with cuda_cpu_shim.h (one std::thread per CUDA thread).
//
//   bf16_rn / pack_bf16x2   float -> bf16 with round-to-nearest-even (cvt.rn.bf16.f32 / __floats2bfloat162_rn; NaN is
//                           kept a quiet NaN); pack_bf16x2(lo, hi) puts `lo` in the low 16 bits.
//   mma_bf16                mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 with the fragment layouts of the PTX ISA
//                           (g = lane / 4, t = lane % 4; element pairs in one register: lower column / row index in the
//                           low half):  A 16x16  a0 (row g, k 2t..2t+1), a1 (row g+8, k 2t..2t+1), a2 (row g, k 2t+8..2t+9),
//                           a3 (row g+8, k 2t+8..2t+9);  B 16x8  b0 (k 2t..2t+1, column g), b1 (k 2t+8..2t+9, column g);
//                           C 16x8  c0/c1 (row g, columns 2t, 2t+1), c2/c3 (row g+8).  Products of bf16 values are exact
//                           in fp32; the 16 of them are summed in k order in fp32 onto c (the hardware's internal
//                           order and precision are not specified; the tests allow for that).  Every lane of the warp
//                           must make the call.
#pragma once
#include <cstdint>
#include <cstring>

struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };

namespace tzk_ib16 {
inline uint16_t bf16_rn(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  if ((u & 0x7fffffffu) > 0x7f800000u) return (uint16_t)((u >> 16) | 0x40u);   // NaN
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
inline uint32_t pack_bf16x2(float lo, float hi) { return (uint32_t)bf16_rn(lo) | ((uint32_t)bf16_rn(hi) << 16); }
inline float bf16_half(uint32_t reg, int hi) { return __uint_as_float(hi ? (reg & 0xffff0000u) : (reg << 16)); }

inline void mma_bf16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  unsigned A[4][32], Bv[2][32];
  for (int q = 0; q < 4; ++q) tzk_shim::warp_allgather(a[q], A[q]);
  for (int q = 0; q < 2; ++q) tzk_shim::warp_allgather(b[q], Bv[q]);
  const int lane = (int)tzk_shim::t_lane, g = lane >> 2, t = lane & 3;
  for (int q = 0; q < 4; ++q) {
    const int row = g + 8 * (q >> 1), col = 2 * t + (q & 1);
    float s = c[q];
    for (int k = 0; k < 16; ++k) {
      // A[row][k]: lane (row % 8) * 4 + (k % 8) / 2, register (row / 8) + 2 * (k / 8), half k % 2
      const float av = bf16_half(A[(row >> 3) + 2 * (k >> 3)][(row & 7) * 4 + ((k & 7) >> 1)], k & 1);
      // B[k][col]: lane col * 4 + (k % 8) / 2, register k / 8, half k % 2
      const float bv = bf16_half(Bv[k >> 3][col * 4 + ((k & 7) >> 1)], k & 1);
      s += av * bv;
    }
    c[q] = s;
  }
}
}  // namespace tzk_ib16
