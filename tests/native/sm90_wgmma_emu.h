// sm90_wgmma_emu.h — host emulation of the warpgroup MMA that tzk_wgmma.cuh issues, for the CPU tests only.  Goes with
// cuda_cpu_shim.h and sm90_cpu_emu.h (included after them: it uses their shared-memory base, SWIZZLE_128B addressing and
// warp exchange).
//
// What is emulated, from the documented semantics (PTX ISA):
//   wgmma.mma_async  m64nNk8 TF32, A from registers, B by a K-major SWIZZLE_128B shared-memory descriptor (start
//                    address, stride byte offset, layout type), scale-d.  D rows 16 w .. 16 w + 15 take warp w's A
//                    fragment, laid out as mma.sync m16n8k8's; B's element (n, k) is at start + (n / 8) * stride +
//                    (n % 8) * 128 + 4 k, swizzled as the TMA wrote it; per D element the 8 products are added to
//                    scale-d ? D : 0 in k order, as sm90_cpu_emu.h's mma_tf32 adds them.  Operands truncated to TF32.
// What is NOT emulated: the asynchrony (the product is computed when issued, so fence / commit / wait are no-ops), any
// descriptor layout but SWIZZLE_128B.
#pragma once

inline void wgmma_fence() {}
inline void wgmma_commit() {}
template <int N> inline void wgmma_wait() {}
inline void wgmma_reg_fence(float&) {}

template <int N>
inline void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc, bool scale_d) {
  static_assert(N % 8 == 0 && N >= 8 && N <= 256, "wgmma m64nNk8: N is a multiple of 8 up to 256");
  if ((desc >> 62) != 1u) tzk_emu::fail("wgmma: only the SWIZZLE_128B descriptor layout is emulated");
  if ((desc >> 49) & 7u) tzk_emu::fail("wgmma: the descriptor's base offset must be 0 (1024-B aligned box)");
  const uint32_t start = (uint32_t)(desc & 0x3fffu) << 4, sbo = (uint32_t)((desc >> 32) & 0x3fffu) << 4;
  if (start % 32u) tzk_emu::fail("wgmma: a k8 TF32 step starts on a 32-B boundary of the swizzle row");
  unsigned A[4][32];
  for (int q = 0; q < 4; ++q) tzk_shim::warp_allgather(a[q], A[q]);
  const uint8_t* sm = tzk_emu::smem_base();
  const int lane = (int)tzk_shim::t_lane, g = lane >> 2, t = lane & 3;
  for (int i = 0; i < N / 8; ++i)
    for (int q = 0; q < 4; ++q) {
      const int row = g + 8 * (q >> 1), col = 8 * i + 2 * t + (q & 1);
      float s = scale_d ? d[4 * i + q] : 0.f;
      for (int k = 0; k < 8; ++k) {
        uint32_t bu;
        memcpy(&bu, sm + tzk_emu::swz(start + (uint32_t)(col >> 3) * sbo + (uint32_t)(col & 7) * 128u + 4u * k), 4);
        const float av = __uint_as_float(A[(row >> 3) + 2 * (k >> 2)][(row & 7) * 4 + (k & 3)] & 0xffffe000u);
        s += av * __uint_as_float(bu & 0xffffe000u);
      }
      d[4 * i + q] = s;
    }
}
