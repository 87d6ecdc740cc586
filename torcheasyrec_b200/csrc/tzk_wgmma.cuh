// tzk_wgmma.cuh — warpgroup MMA (wgmma.mma_async, sm_90a) on TF32 with A in registers and B a K-major SWIZZLE_128B
// box in shared memory: the [rows x 32 floats] boxes of tzk_tma.h, 1024-B aligned, row n at byte 128 n, 16-B chunk index
// XOR-ed with n % 8.  Included inside the includer's anonymous namespace after tzk_sm90_ptx.h (or, for the CPU tests,
// sm90_cpu_emu.h and sm90_wgmma_emu.h, which provides wgmma_fence / wgmma_commit / wgmma_wait / wgmma_tf32 as a host
// emulation) and tzk_tma.h.
//
// Fragments, per warp w of the warpgroup (g = lane / 4, t = lane % 4), those of mma.sync m16n8k8 on rows 16 w ..:
//   A (4 x b32, tf32 bits)  a0 (16w + g, t) a1 (16w + g + 8, t) a2 (16w + g, t + 4) a3 (16w + g + 8, t + 4)
//   D (N / 2 floats)        d[4 i + q]: row 16w + g + 8 (q / 2), column 8 i + 2 t + q % 2 (n8 tile i)
// so D rows 16w .. 16w + 15 depend on warp w's A registers only.  scale_d = false starts from zero (C = 0).
#pragma once

// descriptor of the k-step ks (8 floats = 32 B) of a K-major SWIZZLE_128B box: start address (>> 4, 14 bits),
// leading byte offset 1 (unused: one k-step never leaves the 128-B swizzle row), stride byte offset 1024 (8 rows of
// 128 B), base offset 0 (the box is 1024-B aligned), layout type 1 = SWIZZLE_128B in bits 62 .. 63
__device__ __forceinline__ uint64_t wgmma_desc(const void* box, int ks) {
  const uint32_t a = smem_u32(box) + 32u * (uint32_t)ks;
  return (uint64_t)((a >> 4) & 0x3fffu) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

#ifndef TZK_CPU_SHIM
// orders the warpgroup's register accesses before the wgmma.mma_async that follow (accumulators, A fragments)
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// until at most N committed groups of this warpgroup are pending; the accumulators of the others may be read
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accesses of r across a wgmma_wait
__device__ __forceinline__ void wgmma_reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// d (+)= A [64 x 8] * B [8 x N]; B's column n is row n of the box the descriptor points at
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc, bool scale_d);

template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t desc, bool scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,"
      "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"((int)scale_d));
}

template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[16], const uint32_t (&a)[4], uint64_t desc, bool scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15}, {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc), "r"((int)scale_d));
}
#endif

// One 3xTF32 k-step into a fresh accumulator, as gemm3x_kernel does it with mma.sync: lo.hi (scale-d = 0, i.e. C = 0),
// hi.lo, hi.hi, all three products of a row-column pair in one tensor-core accumulator.  lo_b / hi_b: descriptors of B's
// lo / hi boxes at this k-step.  The caller commits, waits and adds `part` to its running sum.
template <int N>
__device__ __forceinline__ void wgmma_3xtf32(float (&part)[N / 2], const uint32_t (&ah)[4], const uint32_t (&al)[4],
                                             uint64_t hi_b, uint64_t lo_b) {
  wgmma_tf32<N>(part, al, hi_b, false);
  wgmma_tf32<N>(part, ah, lo_b, true);
  wgmma_tf32<N>(part, ah, hi_b, true);
}
