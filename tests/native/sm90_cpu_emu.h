// sm90_cpu_emu.h — host emulation of the PTX used by tzk_gemm3x.cu (the functions of tzk_sm90_ptx.h), for the CPU
// tests only.  Goes with cuda_cpu_shim.h (one std::thread per CUDA thread, blocks one after another).
//
// What is emulated, from the documented semantics (PTX ISA):
//   mbarrier      arrival count + outstanding transaction bytes per phase; try_wait.parity(P) succeeds iff the
//                 current parity != P.
//   TMA 2-D load  box [32 floats x box_rows] from a row-major global tensor, out-of-bounds elements = 0, written to
//                 shared memory as 128-B rows with SWIZZLE_128B (16-B chunk index ^= bits [7,10) of the shared address),
//                 then complete_tx(box bytes) on the barrier.
//   mma.sync      m16n8k8 TF32 with the fragment layouts of the PTX ISA (A row-major 16x8: a0/a1 rows g, g+8 at
//                 column t, a2/a3 at column t+4; B 8x8: b0/b1 rows t, t+4 at column g; C 16x8: c0/c1 row g columns
//                 2t, 2t+1, c2/c3 row g+8), operands truncated to TF32; every lane of the warp must make the call.
// What is NOT emulated: timing, proxies / fences (no-ops: the mutex inside every barrier operation orders memory),
// cluster scope.  Agreement here shows that the kernels' control flow, barrier protocol, swizzled addressing and
// fragment mapping are self-consistent with these semantics — not that the semantics are right.
#pragma once
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <map>
#include <mutex>

struct CUtensorMap {            // host stand-in: what cuTensorMapEncodeTiled was told
  const float* base;
  int64_t rows, cols, ld;
  int box_rows;
};

namespace tzk_emu {
struct Bar { int count = 0, pending = 0, parity = 0; long tx = 0; };
struct Cta {                     // state of the CTA that is currently running (blocks run one at a time)
  std::mutex mu;
  std::condition_variable cv;
  std::map<uint32_t, Bar> bars;  // keyed by shared-memory offset
};
inline Cta& cta() { static Cta c; return c; }
inline void fail(const char* msg) { fprintf(stderr, "sm90 emulation: %s\n", msg); abort(); }
inline uint8_t* smem_base() { return tzk_shim::t_dyn; }
inline void maybe_flip(Bar& b) {
  if (b.pending == 0 && b.tx == 0) { b.parity ^= 1; b.pending = b.count; }
}
inline uint32_t swz(uint32_t a) { return a ^ (((a >> 7) & 7u) << 4); }   // SWIZZLE_128B on a shared-memory address
}  // namespace tzk_emu

inline uint32_t smem_u32(const void* p) {
  return (uint32_t)(reinterpret_cast<const uint8_t*>(p) - tzk_emu::smem_base());
}

// ---- mbarrier ------------------------------------------------------------------------------------------------------
inline void mbar_init(uint64_t* bar, uint32_t count) {
  auto& c = tzk_emu::cta();
  std::lock_guard<std::mutex> g(c.mu);
  tzk_emu::Bar b; b.count = b.pending = (int)count;
  c.bars[smem_u32(bar)] = b;
}
inline void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  auto& c = tzk_emu::cta();
  std::lock_guard<std::mutex> g(c.mu);
  auto& b = c.bars.at(smem_u32(bar));
  if (b.pending <= 0) tzk_emu::fail("more arrivals than the mbarrier's count (expect_tx)");
  b.tx += bytes;
  --b.pending;
  tzk_emu::maybe_flip(b);
  c.cv.notify_all();
}
inline void mbar_wait(uint64_t* bar, uint32_t parity) {
  auto& c = tzk_emu::cta();
  std::unique_lock<std::mutex> g(c.mu);
  auto& b = c.bars.at(smem_u32(bar));
  if (!c.cv.wait_for(g, std::chrono::seconds(60), [&] { return b.parity != (int)parity; }))
    tzk_emu::fail("mbarrier wait timed out (deadlock in the pipeline protocol)");
}
inline void fence_mbarrier_init() {}

// ---- TMA --------------------------------------------------------------------------------------------------------------
inline void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  const uint32_t d0 = smem_u32(dst);
  if (d0 & 1023) tzk_emu::fail("TMA destination of a SWIZZLE_128B box must be 1024-B aligned here");
  uint8_t* sm = tzk_emu::smem_base();
  for (int r = 0; r < map->box_rows; ++r)
    for (int c = 0; c < 32; ++c) {
      const int64_t gr = (int64_t)c1 + r, gc = (int64_t)c0 + c;
      const float v = (gr >= 0 && gr < map->rows && gc >= 0 && gc < map->cols) ? map->base[gr * map->ld + gc] : 0.f;
      memcpy(sm + tzk_emu::swz(d0 + (uint32_t)r * 128u + (uint32_t)c * 4u), &v, 4);
    }
  auto& ct = tzk_emu::cta();
  std::lock_guard<std::mutex> g(ct.mu);
  auto& b = ct.bars.at(smem_u32(bar));
  b.tx -= (long)map->box_rows * 128;
  if (b.tx < 0) tzk_emu::fail("complete_tx exceeds the bytes the barrier expects");
  tzk_emu::maybe_flip(b);
  ct.cv.notify_all();
}

// ---- tensor cores -------------------------------------------------------------------------------------------------------
inline uint32_t tf32_bits(float x) {      // cvt.rna.tf32.f32: round to nearest, ties away from zero
  uint32_t u;
  memcpy(&u, &x, 4);
  if (((u >> 23) & 0xff) != 0xff) u += 0x1000u;
  return u & 0xffffe000u;
}
inline float tf32_rna(float x) { return __uint_as_float(tf32_bits(x)); }

inline void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  unsigned A[4][32], Bv[2][32];
  for (int q = 0; q < 4; ++q) tzk_shim::warp_allgather(a[q], A[q]);
  for (int q = 0; q < 2; ++q) tzk_shim::warp_allgather(b[q], Bv[q]);
  const int lane = (int)tzk_shim::t_lane, g = lane >> 2, t = lane & 3;
  for (int q = 0; q < 4; ++q) {
    const int row = g + 8 * (q >> 1), col = 2 * t + (q & 1);
    float s = c[q];
    for (int k = 0; k < 8; ++k) {
      // A[row][k]: lane (row % 8) * 4 + (k % 4), register (row / 8) + 2 * (k / 4); B[k][col]: lane col * 4 + (k % 4),
      // register k / 4; the tensor core reads 10 explicit mantissa bits of each
      const float av = __uint_as_float(A[(row >> 3) + 2 * (k >> 2)][(row & 7) * 4 + (k & 3)] & 0xffffe000u);
      const float bv = __uint_as_float(Bv[k >> 2][col * 4 + (k & 3)] & 0xffffe000u);
      s += av * bv;
    }
    c[q] = s;
  }
}
