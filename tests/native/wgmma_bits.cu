// wgmma_bits.cu — one k8 step through tzk_wgmma.cuh's wgmma (A from registers, B by descriptor from a SWIZZLE_128B box)
// next to the same products through mma.sync m16n8k8, for tests/test_wgmma_bits_gpu.py.  One CTA (one warpgroup) per
// operand set; set s uses k-step s % 4 of its 32-column B box and scale-d = s % 2 for variant 0.
//   variant 0  D = (scale-d ? C : 0) + A_hi B_hi
//   variant 1  D = A_lo B_hi + A_hi B_lo + A_hi B_hi from a fresh accumulator (the 3xTF32 k-step of the wide layer)
// a [sets, 64, 8], b [sets, N, 32], c [sets, 64, N]; out_* [sets, 2, 64, N].
#include <cuda.h>
#include <stdint.h>

namespace {
#include "tzk_sm90_ptx.h"
#include "tzk_tma.h"
#include "tzk_wgmma.cuh"

template <int N>
__global__ void __launch_bounds__(128) wgmma_bits_kernel(const float* a, const float* b, const float* c, float* out_wg,
                                                          float* out_mma) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint32_t* bh = reinterpret_cast<uint32_t*>(smem);
  uint32_t* bl = bh + N * 32;
  const int set = blockIdx.x, ks = set & 3;
  const bool scale_d = set & 1;
  const float* bs = b + (size_t)set * N * 32;
  for (int i = threadIdx.x; i < N * 32; i += 128) {
    const uint32_t h = tf32_bits(bs[i]);
    bh[swz(i / 32, i % 32)] = h;
    bl[swz(i / 32, i % 32)] = tf32_bits(bs[i] - __uint_as_float(h));
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic stores -> wgmma's reads
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3, r = warp * 16 + g;
  const float* as = a + (size_t)set * 64 * 8;
  const float av[4] = {as[r * 8 + t], as[(r + 8) * 8 + t], as[r * 8 + t + 4], as[(r + 8) * 8 + t + 4]};
  uint32_t ah[4], al[4];
  for (int i = 0; i < 4; ++i) {
    ah[i] = tf32_bits(av[i]);
    al[i] = tf32_bits(av[i] - __uint_as_float(ah[i]));
  }
  const float* cs = c + (size_t)set * 64 * N;
  float d0[N / 2], d1[N / 2], m0[N / 2], m1[N / 2];
  for (int i = 0; i < N / 8; ++i)
    for (int q = 0; q < 4; ++q) {
      const float cv = cs[(r + 8 * (q >> 1)) * N + 8 * i + 2 * t + (q & 1)];
      d0[4 * i + q] = cv;
      m0[4 * i + q] = scale_d ? cv : 0.f;
      d1[4 * i + q] = m1[4 * i + q] = 0.f;
    }

  wgmma_fence();
  wgmma_tf32<N>(d0, ah, wgmma_desc(bh, ks), scale_d);
  wgmma_3xtf32<N>(d1, ah, al, wgmma_desc(bh, ks), wgmma_desc(bl, ks));
  wgmma_commit();
  wgmma_wait<0>();
  for (int i = 0; i < N / 2; ++i) {
    wgmma_reg_fence(d0[i]);
    wgmma_reg_fence(d1[i]);
  }

  for (int i = 0; i < N / 8; ++i) {
    const int n = 8 * i + g, k0 = ks * 8 + t, k1 = k0 + 4;
    const uint32_t fh[2] = {bh[swz(n, k0)], bh[swz(n, k1)]};
    const uint32_t fl[2] = {bl[swz(n, k0)], bl[swz(n, k1)]};
    float c0[4], c1[4];
    for (int q = 0; q < 4; ++q) {
      c0[q] = m0[4 * i + q];
      c1[q] = m1[4 * i + q];
    }
    mma_tf32(c0, ah, fh);
    mma_tf32(c1, al, fh);
    mma_tf32(c1, ah, fl);
    mma_tf32(c1, ah, fh);
    for (int q = 0; q < 4; ++q) {
      m0[4 * i + q] = c0[q];
      m1[4 * i + q] = c1[q];
    }
  }

  float* ow = out_wg + (size_t)set * 2 * 64 * N;
  float* om = out_mma + (size_t)set * 2 * 64 * N;
  for (int i = 0; i < N / 8; ++i)
    for (int q = 0; q < 4; ++q) {
      const int e = (r + 8 * (q >> 1)) * N + 8 * i + 2 * t + (q & 1);
      ow[e] = d0[4 * i + q];
      ow[64 * N + e] = d1[4 * i + q];
      om[e] = m0[4 * i + q];
      om[64 * N + e] = m1[4 * i + q];
    }
}
}  // namespace

extern "C" int wgmma_bits(const float* a, const float* b, const float* c, int sets, int n, float* out_wg,
                          float* out_mma) {
  const size_t smem = 2 * (size_t)n * 128 + 1024;
  if (n == 64)
    wgmma_bits_kernel<64><<<sets, 128, smem>>>(a, b, c, out_wg, out_mma);
  else
    return 1;
  return cudaDeviceSynchronize() == cudaSuccess ? 0 : 2;
}
