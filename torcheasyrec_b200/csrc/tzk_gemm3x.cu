// tzk_gemm3x.cu — libtzk_gemm3x.so: the wide tower layer on the tensor cores (TZK_GEMM3X=1 in dense_gemm.py).
//
// The one wide tower layer of DLRM's final MLP,
//     Y[M,64] = act(X[M,K] @ W[64,K]^T + bias)            (tzrec/modules/mlp.py:20-84, K = 784)
// as hand-written sm_90a kernels with fp32-equivalent accuracy: mma.sync m16n8k8 TF32 with the 3xTF32 split
//     x*w ~= hi(x)*hi(w) + lo(x)*hi(w) + hi(x)*lo(w),  hi = cvt.rna.tf32(v), lo = cvt.rna.tf32(v - hi),
// fed by TMA (SWIZZLE_128B boxes) through a ring of shared-memory stages guarded by mbarriers.
//
// Forward / input gradient (gemm3x_kernel, 256 threads, one 128 x BN output tile per CTA):
//   thread 0    issues the TMA loads of a K-chunk (X[128x32], W_hi / W_lo[BNx32]) STAGES chunks ahead
//   warp w      rows 16w .. 16w+15 of the tile, all BN columns: splits its X fragments into hi / lo in registers
//               (W arrives split: split_w_kernel), three MMAs per k-step, then bias, ReLU and the stores
// The tensor core's fp32 accumulation is not round-to-nearest, and the error grows with the number of accumulations
// into one register: the three products of every k-step are accumulated into fresh registers and added to the running
// sum in fp32 round-to-nearest.
//
// GPU tests: tests/test_kernels_gpu.py (test_gemm3x_kernels_match_fp64, test_wide_layer_on_tcgen05_matches_fp64);
// the same source runs on the CPU under tests/native/sm90_cpu_emu.h (tests/test_gemm3x_emu.py).
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#ifdef TZK_CPU_SHIM
#include "cuda_cpu_shim.h"      // (tests/native, -I) host execution for tests/test_gemm3x_emu.py:
#include "sm90_cpu_emu.h"       // TMA / mbarrier / mma.sync emulated from their documented semantics
#else
#include <cuda.h>
#include <cuda_runtime.h>
#define TZK_DYN_SMEM(type, name) extern __shared__ __align__(1024) type name[]   // TMA swizzled tiles
#include "tzk_launch.cuh"
#endif

namespace {
#ifndef TZK_CPU_SHIM
#include "tzk_sm90_ptx.h"
#endif

constexpr int BM = 128;          // rows per output tile
constexpr int BK = 32;           // K-chunk: 32 floats = one 128-B swizzled row
constexpr int X_BYTES = BM * BK * 4;       // 16 KB
constexpr int NUM_THREADS = 256;
// BN = output columns per tile: 64 for the forward pass (N = 64), 56 for the input-gradient pass (N = 784 = 14 x 56).
// Per stage: X | W hi | W lo, each buffer 1024-B aligned (BN x 128 B is a multiple of 1 KB for both).  Three stages
// (96 / 90 KB) leave room for two CTAs per SM.
template <int BN>
struct Cfg {
  static constexpr int W_BYTES = BN * BK * 4;
  static constexpr int STAGE_BYTES = X_BYTES + 2 * W_BYTES;
  static constexpr int STAGES = 3;
  static_assert(W_BYTES % 1024 == 0, "SWIZZLE_128B boxes need 1 KB alignment");
};

struct Params {
  const float* bias;   // [N] or NULL
  float* y;            // [M, ld_y]
  int64_t ld_y;
  int64_t M;
  int K;               // multiple of 32 after padding (TMA reads the columns past the tensor as zeros)
  int N;               // output columns (multiple of BN)
  int relu;
};

#include "tzk_tma.h"      // swz(), make_map()

template <int BN>
__global__ void __launch_bounds__(NUM_THREADS, 2)
gemm3x_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_whi,
              const __grid_constant__ CUtensorMap map_wlo, Params p) {
  constexpr int W_BYTES = Cfg<BN>::W_BYTES, STAGE_BYTES = Cfg<BN>::STAGE_BYTES, STAGES = Cfg<BN>::STAGES;
  constexpr int NT = BN / 8;                       // n8 tiles per warp
  TZK_DYN_SMEM(uint8_t, smem);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);   // [STAGES] TMA -> all warps

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n_tiles = p.N / BN;                    // n fastest: the X rows of a row tile are re-read from L2
  const int64_t m0 = (int64_t)(blockIdx.x / n_tiles) * BM;
  const int col0 = (int)(blockIdx.x % n_tiles) * BN;
  const int num_k = p.K / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) mbar_init(full + s, 1);
    fence_mbarrier_init();
  }
  __syncthreads();
  auto load = [&](int kb) {                        // thread 0 only
    uint8_t* sb = smem + (kb % STAGES) * STAGE_BYTES;
    uint64_t* bar = full + kb % STAGES;
    mbar_expect_tx(bar, X_BYTES + 2 * W_BYTES);
    tma_load_2d(sb, &map_x, bar, kb * BK, (int)m0);
    tma_load_2d(sb + X_BYTES, &map_whi, bar, kb * BK, col0);
    tma_load_2d(sb + X_BYTES + W_BYTES, &map_wlo, bar, kb * BK, col0);
  };
  if (threadIdx.x == 0)
    for (int kb = 0; kb < STAGES && kb < num_k; ++kb) load(kb);

  const int r = warp * 16 + g;                     // this lane's rows r and r + 8 (both have row % 8 == g)
  float acc[NT][4], part[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[nt][q] = 0.f;
  for (int kb = 0; kb < num_k; ++kb) {
    const int s = kb % STAGES;
    mbar_wait(full + s, (uint32_t)(kb / STAGES) & 1u);
    const float* xs = reinterpret_cast<const float*>(smem + s * STAGE_BYTES);
    const uint32_t* whi = reinterpret_cast<const uint32_t*>(smem + s * STAGE_BYTES + X_BYTES);
    const uint32_t* wlo = whi + W_BYTES / 4;
#pragma unroll
    for (int ks = 0; ks < BK / 8; ++ks) {
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) part[nt][q] = 0.f;
      const int k0 = ks * 8 + t, k1 = k0 + 4;
      const float a[4] = {xs[swz(r, k0)], xs[swz(r + 8, k0)], xs[swz(r, k1)], xs[swz(r + 8, k1)]};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ah[i] = tf32_bits(a[i]);
        al[i] = tf32_bits(a[i] - __uint_as_float(ah[i]));
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const int n = nt * 8 + g;
        const uint32_t bh[2] = {whi[swz(n, k0)], whi[swz(n, k1)]};
        const uint32_t bl[2] = {wlo[swz(n, k0)], wlo[swz(n, k1)]};
        mma_tf32(part[nt], al, bh);                // small terms first
        mma_tf32(part[nt], ah, bl);
        mma_tf32(part[nt], ah, bh);
      }
#pragma unroll
      for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[nt][q] += part[nt][q];
    }
    __syncthreads();                               // every warp is done with stage s: refill it
    if (threadIdx.x == 0 && kb + STAGES < num_k) load(kb + STAGES);
  }

  // ---- epilogue: c0/c1 row r, columns 2t, 2t+1 of the n8 tile; c2/c3 row r + 8 --------------------------------------
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int col = col0 + nt * 8 + 2 * t;
    const float b0 = p.bias ? __ldg(p.bias + col) : 0.f, b1 = p.bias ? __ldg(p.bias + col + 1) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = m0 + r + 8 * h;
      if (row >= p.M) continue;
      float2 o = make_float2(acc[nt][2 * h] + b0, acc[nt][2 * h + 1] + b1);
      if (p.relu) {
        o.x = fmaxf(o.x, 0.f);
        o.y = fmaxf(o.y, 0.f);
      }
      *reinterpret_cast<float2*>(p.y + row * p.ld_y + col) = o;
    }
  }
}

#include "tzk_wgrad3x.cuh"   // wgrad3x_kernel, wgrad_reduce_kernel

__global__ void split_w_kernel(const float* __restrict__ w, int64_t n, float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    const float h = tf32_rna(w[i]);
    hi[i] = h;
    lo[i] = tf32_rna(w[i] - h);   // exactly representable: the tensor core would truncate, not round
  }
}
}  // namespace

template <int BN>
static int launch(const CUtensorMap& mx, const CUtensorMap& mh, const CUtensorMap& ml, const Params& p, cudaStream_t st) {
  const size_t smem = (size_t)Cfg<BN>::STAGES * Cfg<BN>::STAGE_BYTES + 64;
#ifndef TZK_CPU_SHIM
  static bool configured = false;     // once per instantiation: nothing but the launch happens inside a stream capture
  if (!configured) {
    cudaFuncSetAttribute(gemm3x_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    configured = true;
  }
#endif
  const int64_t tiles = (p.M + BM - 1) / BM * (p.N / BN);
  TZK_LAUNCH((gemm3x_kernel<BN>), (unsigned)tiles, NUM_THREADS, smem, st, mx, mh, ml, p);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

// y[M,N] = act(x[M,K] @ w[N,K]^T + bias) with fp32-equivalent accuracy (3xTF32).  N = 64 (forward of the wide tower
// layer, K = 784) or a multiple of 112 (its input gradient: x = dZ [M,64], w = W^T [784,64], no bias / ReLU).
// Rows 16-B aligned, ld % 4 == 0; K columns beyond the tensor are read as zeros up to the next multiple of 32.
// w_hi / w_lo: [N, ld_w] scratch written here.
extern "C" int tzk_gemm3x(const float* x, int64_t ld_x, const float* w, int64_t ld_w, const float* bias, int64_t M,
                          int32_t N, int32_t K, int32_t relu, float* y, int64_t ld_y, float* w_hi, float* w_lo,
                          void* stream) {
  if (M <= 0 || K <= 0 || (ld_x % 4) || (ld_w % 4) || (ld_y % 4)) return 1;
  if (N != 64 && N % 112 != 0) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int BN = N == 64 ? 64 : 56;
  const int64_t nw = (int64_t)N * ld_w;
  TZK_LAUNCH((split_w_kernel), (unsigned)((nw + 255) / 256), 256, 0, st, w, nw, w_hi, w_lo);
  CUtensorMap mx, mh, ml;
  if (make_map(&mx, x, M, K, ld_x, BM) || make_map(&mh, w_hi, N, K, ld_w, BN) || make_map(&ml, w_lo, N, K, ld_w, BN))
    return 2;
  Params p;
  p.bias = bias; p.y = y; p.ld_y = ld_y; p.M = M; p.K = (K + BK - 1) / BK * BK; p.N = N; p.relu = relu;
  return BN == 64 ? launch<64>(mx, mh, ml, p, st) : launch<56>(mx, mh, ml, p, st);
}

// dw[64, K] = dz[M, 64]^T @ x[M, K]  (3xTF32; fixed-order reduction over `slabs` row slabs -> run-to-run deterministic).
// partial: scratch of slabs * ceil(K/128)*128 * 64 floats.
extern "C" int64_t tzk_wgrad3x_partial_floats(int32_t K, int32_t slabs) {
  return (int64_t)slabs * ((K + 127) / 128 * 128) * 64;
}
extern "C" int tzk_wgrad3x(const float* x, int64_t ld_x, const float* dz, int64_t ld_dz, int64_t M, int32_t K,
                           int32_t slabs, float* partial, float* dw, int64_t ld_dw, void* stream) {
  if (M <= 0 || K <= 0 || slabs <= 0 || (ld_x % 4) || (ld_dz % 4)) return 1;
  CUtensorMap mx[WG_SRC], mz;
  if (make_map(&mx[0], x, M, K, ld_x, WG_ROWS) || make_map(&mz, dz, M, 64, ld_dz, WG_ROWS)) return 2;
  mx[1] = mx[2] = mx[0];
  const int boxes = (K + 31) / 32, none = 1 << 20;     // one source: every box, K columns
  const WgSources src = {{0, none, none, boxes}, {0, 0, 0}, {0, 0, 0}, {K, 0, 0}};
  return wgrad3x_launch(mx, mz, src, M, slabs, partial, dw, ld_dw, reinterpret_cast<cudaStream_t>(stream));
}
