// tzk_interact_wide.cu — DLRM-Criteo's dot interaction and the first layer of its final MLP (783 -> 64) without the
// layer's input X [B, 784] or its gradient in global memory (include/tzk.h):
//   tzk_interact_wide_fwd    the interaction's pairs and the layer's output in one kernel; only the pairs are stored
//   tzk_interact_wide_bwd    the layer's input gradient turned into the interaction's input gradients in the CTA
//   tzk_interact_wide_wgrad  the layer's weight gradient with X read from the pairs, dense and sparse (tzk_wgrad3x.cuh's
//                            work items)
//
// The GEMM parts compute what tzk_gemm3x.cu computes (TMA SWIZZLE_128B boxes through mbarrier-guarded stages, the 3xTF32
// split, every k-step's three products in a fresh accumulator, added in round-to-nearest in k order).  The forward and
// the weight gradient issue each k-step as m64n64k8 warpgroup MMAs (tzk_wgmma.cuh) with B straight from shared memory:
// one wgmma k8 gives the bits of the mma.sync m16n8k8 it replaces (tests/test_wgmma_bits_gpu.py).  The input gradient
// stays on mma.sync.  The per-sample interaction is tzk_interact_tc.cuh's.  The same source runs on the CPU under
// tests/native/cuda_cpu_shim.h, sm90_cpu_emu.h and sm90_wgmma_emu.h (tests/test_interact_wide_fused.py,
// tests/test_interact_wide_fwd_fused.py).
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#ifdef TZK_CPU_SHIM
#include "cuda_cpu_shim.h"
#include "sm90_cpu_emu.h"
#include "sm90_wgmma_emu.h"
typedef void* tzk_stream_t;
#define TZK_REQUIRE(cond, ...) do { if (!(cond)) return 1; } while (0)
#define TZK_CHECK_LAUNCH(name) do {} while (0)
#else
#include <cuda.h>
#include "tzk_common.cuh"
#define TZK_DYN_SMEM(type, name) extern __shared__ __align__(1024) type name[]   // TMA swizzled tiles
#include "tzk_launch.cuh"
#endif

namespace {
#ifndef TZK_CPU_SHIM
#include "tzk_sm90_ptx.h"
#endif
#include "tzk_tma.h"
#include "tzk_wgmma.cuh"
namespace tzk_itc {      // what tzk_interact_tc.cuh expects from its includer
__device__ __forceinline__ uint32_t cvt_tf32(float x) { return tf32_bits(x); }
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) { ::mma_tf32(c, a, b); }
}  // namespace tzk_itc
#include "tzk_interact_tc.cuh"

// a float4 this kernel wrote earlier (another thread of the CTA, before a __syncthreads): through L2, not the
// read-only path
__device__ __forceinline__ float4 load_l2(const float* p) {
#ifdef TZK_CPU_SHIM
  return *reinterpret_cast<const float4*>(p);
#else
  return __ldcg(reinterpret_cast<const float4*>(p));
#endif
}

// ======================================================================================================================
// Input gradient of the wide layer fused with the backward of the DLRM interaction that produced its input (DLRM-Criteo:
// X = [351 pairs | 0 | dense 16 | sparse 416], 784 columns).  Per CTA of FB_M samples:
//   1. dX[FB_M x 784] = dZ W, in chunks of 32 columns: dZ's fragments are split once and stay in registers (K = 64), W^T
//      hi / lo chunks arrive by TMA through the stage ring; mma.sync m16n8k8 (m64n8k8 wgmma per warpgroup was slower,
//      DESIGN §8).  The pass-through columns (352 ..) are stored straight into d_dense / d_sparse; the pair columns
//      (0 .. 351) go to a shared-memory tile.  They run second so that the tile is complete when the ring drains.
//   2. per sample, one warp: S from the pair columns, dE = S E + pass-through (tzk_itc::bwd_sample), the pass-through
//      read back from d_dense / d_sparse (written by this CTA in step 1, so an L2 hit).
// dX never reaches global memory.  The MMA order and the per-k-step accumulation are gemm3x_kernel's, so dX and with it
// dE are bit for bit what gemm3x_kernel (dgrad) followed by dot_interact27_bwd_tc_kernel computes.
constexpr int FB_M = 64;                      // samples per CTA
constexpr int FB_THREADS = 512;               // 16 warps: 4 along the samples x 4 along a 32-column chunk
constexpr int FB_WARPS = FB_THREADS / 32;
constexpr int FB_CHUNKS = (tzk_itc::kRow + 31) / 32;   // 25: the last one reads W^T rows 784 .. 799 as zeros
constexpr int FB_PAIR_CHUNKS = tzk_itc::kInter / 32;   // 11: columns 0 .. 351
constexpr int FB_BOX = 32 * 128;              // one W^T box: 32 dX columns x 32 k = 4 KB
constexpr int FB_STAGE = 4 * FB_BOX;          // hi k 0..31 | hi k 32..63 | lo k 0..31 | lo k 32..63
constexpr int FB_STAGES = 3;
constexpr int FB_LDP = 360;                   // row stride of the pair tile: 8 mod 32 words -> conflict-free float2 stores
constexpr int FB_P_OFF = FB_STAGES * FB_STAGE;
constexpr int FB_S_OFF = FB_P_OFF + FB_M * FB_LDP * 4;
constexpr int FB_IJ_OFF = FB_S_OFF + FB_WARPS * 32 * tzk_itc::kSS * 4;
constexpr int FB_BAR_OFF = FB_IJ_OFF + tzk_itc::kInter * 2;
constexpr int FB_SMEM = FB_BAR_OFF + FB_STAGES * 8;    // 215 768 B: one CTA per SM

struct FbParams {
  const float* dz; int64_t ld_dz;
  const float* dense; int64_t ld_dense;
  const float* sparse; int64_t ld_sparse;
  float* d_dense; int64_t ld_ddense;
  float* d_sparse; int64_t ld_dsparse;
  int64_t M;
};

__global__ void __launch_bounds__(FB_THREADS, 1)
interact_wide_bwd_kernel(const __grid_constant__ CUtensorMap map_whi, const __grid_constant__ CUtensorMap map_wlo,
                         FbParams p) {
  TZK_DYN_SMEM(uint8_t, smem);
  float* P = reinterpret_cast<float*>(smem + FB_P_OFF);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + FB_BAR_OFF);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t m0 = (int64_t)blockIdx.x * FB_M;

  if (threadIdx.x == 0) {
    for (int s = 0; s < FB_STAGES; ++s) mbar_init(full + s, 1);
    fence_mbarrier_init();
  }
  float* S = reinterpret_cast<float*>(smem + FB_S_OFF) + warp * (32 * tzk_itc::kSS);
  unsigned short* pair_ij = reinterpret_cast<unsigned short*>(smem + FB_IJ_OFF);
  tzk_itc::init_pair_ij(pair_ij);
  for (int i = lane; i < 32 * tzk_itc::kSS; i += 32) S[i] = 0.f;   // diagonal and padding stay zero
  __syncthreads();
  // chunk c covers dX columns 32 col_chunk(c) ..: the pass-through chunks first, then the pair chunks
  auto col_chunk = [](int c) { return (c + FB_PAIR_CHUNKS) % FB_CHUNKS; };
  auto load = [&](int c) {                        // thread 0 only
    uint8_t* sb = smem + (c % FB_STAGES) * FB_STAGE;
    uint64_t* bar = full + c % FB_STAGES;
    const int n0 = col_chunk(c) * 32;
    mbar_expect_tx(bar, FB_STAGE);
    tma_load_2d(sb, &map_whi, bar, 0, n0);
    tma_load_2d(sb + FB_BOX, &map_whi, bar, 32, n0);
    tma_load_2d(sb + 2 * FB_BOX, &map_wlo, bar, 0, n0);
    tma_load_2d(sb + 3 * FB_BOX, &map_wlo, bar, 32, n0);
  };
  if (threadIdx.x == 0)
    for (int c = 0; c < FB_STAGES; ++c) load(c);

  // A = dZ rows r, r + 8 of this warp's 16, all 64 columns, split once (rows past M are zeros)
  const int wm = warp & 3, wn = warp >> 2;
  const int r = wm * 16 + g;
  uint32_t ah[8][4], al[8][4];
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const int k0 = kk * 8 + t, k1 = k0 + 4;
    const int64_t ra = m0 + r, rb = ra + 8;
    const float a[4] = {ra < p.M ? __ldg(p.dz + ra * p.ld_dz + k0) : 0.f, rb < p.M ? __ldg(p.dz + rb * p.ld_dz + k0) : 0.f,
                        ra < p.M ? __ldg(p.dz + ra * p.ld_dz + k1) : 0.f, rb < p.M ? __ldg(p.dz + rb * p.ld_dz + k1) : 0.f};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      ah[kk][i] = tf32_bits(a[i]);
      al[kk][i] = tf32_bits(a[i] - __uint_as_float(ah[kk][i]));
    }
  }
  const int n = wn * 8 + g;                       // this lane's B column (W^T row) within the chunk
  for (int c = 0; c < FB_CHUNKS; ++c) {
    const int s = c % FB_STAGES;
    mbar_wait(full + s, (uint32_t)(c / FB_STAGES) & 1u);
    const uint32_t* whi = reinterpret_cast<const uint32_t*>(smem + s * FB_STAGE);
    const uint32_t* wlo = whi + 2 * FB_BOX / 4;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int kk = 0; kk < 8; ++kk) {
      const uint32_t* bh_box = whi + (kk >> 2) * (FB_BOX / 4);
      const uint32_t* bl_box = wlo + (kk >> 2) * (FB_BOX / 4);
      const int k0 = (kk & 3) * 8 + t, k1 = k0 + 4;
      const uint32_t bh[2] = {bh_box[swz(n, k0)], bh_box[swz(n, k1)]};
      const uint32_t bl[2] = {bl_box[swz(n, k0)], bl_box[swz(n, k1)]};
      float part[4] = {0.f, 0.f, 0.f, 0.f};
      mma_tf32(part, al[kk], bh);                 // small terms first
      mma_tf32(part, ah[kk], bl);
      mma_tf32(part, ah[kk], bh);
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[q] += part[q];
    }
    // c0/c1: row r, columns col, col + 1; c2/c3: row r + 8
    const int col = col_chunk(c) * 32 + wn * 8 + 2 * t;
    if (col < tzk_itc::kInter) {
      *reinterpret_cast<float2*>(P + r * FB_LDP + col) = make_float2(acc[0], acc[1]);
      *reinterpret_cast<float2*>(P + (r + 8) * FB_LDP + col) = make_float2(acc[2], acc[3]);
    } else if (col < tzk_itc::kRow) {
      const int e = col - tzk_itc::kInter;        // column of [dense 16 | sparse 416]
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = m0 + r + 8 * h;
        if (row >= p.M) continue;
        float* dst = e < tzk_itc::kD ? p.d_dense + row * p.ld_ddense + e : p.d_sparse + row * p.ld_dsparse + (e - tzk_itc::kD);
        *reinterpret_cast<float2*>(dst) = make_float2(acc[2 * h], acc[2 * h + 1]);
      }
    }
    __syncthreads();                              // every warp is done with stage s; at the end: P and the stores
    if (threadIdx.x == 0 && c + FB_STAGES < FB_CHUNKS) load(c + FB_STAGES);
  }

  for (int i = warp; i < FB_M; i += FB_WARPS) {
    const int64_t b = m0 + i;
    if (b >= p.M) break;
    float* dd = p.d_dense + b * p.ld_ddense;
    float* ds = p.d_sparse + b * p.ld_dsparse;
    float4 pass[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int row = g + 8 * q;
      pass[q] = row == 0 ? load_l2(dd + 4 * t)
              : row < tzk_itc::kN ? load_l2(ds + (row - 1) * tzk_itc::kD + 4 * t)
              : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    tzk_itc::bwd_sample(P + i * FB_LDP, p.dense + b * p.ld_dense, p.sparse + b * p.ld_sparse, pass, pair_ij, S, dd, ds,
                        lane);
  }
}

// ======================================================================================================================
// Forward of the same layer fused with the interaction that produces its input: Y = relu(X W^T + b) with X = [351 pairs
// | 0 | dense 16 | sparse 416], and the pair columns [M, 352] (column 351 zero) for the weight gradient.  X is never
// written: 432 of its 784 columns are copies of dense / sparse.  Per CTA of FF_M samples (gemm3x_kernel<64>'s tile):
//   1. per sample, one warp: the pairs (tzk_itc::fwd_sample) -> `pairs` in global memory (the rows stay in L2).
//   2. gemm3x_kernel<64>'s k-loop over X's 25 chunks of 32 columns, on m64n64k8 wgmma.  A comes by TMA: chunks 0 .. 10
//      from `pairs` (written by this CTA in step 1: proxy fence + barrier first), 12 .. 24 from `sparse` at column
//      32 c - 368.  Chunk 11
//      straddles dense 0 .. 15 | sparse 0 .. 15: a dense box in the stage and a sparse box (column 0) in the region
//      that held step 1's staging rows; its k-steps 0, 1 read the first, 2, 3 the second.
// The pair columns have to exist before the first k-step; the other CTA on the SM (two fit) keeps the tensor cores busy
// while this one computes them.  Same k-order and per-k-step accumulation as gemm3x_kernel, so Y is bit for bit what
// dot_interact27_fwd_tc_kernel followed by gemm3x_kernel<64> computes.
constexpr int FF_M = 128;                     // samples per CTA
constexpr int FF_THREADS = 256;               // 8 warps x 16 rows, all 64 columns each
constexpr int FF_WARPS = FF_THREADS / 32;
constexpr int FF_X_BYTES = FF_M * 128;        // A box: FF_M rows x 32 floats
constexpr int FF_W_BYTES = 64 * 128;          // W hi or lo box: 64 rows x 32 floats
constexpr int FF_STAGE = FF_X_BYTES + 2 * FF_W_BYTES;
constexpr int FF_STAGES = 3;
constexpr int FF_E_OFF = FF_STAGES * FF_STAGE;          // step 1: the warps' staging rows; chunk 11: the sparse box
constexpr int FF_BAR_OFF = FF_E_OFF + FF_X_BYTES;
constexpr int FF_SMEM = FF_BAR_OFF + FF_STAGES * 8;    // 114 712 B: two CTAs per SM
static_assert(FF_WARPS * tzk_itc::kInter * 4 <= FF_X_BYTES, "staging rows overflow their region");
constexpr int FF_SPARSE0 = tzk_itc::kInter + tzk_itc::kD;   // X column of sparse column 0

struct FfParams {
  const float* dense; int64_t ld_dense;
  const float* sparse; int64_t ld_sparse;
  float* pairs; int64_t ld_pairs;
  const float* bias;
  float* y; int64_t ld_y;
  int64_t M;
};

// orders this thread's generic-proxy accesses before later async-proxy (TMA) ones: the pair rows in global memory that
// TMA reads back, the staging rows in shared memory that TMA overwrites
__device__ __forceinline__ void fence_proxy_async() {
#ifndef TZK_CPU_SHIM
  asm volatile("fence.proxy.async;" ::: "memory");
#endif
}

__global__ void __launch_bounds__(FF_THREADS, 2)
interact_wide_fwd_kernel(const __grid_constant__ CUtensorMap map_pairs, const __grid_constant__ CUtensorMap map_dense,
                         const __grid_constant__ CUtensorMap map_sparse, const __grid_constant__ CUtensorMap map_whi, const __grid_constant__ CUtensorMap map_wlo,
                         FfParams p) {
  TZK_DYN_SMEM(uint8_t, smem);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + FF_BAR_OFF);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int64_t m0 = (int64_t)blockIdx.x * FF_M;
  const int64_t m_end = p.M - m0 < FF_M ? p.M : m0 + FF_M;

  if (threadIdx.x == 0) {
    for (int s = 0; s < FF_STAGES; ++s) mbar_init(full + s, 1);
    fence_mbarrier_init();
  }
  {   // 1. warp w: samples m0 + w, m0 + w + 8, ..; the next sample's rows are requested before this one is worked on
    float* O = reinterpret_cast<float*>(smem + FF_E_OFF) + warp * tzk_itc::kInter;
    if (lane == 0) O[tzk_itc::kP] = 0.f;
    int rowbase[4];
    tzk_itc::pair_rowbase(g, rowbase);
    int64_t b = m0 + warp;
    float4 x[4];
    if (b < m_end) {
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = tzk_itc::load_x4(p.dense + b * p.ld_dense, p.sparse + b * p.ld_sparse, g + 8 * j, 4 * t);
    }
    for (; b < m_end; b += FF_WARPS) {
      float4 xn[4];
      const int64_t bn = b + FF_WARPS;
      if (bn < m_end) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          xn[j] = tzk_itc::load_x4(p.dense + bn * p.ld_dense, p.sparse + bn * p.ld_sparse, g + 8 * j, 4 * t);
      }
      tzk_itc::fwd_sample(x, rowbase, O, p.pairs + b * p.ld_pairs, lane);
      if (bn < m_end) {
#pragma unroll
        for (int j = 0; j < 4; ++j) x[j] = xn[j];
      }
    }
  }
  fence_proxy_async();
  __syncthreads();                                // the pair rows are written; the mbarriers are initialised

  auto load = [&](int c) {                        // thread 0 only
    uint8_t* sb = smem + (c % FF_STAGES) * FF_STAGE;
    uint64_t* bar = full + c % FF_STAGES;
    mbar_expect_tx(bar, c == FB_PAIR_CHUNKS ? FF_STAGE + FF_X_BYTES : FF_STAGE);
    if (c < FB_PAIR_CHUNKS) {
      tma_load_2d(sb, &map_pairs, bar, 32 * c, (int)m0);
    } else if (c == FB_PAIR_CHUNKS) {
      tma_load_2d(sb, &map_dense, bar, 0, (int)m0);
      tma_load_2d(smem + FF_E_OFF, &map_sparse, bar, 0, (int)m0);
    } else {
      tma_load_2d(sb, &map_sparse, bar, 32 * c - FF_SPARSE0, (int)m0);
    }
    tma_load_2d(sb + FF_X_BYTES, &map_whi, bar, 32 * c, 0);
    tma_load_2d(sb + FF_X_BYTES + FF_W_BYTES, &map_wlo, bar, 32 * c, 0);
  };
  if (threadIdx.x == 0)
    for (int c = 0; c < FF_STAGES; ++c) load(c);

  // 2. gemm3x_kernel<64>'s k-steps on wgmma: warpgroup w / 4 takes rows 64 (w / 4) .., m64n64k8 with A = X hi / lo from
  // registers (rows r and r + 8 of the tile) and B = the W hi / lo boxes
  const int r = warp * 16 + g;
  float acc[32], part[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int c = 0; c < FB_CHUNKS; ++c) {
    const int s = c % FF_STAGES;
    mbar_wait(full + s, (uint32_t)(c / FF_STAGES) & 1u);
    const float* xs = reinterpret_cast<const float*>(smem + s * FF_STAGE);
    const uint8_t* whi = smem + s * FF_STAGE + FF_X_BYTES;
    const uint8_t* wlo = whi + FF_W_BYTES;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const int k0 = ks * 8 + t, k1 = k0 + 4;
      // chunk 11, k-steps 2 and 3: X column 368 + j = sparse column j of the second box.  With k = 16 + j the 16-B
      // chunk index of k is j's with bit 2 set, so swz(., j) = swz(., k) ^ 16.
      const bool sp = ks >= 2 && c == FB_PAIR_CHUNKS;
      const float* as = sp ? reinterpret_cast<const float*>(smem + FF_E_OFF) : xs;
      const int x16 = sp ? 16 : 0;
      const float a[4] = {as[swz(r, k0) ^ x16], as[swz(r + 8, k0) ^ x16], as[swz(r, k1) ^ x16], as[swz(r + 8, k1) ^ x16]};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ah[i] = tf32_bits(a[i]);
        al[i] = tf32_bits(a[i] - __uint_as_float(ah[i]));
      }
      wgmma_fence();
      wgmma_3xtf32<64>(part, ah, al, wgmma_desc(whi, ks), wgmma_desc(wlo, ks));
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        wgmma_reg_fence(part[i]);
        acc[i] += part[i];
      }
    }
    __syncthreads();                              // every warpgroup is done with stage s: refill it
    if (threadIdx.x == 0 && c + FF_STAGES < FB_CHUNKS) load(c + FF_STAGES);
  }
  // acc[4 nt + q], q = 0/1: row r, columns 2t, 2t+1 of the n8 tile nt; q = 2/3: row r + 8
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int col = nt * 8 + 2 * t;
    const float b0 = p.bias ? __ldg(p.bias + col) : 0.f, b1 = p.bias ? __ldg(p.bias + col + 1) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = m0 + r + 8 * h;
      if (row >= p.M) continue;
      float2 o = make_float2(acc[4 * nt + 2 * h] + b0, acc[4 * nt + 2 * h + 1] + b1);
      o.x = fmaxf(o.x, 0.f);
      o.y = fmaxf(o.y, 0.f);
      *reinterpret_cast<float2*>(p.y + row * p.ld_y + col) = o;
    }
  }
}

// W hi / lo [64, K] (row stride K) from W [64, ld_w]
__global__ void split_w_kernel(const float* __restrict__ w, int64_t ld_w, int K, float* __restrict__ hi,
                               float* __restrict__ lo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < K * 64) {
    const float v = w[(int64_t)(i / K) * ld_w + i % K];
    const float h = tf32_rna(v);
    hi[i] = h;
    lo[i] = tf32_rna(v - h);
  }
}

#include "tzk_wgrad3x.cuh"   // the work items, partial layout, wgrad_reduce_kernel and launch of the weight gradient

// ======================================================================================================================
// The weight gradient of the fused layer: wgrad3x_kernel's work items, stages and partial layout, its k-steps on wgmma.
// TF32 wgmma takes B only K-major from shared memory and both operands arrive batch-major, so the roles swap: the
// warpgroups compute dW^T = X^T dZ, warpgroup w / 4 on X columns 64 (w / 4) .. of the tile (m64n64k8), A = X^T read from
// the boxes and split in registers, B = dZ^T hi / lo that the warps write per chunk, transposed, into two K-major
// SWIZZLE_128B boxes [64 n x 32 batch rows].  The products of a k-step are gemm3x's in its order, dZ lo X hi, dZ hi X lo,
// dZ hi X hi, and the partial block is stored as wgrad3x_kernel stores it, so dW keeps its bits.
constexpr int WW_ZT = 64 * 128;                     // one dZ^T box: 64 n rows x 32 batch rows = 8 KB

__global__ void __launch_bounds__(WG_THREADS, 2)
interact_wide_wgrad_kernel(const __grid_constant__ CUtensorMap map_x0, const __grid_constant__ CUtensorMap map_x1,
                           const __grid_constant__ CUtensorMap map_x2, const __grid_constant__ CUtensorMap map_dz,
                           WgParams p) {
  TZK_DYN_SMEM(uint8_t, smem);
  uint8_t* zt = smem + WG_STAGES * WG_STAGE;              // dZ^T hi | lo (1024-B aligned)
  uint64_t* full = reinterpret_cast<uint64_t*>(zt + 2 * WW_ZT);
  int* boxes = reinterpret_cast<int*>(full + WG_STAGES);  // as in wgrad3x_kernel

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int jt = blockIdx.x % p.k_tiles;
  const int64_t slab = blockIdx.x / p.k_tiles;
  const int64_t row0 = slab * p.slab_rows;
  const int64_t rows = (p.M - row0 < p.slab_rows) ? p.M - row0 : p.slab_rows;
  const int num_c = (int)((rows + WG_ROWS - 1) / WG_ROWS);  // rows past M are zero-filled by the TMA

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) mbar_init(full + s, 1);
    fence_mbarrier_init();
    for (int b = 0; b < 4; ++b) {
      const int box = jt * 4 + b, s = wg_source(p.src, box);
      boxes[b] = s;
      boxes[4 + b] = wg_pick(p.src.col0, s) + 32 * (box - wg_pick(p.src.first, s));
    }
  }
  __syncthreads();
  auto load = [&](int c) {                                // thread 0 only
    uint8_t* sb = smem + (c % WG_STAGES) * WG_STAGE;
    uint64_t* bar = full + c % WG_STAGES;
    const int r = (int)(row0 + (int64_t)c * WG_ROWS);
    mbar_expect_tx(bar, WG_A + WG_B);
#pragma unroll 1
    for (int b = 0; b < 4; ++b) {
      const int s = *reinterpret_cast<volatile int*>(boxes + b), col = *reinterpret_cast<volatile int*>(boxes + 4 + b);
      tma_load_2d(sb + b * WG_BOX, s == 0 ? &map_x0 : s == 1 ? &map_x1 : &map_x2, bar, col, r);
    }
#pragma unroll
    for (int b = 0; b < 2; ++b) tma_load_2d(sb + WG_A + b * WG_BOX, &map_dz, bar, b * 32, r);
  };
  if (threadIdx.x == 0)
    for (int c = 0; c < WG_STAGES && c < num_c; ++c) load(c);

  const int xc = (warp >> 2) * 64 + (warp & 3) * 16 + g; // this lane's A rows: X columns xc and xc + 8 of the tile
  const int tn = threadIdx.x & 63, tq = threadIdx.x >> 6; // transpose: n row tn, batch rows 4 tq .. and 16 + 4 tq ..
  uint32_t* zhi = reinterpret_cast<uint32_t*>(zt);
  uint32_t* zlo = zhi + WW_ZT / 4;
  float acc[32], part[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  for (int c = 0; c < num_c; ++c) {
    const int s = c % WG_STAGES;
    mbar_wait(full + s, (uint32_t)(c / WG_STAGES) & 1u);
    const float* xs = reinterpret_cast<const float*>(smem + s * WG_STAGE);
    const float* zs = reinterpret_cast<const float*>(smem + s * WG_STAGE + WG_A);
    auto at = [](const float* base, int m, int col) { return base[(col >> 5) * (WG_BOX / 4) + swz(m, col & 31)]; };
    // dZ^T (n, m) at swz(n, m): 16-B stores, the 8 lanes of a quarter-warp on the 8 chunks of a swizzle row group
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = 4 * tq + 16 * h;
      float hi[4], lo[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = at(zs, m + j, tn);
        hi[j] = tf32_rna(v);
        lo[j] = tf32_rna(v - hi[j]);
      }
      *reinterpret_cast<float4*>(zhi + swz(tn, m)) = make_float4(hi[0], hi[1], hi[2], hi[3]);
      *reinterpret_cast<float4*>(zlo + swz(tn, m)) = make_float4(lo[0], lo[1], lo[2], lo[3]);
    }
    fence_proxy_async();                                  // the generic stores before wgmma's reads
    __syncthreads();
#pragma unroll
    for (int ks = 0; ks < WG_ROWS / 8; ++ks) {
      const int m = ks * 8 + t;                           // batch rows m (a0, a1) and m + 4 (a2, a3)
      const float a[4] = {at(xs, m, xc), at(xs, m, xc + 8), at(xs, m + 4, xc), at(xs, m + 4, xc + 8)};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ah[i] = tf32_bits(a[i]);
        al[i] = tf32_bits(a[i] - __uint_as_float(ah[i]));
      }
      wgmma_fence();
      wgmma_tf32<64>(part, ah, wgmma_desc(zlo, ks), false);
      wgmma_tf32<64>(part, al, wgmma_desc(zhi, ks), true);
      wgmma_tf32<64>(part, ah, wgmma_desc(zhi, ks), true);
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        wgmma_reg_fence(part[i]);
        acc[i] += part[i];
      }
    }
    __syncthreads();                                      // stage s and the dZ^T boxes are free
    if (threadIdx.x == 0 && c + WG_STAGES < num_c) load(c + WG_STAGES);
  }
  // acc[4 i + q]: X column xc + 8 (q / 2), n = 8 i + 2 t + q % 2
  float* out = p.partial + ((int64_t)slab * p.k_tiles + jt) * 128 * 64;
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h)
      *reinterpret_cast<float2*>(out + (int64_t)(xc + 8 * h) * 64 + 8 * i + 2 * t) =
          make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
}

// W^T hi / lo [K, 64] from W [64, ld_w] (K columns used)
__global__ void split_wt_kernel(const float* __restrict__ w, int64_t ld_w, int K, float* __restrict__ hi,
                                float* __restrict__ lo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < K * 64) {
    const int k = i >> 6, o = i & 63;
    const float v = w[(int64_t)o * ld_w + k];
    const float h = tf32_rna(v);
    hi[i] = h;
    lo[i] = tf32_rna(v - h);
  }
}

}  // namespace

extern "C" int tzk_interact_wide_bwd(const float* dz, int64_t ld_dz, const float* w, int64_t ld_w, const float* dense,
                                     int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t M, float* d_dense,
                                     int64_t ld_ddense, float* d_sparse, int64_t ld_dsparse, float* wt_hi, float* wt_lo,
                                     tzk_stream_t stream) {
  TZK_REQUIRE(M > 0, "interact_wide_bwd: M must be positive");
  TZK_REQUIRE(ld_w >= tzk_itc::kRow, "interact_wide_bwd: w needs %d columns", tzk_itc::kRow);
  const int64_t lds[] = {ld_dz, ld_w, ld_dense, ld_sparse, ld_ddense, ld_dsparse};
  for (int64_t ld : lds) TZK_REQUIRE(ld % 4 == 0, "interact_wide_bwd: row strides must be multiples of 4 floats");
  const void* ptrs[] = {dz, w, dense, sparse, d_dense, d_sparse, wt_hi, wt_lo};
  for (const void* q : ptrs)
    TZK_REQUIRE(q && reinterpret_cast<uintptr_t>(q) % 16 == 0, "interact_wide_bwd: NULL or not 16-B aligned pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TZK_LAUNCH((split_wt_kernel), (tzk_itc::kRow * 64 + 255) / 256, 256, 0, st, w, ld_w, tzk_itc::kRow, wt_hi, wt_lo);
  CUtensorMap mh, ml;
  TZK_REQUIRE(!make_map(&mh, wt_hi, tzk_itc::kRow, 64, 64, 32) && !make_map(&ml, wt_lo, tzk_itc::kRow, 64, 64, 32),
              "interact_wide_bwd: tensor-map encoding failed");
  FbParams p;
  p.dz = dz; p.ld_dz = ld_dz; p.dense = dense; p.ld_dense = ld_dense; p.sparse = sparse; p.ld_sparse = ld_sparse;
  p.d_dense = d_dense; p.ld_ddense = ld_ddense; p.d_sparse = d_sparse; p.ld_dsparse = ld_dsparse; p.M = M;
#ifndef TZK_CPU_SHIM
  static bool configured = false;     // once: nothing but the launches happens inside a stream capture
  if (!configured) {
    cudaFuncSetAttribute(interact_wide_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FB_SMEM);
    configured = true;
  }
#endif
  TZK_LAUNCH((interact_wide_bwd_kernel), (unsigned)((M + FB_M - 1) / FB_M), FB_THREADS, FB_SMEM, st, mh, ml, p);
  TZK_CHECK_LAUNCH("interact_wide_bwd_kernel");
  return 0;
}

extern "C" int tzk_interact_wide_fwd(const float* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse,
                                     const float* w, int64_t ld_w, const float* bias, int64_t M, float* y, int64_t ld_y,
                                     float* pairs, int64_t ld_pairs, float* w_hi, float* w_lo, tzk_stream_t stream) {
  TZK_REQUIRE(M > 0, "interact_wide_fwd: M must be positive");
  TZK_REQUIRE(ld_w >= tzk_itc::kRow && ld_y >= 64 && ld_pairs >= tzk_itc::kInter && ld_dense >= tzk_itc::kD &&
              ld_sparse >= tzk_itc::kRow - FF_SPARSE0, "interact_wide_fwd: row stride shorter than the row");
  const int64_t lds[] = {ld_dense, ld_sparse, ld_w, ld_y, ld_pairs};
  for (int64_t ld : lds) TZK_REQUIRE(ld % 4 == 0, "interact_wide_fwd: row strides must be multiples of 4 floats");
  const void* ptrs[] = {dense, sparse, w, y, pairs, w_hi, w_lo};
  for (const void* q : ptrs)
    TZK_REQUIRE(q && reinterpret_cast<uintptr_t>(q) % 16 == 0, "interact_wide_fwd: NULL or not 16-B aligned pointer");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  TZK_LAUNCH((split_w_kernel), (tzk_itc::kRow * 64 + 255) / 256, 256, 0, st, w, ld_w, tzk_itc::kRow, w_hi, w_lo);
  CUtensorMap mp, md, ms, mh, ml;
  TZK_REQUIRE(!make_map(&mp, pairs, M, tzk_itc::kInter, ld_pairs, FF_M) &&
              !make_map(&md, dense, M, tzk_itc::kD, ld_dense, FF_M) &&
              !make_map(&ms, sparse, M, tzk_itc::kRow - FF_SPARSE0, ld_sparse, FF_M) &&
              !make_map(&mh, w_hi, 64, tzk_itc::kRow, tzk_itc::kRow, 64) &&
              !make_map(&ml, w_lo, 64, tzk_itc::kRow, tzk_itc::kRow, 64), "interact_wide_fwd: tensor-map encoding failed");
  FfParams p;
  p.dense = dense; p.ld_dense = ld_dense; p.sparse = sparse; p.ld_sparse = ld_sparse; p.pairs = pairs;
  p.ld_pairs = ld_pairs; p.bias = bias; p.y = y; p.ld_y = ld_y; p.M = M;
#ifndef TZK_CPU_SHIM
  static bool configured = false;     // once: nothing but the launches happens inside a stream capture
  if (!configured) {
    cudaFuncSetAttribute(interact_wide_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FF_SMEM);
    configured = true;
  }
#endif
  TZK_LAUNCH((interact_wide_fwd_kernel), (unsigned)((M + FF_M - 1) / FF_M), FF_THREADS, FF_SMEM, st, mp, md, ms, mh, ml, p);
  TZK_CHECK_LAUNCH("interact_wide_fwd_kernel");
  return 0;
}

extern "C" int tzk_interact_wide_wgrad(const float* dz, int64_t ld_dz, const float* pairs, int64_t ld_pairs,
                                       const float* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse,
                                       int64_t M, int32_t slabs, float* partial, float* dw, int64_t ld_dw,
                                       tzk_stream_t stream) {
  TZK_REQUIRE(M > 0 && slabs > 0, "interact_wide_wgrad: M and slabs must be positive");
  TZK_REQUIRE(ld_dw >= tzk_itc::kRow, "interact_wide_wgrad: dw needs %d columns", tzk_itc::kRow);
  const int64_t lds[] = {ld_dz, ld_pairs, ld_dense, ld_sparse};
  for (int64_t ld : lds) TZK_REQUIRE(ld % 4 == 0, "interact_wide_wgrad: row strides must be multiples of 4 floats");
  const void* ptrs[] = {dz, pairs, dense, sparse, partial, dw};
  for (const void* q : ptrs)
    TZK_REQUIRE(q && reinterpret_cast<uintptr_t>(q) % 16 == 0, "interact_wide_wgrad: NULL or not 16-B aligned pointer");
  CUtensorMap mx[WG_SRC], mz;
  TZK_REQUIRE(!make_map(&mx[0], pairs, M, tzk_itc::kInter, ld_pairs, WG_ROWS) &&
              !make_map(&mx[1], sparse, M, tzk_itc::kRow - FF_SPARSE0, ld_sparse, WG_ROWS) &&
              !make_map(&mx[2], dense, M, tzk_itc::kD, ld_dense, WG_ROWS) &&
              !make_map(&mz, dz, M, 64, ld_dz, WG_ROWS), "interact_wide_wgrad: tensor-map encoding failed");
  // boxes 0 .. 10: pairs -> X columns 0 .. 351; 11 .. 23: sparse -> 368 ..; 24 (and the tile's padding 25 .. 27,
  // past the tensor: zeros, never written): dense -> 352 .. 367
  const WgSources src = {{0, FB_PAIR_CHUNKS, FB_CHUNKS - 1, FB_CHUNKS}, {0, 0, 0}, {0, FF_SPARSE0, tzk_itc::kInter},
                         {tzk_itc::kInter, tzk_itc::kRow - FF_SPARSE0, tzk_itc::kD}};
  TZK_REQUIRE(wgrad3x_launch<interact_wide_wgrad_kernel>(mx, mz, src, M, slabs, partial, dw, ld_dw,
                                                         reinterpret_cast<cudaStream_t>(stream), 2 * WW_ZT) == 0,
              "interact_wide_wgrad: launch failed");
  return 0;
}
