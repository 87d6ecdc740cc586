// tzk_interact_tc.cuh — DLRM dot interaction on the tensor cores (mma.sync m16n8k8, 3xTF32 split: fp32-level products),
// forward and backward, specialised for the DLRM-Criteo shape: N = 27 interacting rows (the bottom-MLP output + 26
// pooled embeddings) of D = 16 floats, output row [351 pairs | 1 zero | 16 dense | 416 sparse] = 784 floats
// (tzrec/modules/interaction.py:80-91 + tzrec/models/dlrm.py:113-131).  Every other shape keeps the FFMA kernels of
// tzk_dense.cu.
//
// One warp per sample.  The point of the layout: a lane's MMA fragments are exactly the 16-B chunks it loads.
//
//   forward   Z = X X^T (32 x 32 padded, K = 16).  Lane (g = lane / 4, t = lane % 4) loads X[g + 8 j][4 t .. 4 t + 3],
//             j = 0..3 — four coalesced 16-B loads, no shared-memory staging.  The contraction index may be permuted
//             freely as long as A and B agree: logical k of k-step ks is mapped to the physical column 4 (k % 4) + 2 ks +
//             (k / 4), so the A fragment of row block mt (rows g + 16 mt, g + 8 + 16 mt) and the B fragment of column
//             block nt (column g + 8 nt) are components of the lane's own registers.  6 of the 8 output tiles touch the
//             strict upper triangle; 6 tiles x 2 k-steps x 3 MMAs (lo*hi, hi*lo, hi*hi).  The pairs go through a
//             352-float shared-memory row (so that the output row leaves in 16-B stores), the dense + sparse copy part
//             of the row is stored straight from the fragment registers.
//   backward  dX = S X with S = G + G^T (zero diagonal) built from the 351 pair gradients: M = 32 (i), N = 16 (d),
//             K = 32 (j).  S goes through shared memory (symmetric scatter, row stride 36: conflict-free fragment
//             reads); the B fragments are 8-B loads X[t + 4 h + 8 ks][2 g .. 2 g + 1] straight from global memory (the
//             output column of n-tile nt is permuted to d = 2 n + nt), which makes a lane's accumulators the four
//             consecutive floats dX[i][4 t .. 4 t + 3]: pass-through gradient added and stored as one 16-B vector.
//
// Accuracy: x = hi + lo with hi = tf32(x), lo = tf32(x - hi); the dropped lo*lo term is 2^-22 relative — the same class as
// the fp32 FFMA kernels (tests hold both to 1e-5).  Summation order differs from a sequential dot product.
//
// The includer provides TZK_DYN_SMEM / TZK_LAUNCH (nvcc: tzk_dense.cu, and tzk_interact_wide.cu for fwd_sample /
// bwd_sample; g++ + tests/native/cuda_cpu_shim.h: tests/test_interact_tc_cpu.py runs this source on the host with an
// emulated mma), tzk_itc::mma_tf32 and tzk_itc::cvt_tf32.
#pragma once
#include <stdint.h>

namespace tzk_itc {
constexpr int kWarps = 8;
constexpr int kN = 27, kD = 16, kP = 351, kInter = 352, kRow = 784;   // kInter = pairs + 1 zero (16-B aligned blocks)
constexpr int kSS = 36;                                               // row stride of S in shared memory

__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = cvt_tf32(x);
  lo = cvt_tf32(x - __uint_as_float(hi));
}

// row r of the interacting matrix, columns [c, c + 4): r = 0 dense, 1..26 sparse, beyond: zeros
__device__ __forceinline__ float4 load_x4(const float* dense_row, const float* sparse_row, int r, int c) {
  if (r == 0) return *reinterpret_cast<const float4*>(dense_row + c);
  if (r < kN) return *reinterpret_cast<const float4*>(sparse_row + (r - 1) * kD + c);
  return make_float4(0.f, 0.f, 0.f, 0.f);
}

// ---- forward --------------------------------------------------------------------------------------------------------
// first pair slot of the four rows lane (g, t)'s accumulators belong to: tri(i, j) = rowbase(i) + j
__device__ __forceinline__ void pair_rowbase(int g, int (&rowbase)[4]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = g + 8 * q;
    rowbase[q] = i * kN - (i * (i + 1)) / 2 - i - 1;
  }
}

// One sample, one warp: the kP pairs of Z = X X^T from the lane's rows x[j] = X[g + 8 j][4 t .. 4 t + 3] (zero beyond
// row 26), written as the kInter floats prow[0 .. kInter) in 16-B stores through the warp's staging row O (kInter floats,
// O[kP] zero).
__device__ __forceinline__ void fwd_sample(const float4 (&x)[4], const int (&rowbase)[4], float* O, float* prow,
                                           int lane) {
  const int g = lane >> 2, t = lane & 3;
  uint32_t hi[4][4], lo[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    split_tf32(x[j].x, hi[j][0], lo[j][0]);
    split_tf32(x[j].y, hi[j][1], lo[j][1]);
    split_tf32(x[j].z, hi[j][2], lo[j][2]);
    split_tf32(x[j].w, hi[j][3], lo[j][3]);
  }
  // tiles (mt, nt) that touch i < j: (0,0) (0,1) (0,2) (0,3) (1,2) (1,3)
  float acc[6][4];
#pragma unroll
  for (int e = 0; e < 6; ++e)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[e][q] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
    for (int e = 0; e < 6; ++e) {
      const int mt = e < 4 ? 0 : 1, nt = e < 4 ? e : e - 2;
      const uint32_t ah[4] = {hi[2 * mt][2 * ks], hi[2 * mt + 1][2 * ks], hi[2 * mt][2 * ks + 1], hi[2 * mt + 1][2 * ks + 1]};
      const uint32_t al[4] = {lo[2 * mt][2 * ks], lo[2 * mt + 1][2 * ks], lo[2 * mt][2 * ks + 1], lo[2 * mt + 1][2 * ks + 1]};
      const uint32_t bh[2] = {hi[nt][2 * ks], hi[nt][2 * ks + 1]};
      const uint32_t bl[2] = {lo[nt][2 * ks], lo[nt][2 * ks + 1]};
      mma_tf32(acc[e], al, bh);
      mma_tf32(acc[e], ah, bl);
      mma_tf32(acc[e], ah, bh);
    }
  }
  // accumulator (q) of tile e: i = g + 16 mt + 8 (q / 2), j = 8 nt + 2 t + (q % 2)
#pragma unroll
  for (int e = 0; e < 6; ++e) {
    const int mt = e < 4 ? 0 : 1, nt = e < 4 ? e : e - 2;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int ri = 2 * mt + (q >> 1);
      const int i = g + 8 * ri, j = 8 * nt + 2 * t + (q & 1);
      if (i < j && j < kN) O[rowbase[ri] + j] = acc[e][q];
    }
  }
  __syncwarp();
  for (int c = lane; c < kInter / 4; c += 32)
    *reinterpret_cast<float4*>(prow + 4 * c) = *reinterpret_cast<const float4*>(O + 4 * c);
  __syncwarp();
}

__global__ void __launch_bounds__(kWarps * 32)
dot_interact27_fwd_tc_kernel(const float* __restrict__ dense, int64_t ld_dense, const float* __restrict__ sparse,
                             int64_t ld_sparse, int64_t B, float* __restrict__ out, int64_t ld_out) {
  TZK_DYN_SMEM(float, smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  float* O = smem + warp * kInter;
  if (lane == 0) O[kP] = 0.f;          // the zero between the pairs and the dense block
  int rowbase[4];
  pair_rowbase(g, rowbase);
  const int64_t stride = (int64_t)gridDim.x * kWarps;
  int64_t b = (int64_t)blockIdx.x * kWarps + warp;
  float4 x[4];
  if (b < B) {
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = load_x4(dense + b * ld_dense, sparse + b * ld_sparse, g + 8 * j, 4 * t);
  }
  for (; b < B; b += stride) {
    // the next sample's rows are requested before this one is worked on
    float4 xn[4];
    const int64_t bn = b + stride;
    if (bn < B) {
#pragma unroll
      for (int j = 0; j < 4; ++j) xn[j] = load_x4(dense + bn * ld_dense, sparse + bn * ld_sparse, g + 8 * j, 4 * t);
    }
    float* orow = out + b * ld_out;
    // copy part of the output row: [kInter + 16 r + 4 t, +4) = X[r][4 t .. 4 t + 3]
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = g + 8 * j;
      if (r < kN) *reinterpret_cast<float4*>(orow + kInter + r * kD + 4 * t) = x[j];
    }
    fwd_sample(x, rowbase, O, orow, lane);
    if (bn < B) {
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = xn[j];
    }
  }
}

// ---- backward -------------------------------------------------------------------------------------------------------
// pair index -> (i << 8) | j, for the kP pairs; written by the whole CTA (the caller synchronises)
__device__ __forceinline__ void init_pair_ij(unsigned short* pair_ij) {
  for (int idx = threadIdx.x; idx < kP; idx += blockDim.x) {
    int i = 0, rs = 0;
    while (idx >= rs + (kN - 1 - i)) { rs += kN - 1 - i; ++i; }
    pair_ij[idx] = (unsigned short)((i << 8) | (i + 1 + (idx - rs)));
  }
}

// One sample, one warp: dE[i][.] = sum_j S[i][j] E[j][.] + pass, S = G + G^T from the kP pair gradients gp[] (global or
// shared memory), E = rows dr (dense) and sr (sparse).  pass[q] = pass-through gradient dE[g + 8 q][4 t .. 4 t + 3] (zero
// beyond row 26), loaded by the caller so that its latency overlaps other work.  S: this warp's [32 x kSS] scratch, zero
// outside the pair entries; dd / ds: the sample's d_dense / d_sparse rows.
__device__ __forceinline__ void bwd_sample(const float* gp, const float* dr, const float* sr, const float4 (&pass)[4],
                                           const unsigned short* pair_ij, float* S, float* dd, float* ds, int lane) {
  const int g = lane >> 2, t = lane & 3;
  // B fragments: X[j = t + 4 h + 8 ks][2 g, 2 g + 1]  (8-B loads; 4 rows x 64 B per instruction)
  float2 xv[4][2];
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = t + 4 * h + 8 * ks;
      float2 v = make_float2(0.f, 0.f);
      if (j == 0) v = *reinterpret_cast<const float2*>(dr + 2 * g);
      else if (j < kN) v = *reinterpret_cast<const float2*>(sr + (j - 1) * kD + 2 * g);
      xv[ks][h] = v;
    }
  // pair gradients -> symmetric S (coalesced reads, 11 per lane)
  {
    float gv[11];
#pragma unroll
    for (int q = 0; q < 11; ++q) {
      const int idx = lane + 32 * q;
      gv[q] = idx < kP ? gp[idx] : 0.f;
    }
#pragma unroll
    for (int q = 0; q < 11; ++q) {
      const int idx = lane + 32 * q;
      if (idx < kP) {
        const int i = pair_ij[idx] >> 8, j = pair_ij[idx] & 0xff;
        S[i * kSS + j] = gv[q];
        S[j * kSS + i] = gv[q];
      }
    }
  }
  __syncwarp();
  uint32_t xh[4][2][2], xl[4][2][2];      // [ks][h][nt]
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      split_tf32(xv[ks][h].x, xh[ks][h][0], xl[ks][h][0]);
      split_tf32(xv[ks][h].y, xh[ks][h][1], xl[ks][h][1]);
    }
  float acc[2][2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[mt][nt][q] = 0.f;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
      // A fragment: S[g + 16 mt (+8)][t + 8 ks (+4)]
      const float* sp = S + (g + 16 * mt) * kSS + t + 8 * ks;
      uint32_t ah[4], al[4];
      split_tf32(sp[0], ah[0], al[0]);
      split_tf32(sp[8 * kSS], ah[1], al[1]);
      split_tf32(sp[4], ah[2], al[2]);
      split_tf32(sp[8 * kSS + 4], ah[3], al[3]);
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
        const uint32_t bh[2] = {xh[ks][0][nt], xh[ks][1][nt]};
        const uint32_t bl[2] = {xl[ks][0][nt], xl[ks][1][nt]};
        mma_tf32(acc[mt][nt], al, bh);
        mma_tf32(acc[mt][nt], ah, bl);
        mma_tf32(acc[mt][nt], ah, bh);
      }
    }
  }
  __syncwarp();        // every lane is done reading S before the next sample's scatter
  // accumulators -> dX[i][4 t .. 4 t + 3]: tile nt holds d = 4 t + nt (q even) and 4 t + 2 + nt (q odd)
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int i = g + 16 * mt + 8 * hrow;
      if (i >= kN) continue;
      float4 v = make_float4(acc[mt][0][2 * hrow], acc[mt][1][2 * hrow], acc[mt][0][2 * hrow + 1],
                             acc[mt][1][2 * hrow + 1]);
      const float4 p = pass[2 * mt + hrow];
      v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
      if (i == 0) *reinterpret_cast<float4*>(dd + 4 * t) = v;
      else *reinterpret_cast<float4*>(ds + (i - 1) * kD + 4 * t) = v;
    }
}

__global__ void __launch_bounds__(kWarps * 32)
dot_interact27_bwd_tc_kernel(const float* __restrict__ dense, int64_t ld_dense, const float* __restrict__ sparse,
                             int64_t ld_sparse, const float* __restrict__ d_out, int64_t ld_dout, int64_t B,
                             float* __restrict__ d_dense, int64_t ld_ddense, float* __restrict__ d_sparse,
                             int64_t ld_dsparse) {
  TZK_DYN_SMEM(float, smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  // CTA-wide table: pair index -> (i, j); then one S matrix per warp
  unsigned short* pair_ij = reinterpret_cast<unsigned short*>(smem);
  float* S = smem + kInter / 2 + warp * (32 * kSS);       // (352 u16 = 176 floats)
  init_pair_ij(pair_ij);
  for (int i = lane; i < 32 * kSS; i += 32) S[i] = 0.f;   // diagonal and padding stay zero for the whole kernel
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * kWarps;
  for (int64_t b = (int64_t)blockIdx.x * kWarps + warp; b < B; b += stride) {
    const float* go = d_out + b * ld_dout;
    float4 pass[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = g + 8 * q;
      pass[q] = i < kN ? *reinterpret_cast<const float4*>(go + kInter + i * kD + 4 * t) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    bwd_sample(go, dense + b * ld_dense, sparse + b * ld_sparse, pass, pair_ij, S, d_dense + b * ld_ddense,
               d_sparse + b * ld_dsparse, lane);
  }
}

inline size_t fwd_smem() { return (size_t)kWarps * kInter * sizeof(float); }
inline size_t bwd_smem() { return ((size_t)kInter / 2 + (size_t)kWarps * 32 * kSS) * sizeof(float); }
inline int grid_for(int64_t B, int max_ctas) {
  const int64_t g = (B + kWarps - 1) / kWarps;
  return (int)(g < 1 ? 1 : (g < max_ctas ? g : max_ctas));
}

// whether the shape / layout is the one these kernels are written for
inline bool covers(const float* dense, int64_t ld_dense, int64_t ld_sparse, int Ns, int D, int copy_dense, int copy_sparse,
                   int p_pad, const float* io, int64_t ld_io) {
  return dense != nullptr && Ns == kN - 1 && D == kD && copy_dense && copy_sparse && p_pad == 1 && (ld_dense % 4) == 0 &&
         (ld_sparse % 4) == 0 && (ld_io % 4) == 0 && (reinterpret_cast<uintptr_t>(io) % 16) == 0;
}
}  // namespace tzk_itc
