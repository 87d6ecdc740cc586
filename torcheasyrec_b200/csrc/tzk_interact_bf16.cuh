// tzk_interact_bf16.cuh — DLRM-Criteo dot interaction in BF16 on the tensor cores (mma.sync m16n8k16 bf16, fp32
// accumulation), forward and backward, for training under bf16 autocast.  Shape: N = 27 interacting rows (the bottom-MLP
// output + 26 pooled embeddings) of D = 16, output row [351 pairs | 1 zero | 16 dense | 416 sparse] = 784 bf16 — the input
// of the first final-MLP layer, which autocast runs in bf16 anyway.
//
// Rounding points (those of tzrec/models/dlrm.py:113-131 under torch.autocast(dtype=torch.bfloat16)):
//   forward   F = [dense (bf16 as it is) ; bf16_rn(sparse)]; pair (i, j) = bf16_rn(sum_k F[i][k] F[j][k]), products exact,
//             fp32 accumulation (autocast's bmm).  The copied columns are dense and bf16_rn(sparse).
//   backward  G = upper triangle of the pair gradient (bf16).  Autograd's bmm backward gives two bf16 GEMMs,
//             g1 = bf16_rn(G F) and g2 = bf16_rn(G^T F), which meet in fp32 at the fp32 `cat` of dense and sparse:
//             s = fp32(g1 + g2).  Then
//               d_dense  = bf16_rn(bf16_rn(s) + dX_dense)       (the cat's backward casts s to the bf16 dense_feat, whose
//                                                              two incoming bf16 gradients are added in bf16)
//               d_sparse = s + dX_sparse                        (fp32)
//
// One warp per sample, as in tzk_interact_tc.cuh.
//   forward   Z = F F^T (32 x 32 padded, K = 16: one k-step).  Lane (g = lane / 4, t = lane % 4) loads F[g + 8 j][4 t .. 4 t
//             + 3], j = 0..3, and packs it into two bf16x2 registers.  The contraction index is permuted (logical k 2t, 2t+1
//             -> physical 4t, 4t+1; logical 2t+8, 2t+9 -> physical 4t+2, 4t+3), so the A fragment of row block mt and the B
//             fragment of column block nt are the lane's own registers.  6 of the 8 tiles hold strict-upper pairs: 6
//             MMAs.  Pairs go through a 352-bf16 shared-memory row and leave in 16-B stores; the copy part is stored
//             from the packed registers (8-B stores).
//   backward  g1 / g2 = U F / L F with U = G, L = G^T: M = 32 (i), N = 16 (d), K = 32 (j), two k-steps, 2 x 8 MMAs.  U and
//             L are scattered as bf16 into two [32 x kS] shared-memory matrices (row stride 40 bf16 = 20 words:
//             conflict-free fragment reads).  B fragments pack F[j][d], F[j + 1][d]; the output column of n-tile nt is
//             permuted to d = 2 n + nt, so a lane loads F[j][2 g .. 2 g + 1] (8 B) and its accumulators are
//             dF[i][4 t .. 4 t + 3].
//
// The includer provides TZK_DYN_SMEM, uint2 / uint4 and, in namespace tzk_ib16, mma_bf16 (m16n8k16, row.col, f32
// accumulate), pack_bf16x2(lo, hi) (two round-to-nearest-even conversions, `lo` in the low half) and bf16_rn(x)
// (nvcc: tzk_interact_bf16.cu; g++: tests/native/interact_bf16_standalone.cu with the emulation in
// tests/native/bf16_mma_emu.h).
#pragma once
#include <stdint.h>

namespace tzk_ib16 {
constexpr int kWarps = 8;
constexpr int kN = 27, kD = 16, kP = 351, kInter = 352, kRow = 784;
constexpr int kS = 40;                                           // row stride (bf16) of U and L in shared memory

__device__ __forceinline__ float bf16_to_f(uint16_t h) { return __uint_as_float((uint32_t)h << 16); }
__device__ __forceinline__ float bf16_round(float x) { return bf16_to_f(bf16_rn(x)); }

// row r of F, physical columns [c, c + 4) as bf16x2 (c, c+1) and (c+2, c+3): r = 0 dense, 1..26 sparse, beyond: zeros
__device__ __forceinline__ uint2 load_f4(const uint16_t* dense_row, const float* sparse_row, int r, int c) {
  if (r == 0) return *reinterpret_cast<const uint2*>(dense_row + c);
  if (r < kN) {
    const float4 v = *reinterpret_cast<const float4*>(sparse_row + (r - 1) * kD + c);
    uint2 p;
    p.x = pack_bf16x2(v.x, v.y);
    p.y = pack_bf16x2(v.z, v.w);
    return p;
  }
  uint2 z;
  z.x = 0u;
  z.y = 0u;
  return z;
}

// ---- forward --------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kWarps * 32)
dot_interact27_fwd_bf16_kernel(const uint16_t* __restrict__ dense, int64_t ld_dense, const float* __restrict__ sparse,
                               int64_t ld_sparse, int64_t B, uint16_t* __restrict__ out, int64_t ld_out) {
  TZK_DYN_SMEM(uint16_t, smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  uint16_t* O = smem + warp * kInter;
  if (lane == 0) O[kP] = 0;            // the zero between the pairs and the dense block
  int rowbase[4];                      // tri(i, j) = rowbase(i) + j
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int i = g + 8 * q;
    rowbase[q] = i * kN - (i * (i + 1)) / 2 - i - 1;
  }
  const int64_t stride = (int64_t)gridDim.x * kWarps;
  int64_t b = (int64_t)blockIdx.x * kWarps + warp;
  uint2 x[4];
  if (b < B) {
#pragma unroll
    for (int j = 0; j < 4; ++j) x[j] = load_f4(dense + b * ld_dense, sparse + b * ld_sparse, g + 8 * j, 4 * t);
  }
  for (; b < B; b += stride) {
    uint2 xn[4];                       // the next sample's rows are requested before this one is worked on
    const int64_t bn = b + stride;
    if (bn < B) {
#pragma unroll
      for (int j = 0; j < 4; ++j) xn[j] = load_f4(dense + bn * ld_dense, sparse + bn * ld_sparse, g + 8 * j, 4 * t);
    }
    uint16_t* orow = out + b * ld_out;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = g + 8 * j;
      if (r < kN) *reinterpret_cast<uint2*>(orow + kInter + r * kD + 4 * t) = x[j];
    }
    // tiles (mt, nt) that touch i < j: (0,0) (0,1) (0,2) (0,3) (1,2) (1,3)
    float acc[6][4];
#pragma unroll
    for (int e = 0; e < 6; ++e) {
      const int mt = e < 4 ? 0 : 1, nt = e < 4 ? e : e - 2;
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[e][q] = 0.f;
      const uint32_t a[4] = {x[2 * mt].x, x[2 * mt + 1].x, x[2 * mt].y, x[2 * mt + 1].y};
      const uint32_t bb[2] = {x[nt].x, x[nt].y};
      mma_bf16(acc[e], a, bb);
    }
    // accumulator q of tile e: i = g + 16 mt + 8 (q / 2), j = 8 nt + 2 t + (q % 2)
#pragma unroll
    for (int e = 0; e < 6; ++e) {
      const int mt = e < 4 ? 0 : 1, nt = e < 4 ? e : e - 2;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int ri = 2 * mt + (q >> 1);
        const int i = g + 8 * ri, j = 8 * nt + 2 * t + (q & 1);
        if (i < j && j < kN) O[rowbase[ri] + j] = bf16_rn(acc[e][q]);
      }
    }
    __syncwarp();
    for (int c = lane; c < kInter / 8; c += 32)
      *reinterpret_cast<uint4*>(orow + 8 * c) = *reinterpret_cast<const uint4*>(O + 8 * c);
    __syncwarp();
    if (bn < B) {
#pragma unroll
      for (int j = 0; j < 4; ++j) x[j] = xn[j];
    }
  }
}

// ---- backward -------------------------------------------------------------------------------------------------------
// F[j][2 g .. 2 g + 1] as floats (bf16 values), zero beyond row 26
__device__ __forceinline__ float2 load_f2(const uint16_t* dr, const float* sr, int j, int g) {
  if (j == 0) {
    const uint32_t p = *reinterpret_cast<const uint32_t*>(dr + 2 * g);
    return make_float2(bf16_to_f((uint16_t)(p & 0xffffu)), bf16_to_f((uint16_t)(p >> 16)));
  }
  if (j < kN) {
    const float2 v = *reinterpret_cast<const float2*>(sr + (j - 1) * kD + 2 * g);
    return make_float2(bf16_round(v.x), bf16_round(v.y));
  }
  return make_float2(0.f, 0.f);
}

__global__ void __launch_bounds__(kWarps * 32)
dot_interact27_bwd_bf16_kernel(const uint16_t* __restrict__ dense, int64_t ld_dense, const float* __restrict__ sparse,
                               int64_t ld_sparse, const uint16_t* __restrict__ d_out, int64_t ld_dout, int64_t B,
                               uint16_t* __restrict__ d_dense, int64_t ld_ddense, float* __restrict__ d_sparse,
                               int64_t ld_dsparse) {
  TZK_DYN_SMEM(uint16_t, smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  uint16_t* pair_ij = smem;                                       // pair index -> (i << 8) | j
  uint16_t* U = smem + kInter + warp * (2 * 32 * kS);
  uint16_t* L = U + 32 * kS;
  for (int idx = threadIdx.x; idx < kP; idx += blockDim.x) {
    int i = 0, rs = 0;
    while (idx >= rs + (kN - 1 - i)) { rs += kN - 1 - i; ++i; }
    pair_ij[idx] = (uint16_t)((i << 8) | (i + 1 + (idx - rs)));
  }
  for (int i = lane; i < 2 * 32 * kS; i += 32) U[i] = 0;         // everything but the pair entries stays zero
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * kWarps;
  for (int64_t b = (int64_t)blockIdx.x * kWarps + warp; b < B; b += stride) {
    const uint16_t* go = d_out + b * ld_dout;
    const uint16_t* dr = dense + b * ld_dense;
    const float* sr = sparse + b * ld_sparse;
    uint2 pass[4];                     // dX[g + 8 q][4 t .. 4 t + 3] (bf16), zero beyond row 26
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = g + 8 * q;
      pass[q].x = 0u;
      pass[q].y = 0u;
      if (i < kN) pass[q] = *reinterpret_cast<const uint2*>(go + kInter + i * kD + 4 * t);
    }
    // B fragments: rows j = 16 ks + 8 h + 2 t + e (e = 0, 1 packed into one register), columns d = 2 g + nt
    float2 fv[2][2][2];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int e = 0; e < 2; ++e) fv[ks][h][e] = load_f2(dr, sr, 16 * ks + 8 * h + 2 * t + e, g);
    {
      uint16_t gv[11];
#pragma unroll
      for (int q = 0; q < 11; ++q) {
        const int idx = lane + 32 * q;
        gv[q] = idx < kP ? go[idx] : (uint16_t)0;
      }
#pragma unroll
      for (int q = 0; q < 11; ++q) {
        const int idx = lane + 32 * q;
        if (idx < kP) {
          const int i = pair_ij[idx] >> 8, j = pair_ij[idx] & 0xff;
          U[i * kS + j] = gv[q];
          L[j * kS + i] = gv[q];
        }
      }
    }
    __syncwarp();
    uint32_t bf[2][2][2];              // [ks][h][nt]
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        bf[ks][h][0] = pack_bf16x2(fv[ks][h][0].x, fv[ks][h][1].x);
        bf[ks][h][1] = pack_bf16x2(fv[ks][h][0].y, fv[ks][h][1].y);
      }
    float au[2][2][4], al[2][2][4];    // [mt][nt][q]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) au[mt][nt][q] = al[mt][nt][q] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        // A fragments: rows g + 16 mt (+8), columns 16 ks + 2 t (+1) and (+8, +9)
        const int o = (g + 16 * mt) * kS + 16 * ks + 2 * t;
        const uint32_t a_u[4] = {*reinterpret_cast<const uint32_t*>(U + o), *reinterpret_cast<const uint32_t*>(U + o + 8 * kS),
                                 *reinterpret_cast<const uint32_t*>(U + o + 8),
                                 *reinterpret_cast<const uint32_t*>(U + o + 8 * kS + 8)};
        const uint32_t a_l[4] = {*reinterpret_cast<const uint32_t*>(L + o), *reinterpret_cast<const uint32_t*>(L + o + 8 * kS),
                                 *reinterpret_cast<const uint32_t*>(L + o + 8),
                                 *reinterpret_cast<const uint32_t*>(L + o + 8 * kS + 8)};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt) {
          const uint32_t bb[2] = {bf[ks][0][nt], bf[ks][1][nt]};
          mma_bf16(au[mt][nt], a_u, bb);
          mma_bf16(al[mt][nt], a_l, bb);
        }
      }
    }
    __syncwarp();                      // every lane is done reading U / L before the next sample's scatter
    // accumulators -> dF[i][4 t .. 4 t + 3]: tile nt holds d = 4 t + nt (q even) and 4 t + 2 + nt (q odd)
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int hrow = 0; hrow < 2; ++hrow) {
        const int i = g + 16 * mt + 8 * hrow;
        if (i >= kN) continue;
        const int qs[4] = {2 * hrow, 2 * hrow, 2 * hrow + 1, 2 * hrow + 1};
        const int ns[4] = {0, 1, 0, 1};
        float s[4];
#pragma unroll
        for (int c = 0; c < 4; ++c)
          s[c] = bf16_round(au[mt][ns[c]][qs[c]]) + bf16_round(al[mt][ns[c]][qs[c]]);
        const uint2 p = pass[2 * mt + hrow];
        const float pf[4] = {bf16_to_f((uint16_t)(p.x & 0xffffu)), bf16_to_f((uint16_t)(p.x >> 16)),
                             bf16_to_f((uint16_t)(p.y & 0xffffu)), bf16_to_f((uint16_t)(p.y >> 16))};
        if (i == 0) {
          uint2 v;
          v.x = pack_bf16x2(bf16_round(s[0]) + pf[0], bf16_round(s[1]) + pf[1]);
          v.y = pack_bf16x2(bf16_round(s[2]) + pf[2], bf16_round(s[3]) + pf[3]);
          *reinterpret_cast<uint2*>(d_dense + b * ld_ddense + 4 * t) = v;
        } else {
          *reinterpret_cast<float4*>(d_sparse + b * ld_dsparse + (i - 1) * kD + 4 * t) =
              make_float4(s[0] + pf[0], s[1] + pf[1], s[2] + pf[2], s[3] + pf[3]);
        }
      }
  }
}

inline size_t fwd_smem() { return (size_t)kWarps * kInter * sizeof(uint16_t); }
inline size_t bwd_smem() { return ((size_t)kInter + (size_t)kWarps * 2 * 32 * kS) * sizeof(uint16_t); }
inline int grid_for(int64_t B, int max_ctas) {
  const int64_t g = (B + kWarps - 1) / kWarps;
  return (int)(g < 1 ? 1 : (g < max_ctas ? g : max_ctas));
}
}  // namespace tzk_ib16
