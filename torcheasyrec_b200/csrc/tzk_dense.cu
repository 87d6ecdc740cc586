// tzk_dense.cu — K6 regroup (column gather-sum), K7 jagged<->padded, A7 FM, A9/A10 DLRM dot interaction.
// All HBM-bound fp32 movers; the interaction is 7.4 FLOP/B (SURVEY §8a A9) so it is written as a
// register-tiled FFMA kernel that reads each pooled row once and emits the whole final-MLP input.
#include <cstdlib>

#include "tzk_common.cuh"

using namespace tzk;

// ---- tensor-core variant of the DLRM interaction (mma.sync m16n8k8, 3xTF32) -------------------------------------------
#include "tzk_launch.cuh"
namespace tzk_itc {
__device__ __forceinline__ uint32_t cvt_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
}  // namespace tzk_itc
#include "tzk_interact_tc.cuh"


namespace {
constexpr int kThreads = 256;

// ---------------------------------------------------------------------------------------------------
// K6: out[row, c] = sum_{k in [col_start[c], col_start[c+1])} srcs[col_src[k]][row*ld + col_srccol[k]]
// ---------------------------------------------------------------------------------------------------
constexpr int kMaxSrc = 16;
struct SrcTable {  // passed by value: no device-side pointer table, so the call is CUDA-graph safe
  const float* p[kMaxSrc];
  int64_t ld[kMaxSrc];
};

__global__ void __launch_bounds__(kThreads)
col_gather_sum_kernel(const SrcTable srcs, const int32_t* __restrict__ col_start, const int32_t* __restrict__ col_src,
                      const int32_t* __restrict__ col_srccol, int C, int64_t rows, float* __restrict__ out,
                      int64_t ld_out) {
  const int64_t n = rows * C;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t row = i / C;
    const int c = (int)(i - row * C);
    const int k0 = __ldg(col_start + c), k1 = __ldg(col_start + c + 1);
    float acc = 0.f;
    for (int k = k0; k < k1; ++k) {
      const int s = __ldg(col_src + k);
      acc += __ldg(srcs.p[s] + row * srcs.ld[s] + __ldg(col_srccol + k));
    }
    out[row * ld_out + c] = acc;
  }
}

// ---------------------------------------------------------------------------------------------------
// K7
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
jagged_to_padded_kernel(const float* __restrict__ values, const int64_t* __restrict__ offsets, int B, int T,
                        int D, float* __restrict__ out) {
  const int64_t n = (int64_t)B * T * D;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int d = (int)(i % D);
    const int64_t bt = i / D;
    const int t = (int)(bt % T);
    const int b = (int)(bt / T);
    const int64_t s = __ldg(offsets + b), e = __ldg(offsets + b + 1);
    out[i] = (s + t < e) ? __ldg(values + (s + t) * D + d) : 0.f;
  }
}

__global__ void __launch_bounds__(kThreads)
padded_to_jagged_kernel(const float* __restrict__ grad_out, const int64_t* __restrict__ offsets, int B, int T,
                        int D, int64_t nnz, float* __restrict__ grad_values) {
  // one thread per (jagged row, d): find b by binary search over offsets
  const int64_t n = nnz * D;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t l = i / D;
    const int d = (int)(i - l * D);
    int lo = 0, hi = B;  // largest b with offsets[b] <= l
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (__ldg(offsets + mid) <= l) lo = mid; else hi = mid;
    }
    const int64_t t = l - __ldg(offsets + lo);
    grad_values[i] = (t < T) ? __ldg(grad_out + ((int64_t)lo * T + t) * D + d) : 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------
// A7: FM.  one thread per (b, d): two running sums over n.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
fm_fwd_kernel(const float* __restrict__ x, int64_t ld_x, int64_t B, int N, int D, float* __restrict__ y,
              int64_t ld_y) {
  const int64_t n = B * D;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t b = i / D;
    const int d = (int)(i - b * D);
    const float* xb = x + b * ld_x + d;
    float s = 0.f, q = 0.f;
#pragma unroll 4
    for (int k = 0; k < N; ++k) {
      const float v = __ldg(xb + (int64_t)k * D);
      s += v;
      q += v * v;
    }
    y[b * ld_y + d] = 0.5f * (s * s - q);
  }
}

__global__ void __launch_bounds__(kThreads)
fm_bwd_kernel(const float* __restrict__ x, int64_t ld_x, const float* __restrict__ dy, int64_t ld_dy,
              int64_t B, int N, int D, float* __restrict__ dx, int64_t ld_dx) {
  const int64_t n = B * D;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t b = i / D;
    const int d = (int)(i - b * D);
    const float* xb = x + b * ld_x + d;
    float s = 0.f;
#pragma unroll 4
    for (int k = 0; k < N; ++k) s += __ldg(xb + (int64_t)k * D);
    const float g = __ldg(dy + b * ld_dy + d);
    float* dxb = dx + b * ld_dx + d;
#pragma unroll 4
    for (int k = 0; k < N; ++k) dxb[(int64_t)k * D] = g * (s - __ldg(xb + (int64_t)k * D));
  }
}

// ---------------------------------------------------------------------------------------------------
// A9/A10: dot interaction.  One warp per sample, persistent over samples.
//  * X_b (N x D) is staged in shared memory, row stride D+4 floats, 16-B chunks XOR-swizzled by (row>>3) so
//    that the eight lanes of a quarter-warp, which read the same chunk of rows 4 apart, hit eight different
//    bank groups (unswizzled they collide 4-way);
//  * each lane owns 4x4 blocks of the Gram matrix (only blocks touching the strict upper triangle): every k
//    step costs 2 LDS.128 per 16 FMAs; the (bi,bj) decode is a per-CTA lookup table, not per-sample maths;
//  * results are staged in shared memory and the whole output row [P | D | Ns*D] leaves with coalesced stores.
// ---------------------------------------------------------------------------------------------------
constexpr int kIWarps = 8;  // most warps (= samples in flight) per CTA; the kernels read the count from blockDim.x
constexpr size_t kIMaxSmem = 227 * 1024;  // largest dynamic shared memory one CTA may opt into (sm_90)

__device__ __forceinline__ int tri_index(int i, int j, int N) {  // i < j
  return i * N - (i * (i + 1)) / 2 + (j - i - 1);
}
__device__ __forceinline__ int swz_mask(int D4) {  // XOR range must stay inside the row's D4 chunks
  return ((D4 & (D4 - 1)) == 0) ? (D4 - 1 < 3 ? D4 - 1 : 3) : 0;
}
// float offset of chunk c4 of row `row`
__device__ __forceinline__ int xoff(int row, int c4, int DS, int swm) { return row * DS + ((c4 ^ ((row >> 3) & swm)) << 2); }

// All row loads of a sample are issued before the first one is consumed (4 float4 per lane cover Ns*D/4 <= 128
// chunks in one batch): one exposed memory latency per sample instead of one per 32 chunks.
__device__ __forceinline__ void stage_x(float* X, const float* dense, int64_t ld_dense, const float* sparse,
                                        int64_t ld_sparse, int64_t b, int Ns, int N, int Np, int D4, int DS, int swm,
                                        int lane) {
  const int doff = dense ? 1 : 0;
  const float* sp = sparse + b * ld_sparse;
  const int n_chunks = Ns * D4;
  float4 dv = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool has_dv = dense && lane < D4;
  if (has_dv) dv = ld_row_f4(dense + b * ld_dense + lane * 4);
  for (int i0 = lane; i0 < n_chunks; i0 += 128) {
    float4 v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = i0 + 32 * q;
      if (i < n_chunks) v[q] = ld_row_f4(sp + (int64_t)i * 4);
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int i = i0 + 32 * q;
      if (i < n_chunks) {
        const int r = i / D4, c4 = i - r * D4;
        *reinterpret_cast<float4*>(X + xoff(r + doff, c4, DS, swm)) = v[q];
      }
    }
  }
  if (has_dv) *reinterpret_cast<float4*>(X + xoff(0, lane, DS, swm)) = dv;
  if (dense)
    for (int c4 = lane + 32; c4 < D4; c4 += 32)
      *reinterpret_cast<float4*>(X + xoff(0, c4, DS, swm)) = ld_row_f4(dense + b * ld_dense + c4 * 4);
}

// DT = compile-time embedding dim (0 = take the runtime value): with DT known every /D, %D and swizzle offset
// folds into shifts and the k loop unrolls — the kernel is issue-bound, not bandwidth-bound, otherwise.
// 4 CTAs/SM (64 registers, a few spilled words) rather than 3 CTAs/SM (80 registers): the occupancy hides the latency.
template <int DT, bool ONE, int NT>
__global__ void __launch_bounds__(kIWarps * 32, 4)
dot_interact_fwd_kernel(const float* __restrict__ dense, int64_t ld_dense, const float* __restrict__ sparse,
                        int64_t ld_sparse, int64_t B, int Ns, int D_rt, int copy_dense, int copy_sparse, int p_pad,
                        int aligned, float* __restrict__ out, int64_t ld_out) {
  extern __shared__ __align__(16) float smem[];
  const int D = DT ? DT : D_rt;
  if (NT) Ns = NT - 1;                // NT > 0: compile-time feature count incl. the dense row (dense != NULL)
  const int N = NT ? NT : Ns + (dense != nullptr);
  const int Np = (N + 3) & ~3;        // rows padded to a multiple of 4 (pad rows are zero)
  const int DS = D + 4;               // row stride
  const int P = N * (N - 1) / 2;
  const int Pp = (P + 3 + 4) & ~3;    // room for p_pad zeros; keeps every warp's slab 16-B aligned
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
  const int nb = Np / 4;
  const int n_blocks = nb * (nb + 1) / 2;
  const int D4 = D / 4;  // D % 4 == 0 enforced by the host wrapper
  const int swm = swz_mask(D4);
  // CTA-wide lookup: block index -> (bi, bj)
  unsigned short* blk_ij = reinterpret_cast<unsigned short*>(smem);
  float* slabs = smem + ((n_blocks + 7) / 8) * 4;  // n_blocks u16 rounded up to 16 B
  for (int blk = threadIdx.x; blk < n_blocks; blk += blockDim.x) {
    int bi = 0, rem = blk;
    while (rem >= nb - bi) { rem -= nb - bi; ++bi; }
    blk_ij[blk] = (unsigned short)((bi << 8) | (bi + rem));
  }
  float* X = slabs + (size_t)warp * (Np * DS + Pp);
  float* O = X + Np * DS;
  // pad rows are zero for the whole kernel
  for (int i = lane; i < (Np - N) * D4; i += 32) {
    const int r = N + i / D4, c4 = i % D4;
    *reinterpret_cast<float4*>(X + xoff(r, c4, DS, swm)) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __syncthreads();
  const int doff = dense ? 1 : 0;
  // lane-constant block description (used when the triangle has at most 32 blocks, e.g. N = 27 -> 28)
  constexpr bool one_block = ONE;   // host guarantees n_blocks <= 32 when ONE
  int lb_a = 0, lb_b = 0, lb_asw = 0, lb_bsw = 0, lb_o[4] = {0, 0, 0, 0};
  unsigned lb_valid = 0;
  if (one_block && lane < n_blocks) {
    const int bi = blk_ij[lane] >> 8, bj = blk_ij[lane] & 0xff;
    lb_a = bi * 4 * DS;
    lb_b = bj * 4 * DS;
    lb_asw = ((bi * 4) >> 3) & swm;   // the 4 rows of a block share (row >> 3)
    lb_bsw = ((bj * 4) >> 3) & swm;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int i = bi * 4 + r;
      lb_o[r] = i * N - (i * (i + 1)) / 2 + (bj * 4 - i - 1);   // tri_index(i, bj*4 + c) = lb_o[r] + c
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = bj * 4 + c;
        if (i < j && j < N) lb_valid |= 1u << (r * 4 + c);
      }
    }
  }

  for (int64_t b = (int64_t)blockIdx.x * n_warps + warp; b < B; b += (int64_t)gridDim.x * n_warps) {
    stage_x(X, dense, ld_dense, sparse, ld_sparse, b, Ns, N, Np, D4, DS, swm, lane);
    __syncwarp();
    // ---- Gram blocks ------------------------------------------------------------------------------
    if constexpr (one_block) {
      // every lane owns at most ONE block for the whole kernel: addresses, swizzles and output slots were
      // computed once before the sample loop
      if (lane < n_blocks) {
        float acc[4][4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
        const float* pa = X + lb_a;
        const float* pb = X + lb_b;
#pragma unroll DT ? DT / 4 : 1
        for (int c4 = 0; c4 < D4; ++c4) {
          const int oa = (c4 ^ lb_asw) << 2, ob = (c4 ^ lb_bsw) << 2;
          float4 a[4], bb[4];
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            a[r] = *reinterpret_cast<const float4*>(pa + r * DS + oa);
            bb[r] = *reinterpret_cast<const float4*>(pb + r * DS + ob);
          }
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              acc[r][c] = fmaf(a[r].x, bb[c].x, acc[r][c]);
              acc[r][c] = fmaf(a[r].y, bb[c].y, acc[r][c]);
              acc[r][c] = fmaf(a[r].z, bb[c].z, acc[r][c]);
              acc[r][c] = fmaf(a[r].w, bb[c].w, acc[r][c]);
            }
        }
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if ((lb_valid >> (r * 4 + c)) & 1) O[lb_o[r] + c] = acc[r][c];
      }
    } else {
    for (int blk = lane; blk < n_blocks; blk += 32) {
      const int bi = blk_ij[blk] >> 8, bj = blk_ij[blk] & 0xff;
      float acc[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
      // row bases / swizzles of the 8 rows this block touches (rows bi*4..+3 share (row>>3) pairwise)
      const float* arow[4];
      const float* brow[4];
      int asw[4], bsw[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        arow[r] = X + (bi * 4 + r) * DS;
        brow[r] = X + (bj * 4 + r) * DS;
        asw[r] = ((bi * 4 + r) >> 3) & swm;
        bsw[r] = ((bj * 4 + r) >> 3) & swm;
      }
#pragma unroll DT ? DT / 4 : 1
      for (int c4 = 0; c4 < D4; ++c4) {
        float4 a[4], bb[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          a[r] = *reinterpret_cast<const float4*>(arow[r] + ((c4 ^ asw[r]) << 2));
          bb[r] = *reinterpret_cast<const float4*>(brow[r] + ((c4 ^ bsw[r]) << 2));
        }
        // accumulate in k order so the sum order matches a sequential dot product
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            acc[r][c] = fmaf(a[r].x, bb[c].x, acc[r][c]);
            acc[r][c] = fmaf(a[r].y, bb[c].y, acc[r][c]);
            acc[r][c] = fmaf(a[r].z, bb[c].z, acc[r][c]);
            acc[r][c] = fmaf(a[r].w, bb[c].w, acc[r][c]);
          }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int i = bi * 4 + r, j = bj * 4 + c;
          if (i < j && j < N) O[tri_index(i, j, N)] = acc[r][c];
        }
    }
    }
    __syncwarp();
    // ---- coalesced output row ---------------------------------------------------------------------
    float* orow = out + b * ld_out;
    int o = P + p_pad;   // layout: [P interactions | p_pad zeros | D dense | Ns*D sparse]
    if (aligned) {
      // rows, the dense block and the sparse block all start on 16-B boundaries: 128-bit stores throughout
      if (lane < p_pad) O[P + lane] = 0.f;
      __syncwarp();
      for (int i = lane; i < (o >> 2); i += 32)
        st_stream_f4(orow + i * 4, *reinterpret_cast<const float4*>(O + i * 4));
      if (copy_dense && dense) {
        for (int c4 = lane; c4 < D4; c4 += 32)
          st_stream_f4(orow + o + c4 * 4, *reinterpret_cast<const float4*>(X + xoff(0, c4, DS, swm)));
        o += D;
      }
      if (copy_sparse) {
        for (int i = lane; i < Ns * D4; i += 32) {
          const int r = i / D4, c4 = i - r * D4;
          st_stream_f4(orow + o + i * 4, *reinterpret_cast<const float4*>(X + xoff(r + doff, c4, DS, swm)));
        }
      }
    } else {
      for (int i = lane; i < P; i += 32) orow[i] = O[i];
      for (int i = lane; i < p_pad; i += 32) orow[P + i] = 0.f;
      if (copy_dense && dense) {
        for (int c = lane; c < D; c += 32) orow[o + c] = X[xoff(0, c >> 2, DS, swm) + (c & 3)];
        o += D;
      }
      if (copy_sparse) {
        for (int i = lane; i < Ns * D; i += 32) {
          const int r = i / D, c = i - r * D;
          orow[o + i] = X[xoff(r + doff, c >> 2, DS, swm) + (c & 3)];
        }
      }
    }
    __syncwarp();
  }
}

// backward: dX = (G + G^T) X (+ pass-through grads); lane owns 4 rows x 4 cols blocks of dX.
// NT = compile-time feature count INCLUDING the dense row (0 = runtime; NT > 0 requires dense != NULL): the j loop
// unrolls completely and every shared-memory address becomes base register + immediate.
template <int DT, int NT>
__global__ void __launch_bounds__(kIWarps * 32, 4)
dot_interact_bwd_kernel(const float* __restrict__ dense, int64_t ld_dense, const float* __restrict__ sparse,
                        int64_t ld_sparse, const float* __restrict__ d_out, int64_t ld_dout, int64_t B,
                        int Ns, int D_rt, int copy_dense, int copy_sparse, int p_pad, int aligned,
                        float* __restrict__ d_dense, int64_t ld_ddense, float* __restrict__ d_sparse,
                        int64_t ld_dsparse) {
  extern __shared__ __align__(16) float smem[];
  const int D = DT ? DT : D_rt;
  if (NT) Ns = NT - 1;
  const int N = NT ? NT : Ns + (dense != nullptr);
  const int Np = (N + 3) & ~3;
  const int DS = D + 4;
  const int SS = Np + 8;  // stride of the symmetric grad matrix: the transposed scatter is 4-way, not 32-way
  const int P = N * (N - 1) / 2;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, n_warps = blockDim.x >> 5;
  const int D4 = D / 4;
  const int swm = swz_mask(D4);
  const int nb = Np / 4;
  const int doff = dense ? 1 : 0;
  // CTA-wide lookup: triangular index -> (i, j)
  unsigned short* pair_ij = reinterpret_cast<unsigned short*>(smem);
  float* slabs = smem + ((P + 7) / 8) * 4;
  for (int idx = threadIdx.x; idx < P; idx += blockDim.x) {
    int i = 0, rs = 0;
    while (idx >= rs + (N - 1 - i)) { rs += N - 1 - i; ++i; }
    pair_ij[idx] = (unsigned short)((i << 8) | (i + 1 + (idx - rs)));
  }
  float* X = slabs + (size_t)warp * (Np * DS + Np * SS);
  float* S = X + Np * DS;
  for (int i = lane; i < (Np - N) * D4; i += 32) {
    const int r = N + i / D4, c4 = i % D4;
    *reinterpret_cast<float4*>(X + xoff(r, c4, DS, swm)) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int i = lane; i < Np * SS; i += 32) S[i] = 0.f;  // diagonal + padding stay zero for the whole kernel
  __syncthreads();

  for (int64_t b = (int64_t)blockIdx.x * n_warps + warp; b < B; b += (int64_t)gridDim.x * n_warps) {
    stage_x(X, dense, ld_dense, sparse, ld_sparse, b, Ns, N, Np, D4, DS, swm, lane);
    const float* go = d_out + b * ld_dout;
    for (int idx0 = lane; idx0 < P; idx0 += 32 * 6) {  // coalesced read of d_out (6 loads in flight), symmetric scatter
      float gv[6];
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const int idx = idx0 + 32 * q;
        gv[q] = idx < P ? __ldg(go + idx) : 0.f;
      }
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const int idx = idx0 + 32 * q;
        if (idx < P) {
          const int i = pair_ij[idx] >> 8, j = pair_ij[idx] & 0xff;
          S[i * SS + j] = gv[q];
          S[j * SS + i] = gv[q];
        }
      }
    }
    __syncwarp();
    // dX[i0..i0+3][k..k+3] = sum_j S[j][i0..i0+3] * X[j][k..k+3]
    const int n_blocks = nb * D4;
    for (int blk = lane; blk < n_blocks; blk += 32) {
      const int bi = blk / D4, c4 = blk - bi * D4;
      float acc[4][4];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) acc[r][c] = 0.f;
      const float* Sb = S + bi * 4;
      if (NT) {
        int xo[4];  // swizzled chunk offset for (j >> 3) & 3 = 0..3
#pragma unroll
        for (int q = 0; q < 4; ++q) xo[q] = (c4 ^ (q & swm)) << 2;
#pragma unroll
        for (int j = 0; j < (NT ? NT : 1); ++j) {
          const float4 s4 = *reinterpret_cast<const float4*>(Sb + j * SS);
          const float4 x4 = *reinterpret_cast<const float4*>(X + j * DS + xo[(j >> 3) & 3]);
          const float sv[4] = {s4.x, s4.y, s4.z, s4.w};
          const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(sv[r], xv[c], acc[r][c]);
        }
      } else {
#pragma unroll 3
        for (int j = 0; j < N; ++j) {
          const float4 s4 = *reinterpret_cast<const float4*>(Sb + j * SS);
          const float4 x4 = *reinterpret_cast<const float4*>(X + xoff(j, c4, DS, swm));
          const float sv[4] = {s4.x, s4.y, s4.z, s4.w};
          const float xv[4] = {x4.x, x4.y, x4.z, x4.w};
#pragma unroll
          for (int r = 0; r < 4; ++r)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[r][c] = fmaf(sv[r], xv[c], acc[r][c]);
        }
      }
      // pass-through grads and store (16-B vector stores; d_out offsets are not 16-B aligned -> scalar loads)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = bi * 4 + r;
        if (i >= N) continue;
        float4 v = make_float4(acc[r][0], acc[r][1], acc[r][2], acc[r][3]);
        if (dense && i == 0) {
          if (copy_dense) {
            const float* gp = go + P + p_pad + c4 * 4;
            if (aligned) {
              v = f4_add(v, __ldg(reinterpret_cast<const float4*>(gp)));  // not the asm load: a non-volatile asm may be speculated above `aligned`
            } else {
              v.x += __ldg(gp); v.y += __ldg(gp + 1); v.z += __ldg(gp + 2); v.w += __ldg(gp + 3);
            }
          }
          *reinterpret_cast<float4*>(d_dense + b * ld_ddense + c4 * 4) = v;
        } else {
          const int r_s = i - doff;
          if (copy_sparse) {
            const float* gp = go + P + p_pad + ((copy_dense && dense) ? D : 0) + r_s * D + c4 * 4;
            if (aligned) {
              v = f4_add(v, __ldg(reinterpret_cast<const float4*>(gp)));  // not the asm load: a non-volatile asm may be speculated above `aligned`
            } else {
              v.x += __ldg(gp); v.y += __ldg(gp + 1); v.z += __ldg(gp + 2); v.w += __ldg(gp + 3);
            }
          }
          *reinterpret_cast<float4*>(d_sparse + b * ld_dsparse + (int64_t)r_s * D + c4 * 4) = v;
        }
      }
    }
    __syncwarp();
  }
}

// The DLRM-Criteo shape (27 x 16, aligned output row) on the tensor cores (tzk_interact_tc.cuh); read per call (tests flip
// it).  Forward: default on, TZK_INTERACT_TC=0 / TZK_INTERACT_TC_FWD=0
// selects the FFMA kernel.  Backward: default on since its pass-through loads are requested up front (step 1.031 -> 1.010 ms);
// TZK_INTERACT_TC_BWD=0 selects the FFMA kernel.
inline bool env_is(const char* name, char v) {
  const char* e = getenv(name);
  return e && e[0] == v;
}
inline bool use_interact_tc_fwd() { return !env_is("TZK_INTERACT_TC", '0') && !env_is("TZK_INTERACT_TC_FWD", '0'); }
inline bool use_interact_tc_bwd() { return !env_is("TZK_INTERACT_TC", '0') && !env_is("TZK_INTERACT_TC_BWD", '0'); }

inline int grid_for(int64_t n, int per_block, int max_blocks) {
  int64_t g = ceil_div64(n, per_block);
  if (g < 1) g = 1;
  return (int)(g < max_blocks ? g : max_blocks);
}

// Warps per CTA of the FFMA interaction kernels: the largest of kIWarps, kIWarps/2, ..., 1 whose shared memory (a
// CTA-wide table of `table` floats plus one slab of `slab` floats per warp) fits kIMaxSmem, with its size in *smem;
// 0 when not even one warp fits.  Wide features (e.g. 64 x 64 in the backward) do not fit 8 slabs.
inline int interact_warps(size_t table, size_t slab, size_t* smem) {
  for (int w = kIWarps; w >= 1; w >>= 1) {
    *smem = (table + (size_t)w * slab) * sizeof(float);
    if (*smem <= kIMaxSmem) return w;
  }
  return 0;
}
}  // namespace

extern "C" int tzk_col_gather_sum(const float* const* srcs_host, const int64_t* src_ld_host, int32_t n_src,
                                  const int32_t* col_start, const int32_t* col_src, const int32_t* col_srccol,
                                  int32_t C, int64_t rows, float* out, int64_t ld_out, tzk_stream_t stream) {
  TZK_REQUIRE(C >= 0 && rows >= 0, "col_gather_sum: negative size");
  if (C == 0 || rows == 0) return 0;
  TZK_REQUIRE(srcs_host && src_ld_host && col_start && col_src && col_srccol && out,
              "col_gather_sum: NULL argument");
  TZK_REQUIRE(n_src >= 1 && n_src <= kMaxSrc, "col_gather_sum: n_src=%d out of range [1,%d]", n_src, kMaxSrc);
  SrcTable srcs;
  for (int i = 0; i < kMaxSrc; ++i) {
    srcs.p[i] = i < n_src ? srcs_host[i] : nullptr;
    srcs.ld[i] = i < n_src ? src_ld_host[i] : 0;
  }
  col_gather_sum_kernel<<<grid_for(rows * C, kThreads, kSmCountH100 * 16), kThreads, 0, as_stream(stream)>>>(
      srcs, col_start, col_src, col_srccol, C, rows, out, ld_out);
  TZK_CHECK_LAUNCH("col_gather_sum_kernel");
  return 0;
}

extern "C" int tzk_jagged_to_padded(const float* values, const int64_t* offsets, int32_t B, int32_t T,
                                    int32_t D, float* out, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && T >= 0 && D >= 1, "jagged_to_padded: bad sizes");
  if (B == 0 || T == 0) return 0;
  TZK_REQUIRE(offsets && out, "jagged_to_padded: NULL argument");
  jagged_to_padded_kernel<<<grid_for((int64_t)B * T * D, kThreads, kSmCountH100 * 16), kThreads, 0,
                            as_stream(stream)>>>(values, offsets, B, T, D, out);
  TZK_CHECK_LAUNCH("jagged_to_padded_kernel");
  return 0;
}

extern "C" int tzk_padded_to_jagged(const float* grad_out, const int64_t* offsets, int32_t B, int32_t T,
                                    int32_t D, int64_t nnz, float* grad_values, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && T >= 0 && D >= 1 && nnz >= 0, "padded_to_jagged: bad sizes");
  if (nnz == 0) return 0;
  TZK_REQUIRE(B > 0 && offsets && grad_values && (T == 0 || grad_out), "padded_to_jagged: NULL argument");
  padded_to_jagged_kernel<<<grid_for(nnz * D, kThreads, kSmCountH100 * 16), kThreads, 0, as_stream(stream)>>>(
      grad_out, offsets, B, T, D, nnz, grad_values);
  TZK_CHECK_LAUNCH("padded_to_jagged_kernel");
  return 0;
}

extern "C" int tzk_fm_fwd(const float* x, int64_t ld_x, int64_t B, int32_t N, int32_t D, float* y,
                          int64_t ld_y, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && N >= 0 && D >= 1, "fm_fwd: bad sizes");
  if (B == 0) return 0;
  TZK_REQUIRE(x && y, "fm_fwd: NULL argument");
  fm_fwd_kernel<<<grid_for(B * D, kThreads, kSmCountH100 * 16), kThreads, 0, as_stream(stream)>>>(
      x, ld_x, B, N, D, y, ld_y);
  TZK_CHECK_LAUNCH("fm_fwd_kernel");
  return 0;
}

extern "C" int tzk_fm_bwd(const float* x, int64_t ld_x, const float* dy, int64_t ld_dy, int64_t B, int32_t N,
                          int32_t D, float* dx, int64_t ld_dx, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && N >= 0 && D >= 1, "fm_bwd: bad sizes");
  if (B == 0) return 0;
  TZK_REQUIRE(x && dy && dx, "fm_bwd: NULL argument");
  fm_bwd_kernel<<<grid_for(B * D, kThreads, kSmCountH100 * 16), kThreads, 0, as_stream(stream)>>>(
      x, ld_x, dy, ld_dy, B, N, D, dx, ld_dx);
  TZK_CHECK_LAUNCH("fm_bwd_kernel");
  return 0;
}

static int interact_check(const char* who, const float* dense, int64_t ld_dense, const float* sparse,
                          int64_t ld_sparse, int64_t B, int32_t Ns, int32_t D) {
  TZK_REQUIRE(B >= 0 && Ns >= 1 && D >= 4, "%s: bad sizes", who);
  TZK_REQUIRE(D % 4 == 0 && D <= 128, "%s: D=%d must be a multiple of 4 and <= 128", who, D);
  TZK_REQUIRE(Ns + (dense != nullptr) <= 64, "%s: more than 64 interacting features", who);
  TZK_REQUIRE(sparse != nullptr, "%s: sparse is NULL", who);
  TZK_REQUIRE(((uintptr_t)sparse % 16 == 0) && (ld_sparse % 4 == 0), "%s: sparse must be 16-B aligned", who);
  TZK_REQUIRE(!dense || (((uintptr_t)dense % 16 == 0) && (ld_dense % 4 == 0)), "%s: dense must be 16-B aligned",
              who);
  return 0;
}

extern "C" int tzk_dot_interact_fwd(const float* dense, int64_t ld_dense, const float* sparse,
                                    int64_t ld_sparse, int64_t B, int32_t Ns, int32_t D, int32_t copy_dense,
                                    int32_t copy_sparse, int32_t p_pad, float* out, int64_t ld_out,
                                    tzk_stream_t stream) {
  int rc = interact_check("dot_interact_fwd", dense, ld_dense, sparse, ld_sparse, B, Ns, D);
  if (rc) return rc;
  if (B == 0) return 0;
  TZK_REQUIRE(out, "dot_interact_fwd: out is NULL");
  const int N = Ns + (dense != nullptr);
  const int Np = (N + 3) & ~3;
  const int P = N * (N - 1) / 2;
  TZK_REQUIRE(p_pad >= 0 && p_pad < 4, "dot_interact_fwd: p_pad must be in [0,3]");
  if (use_interact_tc_fwd() && tzk_itc::covers(dense, ld_dense, ld_sparse, Ns, D, copy_dense, copy_sparse, p_pad, out, ld_out)) {
    tzk_itc::dot_interact27_fwd_tc_kernel<<<tzk_itc::grid_for(B, kSmCountH100 * 8), tzk_itc::kWarps * 32,
                                            tzk_itc::fwd_smem(), as_stream(stream)>>>(dense, ld_dense, sparse, ld_sparse,
                                                                                      B, out, ld_out);
    TZK_CHECK_LAUNCH("dot_interact27_fwd_tc_kernel");
    return 0;
  }
  const int aligned = (((P + p_pad) % 4) == 0) && (ld_out % 4 == 0) && ((uintptr_t)out % 16 == 0);
  const int nb = Np / 4, n_blocks = nb * (nb + 1) / 2;
  size_t smem = 0;
  const int warps = interact_warps((size_t)((n_blocks + 7) / 8) * 4, (size_t)Np * (D + 4) + ((P + 3 + 4) & ~3), &smem);
  TZK_REQUIRE(warps > 0, "dot_interact_fwd: N=%d, D=%d needs %zu B of shared memory with one warp, more than %zu", N, D,
              smem, kIMaxSmem);
#define TZK_IFWD3(DT_, ONE_, NT_)                                                                              \
  do {                                                                                                       \
    if (smem > 48 * 1024 &&                                                                                  \
        cudaFuncSetAttribute(dot_interact_fwd_kernel<DT_, ONE_, NT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                             (int)smem) != cudaSuccess) {                                                    \
      TZK_REQUIRE(false, "dot_interact_fwd: %zu B of shared memory refused: %s", smem,                       \
                  cudaGetErrorString(cudaGetLastError()));                                                   \
    }                                                                                                        \
    dot_interact_fwd_kernel<DT_, ONE_, NT_><<<grid_for(B, warps, kSmCountH100 * 8), warps * 32, smem,         \
                                              as_stream(stream)>>>(                                          \
        dense, ld_dense, sparse, ld_sparse, B, Ns, D, copy_dense, copy_sparse, p_pad, aligned, out, ld_out); \
  } while (0)
#define TZK_IFWD2(DT_, ONE_)                                                   \
  do {                                                                         \
    if (DT_ == 16 && ONE_ && N == 27 && dense) TZK_IFWD3(16, true, 27);        \
    else TZK_IFWD3(DT_, ONE_, 0);                                              \
  } while (0)
#define TZK_IFWD(DT_)                          \
  do {                                         \
    if (n_blocks <= 32) TZK_IFWD2(DT_, true);  \
    else TZK_IFWD2(DT_, false);                \
  } while (0)
  switch (D) {
    case 8: TZK_IFWD(8); break;
    case 16: TZK_IFWD(16); break;
    case 32: TZK_IFWD(32); break;
    case 64: TZK_IFWD(64); break;
    default: TZK_IFWD(0); break;
  }
#undef TZK_IFWD
#undef TZK_IFWD2
#undef TZK_IFWD3
  TZK_CHECK_LAUNCH("dot_interact_fwd_kernel");
  return 0;
}

extern "C" int tzk_dot_interact_bwd(const float* dense, int64_t ld_dense, const float* sparse,
                                    int64_t ld_sparse, const float* d_out, int64_t ld_dout, int64_t B,
                                    int32_t Ns, int32_t D, int32_t copy_dense, int32_t copy_sparse, int32_t p_pad,
                                    float* d_dense, int64_t ld_ddense, float* d_sparse, int64_t ld_dsparse,
                                    tzk_stream_t stream) {
  int rc = interact_check("dot_interact_bwd", dense, ld_dense, sparse, ld_sparse, B, Ns, D);
  if (rc) return rc;
  if (B == 0) return 0;
  TZK_REQUIRE(d_out && d_sparse && (!dense || d_dense), "dot_interact_bwd: NULL argument");
  TZK_REQUIRE(((uintptr_t)d_sparse % 16 == 0) && (ld_dsparse % 4 == 0) &&
                  (!dense || (((uintptr_t)d_dense % 16 == 0) && (ld_ddense % 4 == 0))),
              "dot_interact_bwd: gradient outputs must be 16-B aligned");
  const int N = Ns + (dense != nullptr);
  const int Np = (N + 3) & ~3;
  const int P = N * (N - 1) / 2;
  TZK_REQUIRE(p_pad >= 0 && p_pad < 4, "dot_interact_bwd: p_pad must be in [0,3]");
  if (use_interact_tc_bwd() && tzk_itc::covers(dense, ld_dense, ld_sparse, Ns, D, copy_dense, copy_sparse, p_pad, d_out, ld_dout)) {
    tzk_itc::dot_interact27_bwd_tc_kernel<<<tzk_itc::grid_for(B, kSmCountH100 * 8), tzk_itc::kWarps * 32,
                                            tzk_itc::bwd_smem(), as_stream(stream)>>>(
        dense, ld_dense, sparse, ld_sparse, d_out, ld_dout, B, d_dense, ld_ddense, d_sparse, ld_dsparse);
    TZK_CHECK_LAUNCH("dot_interact27_bwd_tc_kernel");
    return 0;
  }
  const int aligned = (((P + p_pad) % 4) == 0) && (ld_dout % 4 == 0) && ((uintptr_t)d_out % 16 == 0);
  size_t smem = 0;
  const int warps = interact_warps((size_t)((P + 7) / 8) * 4, (size_t)Np * (D + 4) + (size_t)Np * (Np + 8), &smem);
  TZK_REQUIRE(warps > 0, "dot_interact_bwd: N=%d, D=%d needs %zu B of shared memory with one warp, more than %zu", N, D,
              smem, kIMaxSmem);
#define TZK_IBWD(DT_, NT_)                                                                                    \
  do {                                                                                                       \
    if (smem > 48 * 1024 &&                                                                                  \
        cudaFuncSetAttribute(dot_interact_bwd_kernel<DT_, NT_>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                             (int)smem) != cudaSuccess) {                                                    \
      TZK_REQUIRE(false, "dot_interact_bwd: %zu B of shared memory refused: %s", smem,                       \
                  cudaGetErrorString(cudaGetLastError()));                                                   \
    }                                                                                                        \
    dot_interact_bwd_kernel<DT_, NT_><<<grid_for(B, warps, kSmCountH100 * 8), warps * 32, smem,               \
                                        as_stream(stream)>>>(                                                \
        dense, ld_dense, sparse, ld_sparse, d_out, ld_dout, B, Ns, D, copy_dense, copy_sparse, p_pad, aligned, \
        d_dense, ld_ddense, d_sparse, ld_dsparse);                                                           \
  } while (0)
  switch (D) {
    case 8: TZK_IBWD(8, 0); break;
    case 16:
      if (N == 27 && dense) TZK_IBWD(16, 27);   // DLRM-Criteo: 26 sparse + the dense row, fully unrolled
      else TZK_IBWD(16, 0);
      break;
    case 32: TZK_IBWD(32, 0); break;
    case 64: TZK_IBWD(64, 0); break;
    default: TZK_IBWD(0, 0); break;
  }
#undef TZK_IBWD
  TZK_CHECK_LAUNCH("dot_interact_bwd_kernel");
  return 0;
}

// ---------------------------------------------------------------------------------------------------
// Dense-tower helpers (caller-side of the hot path: tzrec/modules/mlp.py Perceptron = Linear -> ReLU).
// The GEMMs are library calls (dense_gemm.py); these two kernels fuse what PyTorch runs as four separate
// passes around them: bias add + ReLU, and ReLU backward + bias gradient (column sum).
// ---------------------------------------------------------------------------------------------------
namespace {
__global__ void __launch_bounds__(kThreads)
bias_act_kernel(float* __restrict__ y, int64_t ld, const float* __restrict__ bias, int64_t M, int N, int relu) {
  const int64_t n = M * N;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int64_t r = i / N;
    const int c = (int)(i - r * N);
    float v = y[r * ld + c] + (bias ? __ldg(bias + c) : 0.f);
    if (relu) v = v > 0.f ? v : 0.f;
    y[r * ld + c] = v;
  }
}

// 16-B variant: N % 4 == 0, ld % 4 == 0, y 16-B aligned, M * N / 4 < 2^31
__global__ void __launch_bounds__(kThreads)
bias_act_vec_kernel(float* __restrict__ y, int64_t ld, const float* __restrict__ bias, int n4_total, int N4,
                    int relu) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4_total; i += stride) {
    const int r = i / N4, c4 = i - r * N4;
    float4* p = reinterpret_cast<float4*>(y + (int64_t)r * ld) + c4;
    float4 v = *p;
    if (bias) {
      const float4 b = __ldg(reinterpret_cast<const float4*>(bias) + c4);
      v.x += b.x; v.y += b.y; v.z += b.z; v.w += b.w;
    }
    if (relu) {
      v.x = v.x > 0.f ? v.x : 0.f; v.y = v.y > 0.f ? v.y : 0.f;
      v.z = v.z > 0.f ? v.z : 0.f; v.w = v.w > 0.f ? v.w : 0.f;
    }
    *p = v;
  }
}

constexpr int kSlabRows = 128;
// N divides 256: thread (tid / N, tid % N) walks its rows of the slab; fixed-order reduction over row groups
__global__ void __launch_bounds__(kThreads)
act_bwd_colsum_kernel(const float* __restrict__ dy, int64_t ld_dy, const float* __restrict__ y, int64_t ld_y,
                      int64_t M, int N, int relu, float* __restrict__ dz, int64_t ld_dz,
                      float* __restrict__ partial) {
  __shared__ float red[kThreads];
  const int rg = kThreads / N;           // row groups per pass
  const int c = threadIdx.x % N, r0 = threadIdx.x / N;
  const int64_t row_lo = (int64_t)blockIdx.x * kSlabRows;
  const int64_t row_hi = row_lo + kSlabRows < M ? row_lo + kSlabRows : M;
  float acc = 0.f;
#pragma unroll 4
  for (int64_t r = row_lo + r0; r < row_hi; r += rg) {
    float g = __ldg(dy + r * ld_dy + c);
    if (relu && !(__ldg(y + r * ld_y + c) > 0.f)) g = 0.f;
    if (dz) dz[r * ld_dz + c] = g;
    acc += g;
  }
  red[threadIdx.x] = acc;
  __syncthreads();
  if (r0 == 0) {
    float s = 0.f;
    for (int k = 0; k < rg; ++k) s += red[k * N + c];
    partial[(int64_t)blockIdx.x * N + c] = s;
  }
}

// 32 columns x 8 partial-groups per CTA, fixed-order fold: deterministic
__global__ void __launch_bounds__(256)
colsum_final_kernel(const float* __restrict__ partial, int64_t n_blocks, int N, float* __restrict__ out) {
  __shared__ float red[8][32];
  const int o = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + o;
  float s = 0.f;
  if (c < N) {
    int64_t b = g;
    for (; b + 24 < n_blocks; b += 32) {
      const float a0 = partial[b * N + c], a1 = partial[(b + 8) * N + c];
      const float a2 = partial[(b + 16) * N + c], a3 = partial[(b + 24) * N + c];
      s += a0; s += a1; s += a2; s += a3;
    }
    for (; b < n_blocks; b += 8) s += partial[b * N + c];
  }
  red[g][o] = s;
  __syncthreads();
  if (g == 0 && c < N) {
    float r = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) r += red[k][o];
    out[c] = r;
  }
}
}  // namespace

void tzk::colsum_final(const float* partial, int64_t n_blocks, int N, float* colsum, cudaStream_t st) {
  colsum_final_kernel<<<(N + 31) / 32, 256, 0, st>>>(partial, n_blocks, N, colsum);
}

extern "C" int tzk_bias_act(float* y, int64_t ld_y, const float* bias, int64_t M, int32_t N, int32_t relu,
                            tzk_stream_t stream) {
  TZK_REQUIRE(M >= 0 && N >= 1, "bias_act: bad sizes");
  if (M == 0) return 0;
  TZK_REQUIRE(y != nullptr, "bias_act: y is NULL");
  const bool vec = (N % 4 == 0) && (ld_y % 4 == 0) && ((uintptr_t)y % 16 == 0) &&
                   (!bias || (uintptr_t)bias % 16 == 0) && (M * N / 4 < ((int64_t)1 << 31));
  if (vec)
    bias_act_vec_kernel<<<grid_for(M * N / 4, kThreads, kSmCountH100 * 16), kThreads, 0, as_stream(stream)>>>(
        y, ld_y, bias, (int)(M * N / 4), N / 4, relu);
  else
    bias_act_kernel<<<grid_for(M * N, kThreads, kSmCountH100 * 16), kThreads, 0, as_stream(stream)>>>(y, ld_y, bias,
                                                                                                    M, N, relu);
  TZK_CHECK_LAUNCH("bias_act_kernel");
  return 0;
}

extern "C" size_t tzk_act_bwd_colsum_workspace_bytes(int64_t M, int32_t N) {
  return (size_t)ceil_div64(M < 1 ? 1 : M, kSlabRows) * (size_t)(N < 1 ? 1 : N) * sizeof(float);
}

extern "C" int tzk_act_bwd_colsum(const float* dy, int64_t ld_dy, const float* y, int64_t ld_y, int64_t M,
                                  int32_t N, int32_t relu, float* dz, int64_t ld_dz, float* colsum,
                                  void* workspace, size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(M >= 1 && N >= 1, "act_bwd_colsum: bad sizes");
  TZK_REQUIRE(N <= kThreads && kThreads % N == 0, "act_bwd_colsum: N=%d must divide %d", N, kThreads);
  TZK_REQUIRE(dy && colsum && (!relu || y), "act_bwd_colsum: NULL argument");
  TZK_REQUIRE(workspace && workspace_bytes >= tzk_act_bwd_colsum_workspace_bytes(M, N),
              "act_bwd_colsum: workspace too small");
  const int64_t nb = ceil_div64(M, kSlabRows);
  float* partial = static_cast<float*>(workspace);
  act_bwd_colsum_kernel<<<(unsigned)nb, kThreads, 0, as_stream(stream)>>>(dy, ld_dy, y, ld_y, M, N, relu, dz, ld_dz,
                                                                          partial);
  TZK_CHECK_LAUNCH("act_bwd_colsum_kernel");
  colsum_final(partial, nb, N, colsum, as_stream(stream));
  TZK_CHECK_LAUNCH("colsum_final_kernel");
  return 0;
}
