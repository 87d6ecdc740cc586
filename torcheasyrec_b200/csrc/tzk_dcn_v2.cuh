// tzk_dcn_v2.cuh — DCN-v2's low-rank cross network (tzrec/modules/interaction.py CrossV2) on the tensor cores.
//
//   x_{l+1} = x0 * (V_l (U_l x_l) + c_l) + x_l,   U_l [r, D], V_l [D, r], l = 0 .. L-1,   y = x_L
//
// Every tile product is mma.sync m16n8k8 with the 3xTF32 split (x = hi + lo, acc += lo*hi + hi*lo + hi*hi): fp32-level
// results.  The weights are split once per call by prep_kernel into B fragments in `work` (four arrays, below), laid
// out so that a lane's fragment is one 16-B load {b0 hi, b1 hi, b0 lo, b1 lo} and a warp's is 512 contiguous bytes.
// r is zero-padded to r8 (a multiple of 8) and D to D8, so the padded products add exact zeros.
//
//   fwd        a warp per 16-row tile, up to four warps per CTA going through the layers together.  x_l lives in
//              shared memory [16][D8 + 4] across all layers; per layer v = x_l U_l^T (K = D8) goes out to HBM and into
//              a [16][r8 + 4] tile, w = v V_l^T + c_l (K = r8) and the epilogue does x_l <- x0 * w + x_l in place.
//              Only y and v [B, L r] are written.
//   bwd_data   tiles as fwd, dx in shared memory.  For l = L-1 .. 0: w_l = V_l v_l + c_l, dx0 += dx_{l+1} * w_l (in
//              the dx0 rows, which stay in L2); dv_l = (dx_{l+1} * x0) V_l (K = D8; the product is formed as the A
//              fragment is read); dx_l = dx_{l+1} + dv_l U_l (K = r8).  dx0 += dx_0 at the end.  x_l is never needed.
//   Both are instantiated per r8 / 8, so the fragment arrays of a rank take only the registers it needs.
//   bwd_weight work item (32-column block, batch chunk), four warps over 64-row tiles.  Over a column block every
//              quantity is local once v and dv are known: x_l[cols] from x0[cols] and w_j[cols] (j < l), dx_{l+1}[cols]
//              = dy[cols] + sum_{j>l} dv_j U_j[:, cols].  Per layer dU_l[:, cols] += dv_l^T x_l and
//              dV_l[cols, :]^T += v_l^T g_l (g_l = dx_{l+1} * x0; M = r, N = 32 columns, K = the tile's 64 rows) go into
//              the CTA's accumulators in shared memory, each 16 x 8 output tile owned by one warp, and dc_l[cols] +=
//              the column sums of g_l, rows in order.  Chunk k writes row k of the partials;
//              tzk_batch_sum::reduce adds the rows in chunk order.  The bits depend only on the chunk count.
//
// nvcc builds this in tzk_dcn_v2.cu with tzk_sm90_ptx.h; g++ with tests/native/cuda_cpu_shim.h and sm90_cpu_emu.h
// (emulated mma.sync) runs the same source in tests/test_dcn_v2_cpu.py.  The includer provides tf32_bits and mma_tf32.
#pragma once
#include <stdint.h>

#include "../../include/tzk.h"
#include "tzk_batch_sum.cuh"
#include "tzk_launch.cuh"

namespace tzk_dcn_v2 {
constexpr int kMaxD = 512, kMaxR = 64, kMaxL = TZK_DCN_V2_MAX_LAYERS;
constexpr int kMaxNT = kMaxR / 8;             // n-tiles (or k-steps) over r8
constexpr int kNB = 32;                       // bwd_weight column block
constexpr int kLdn = kNB + 8;                 // row pitch of its [64][kNB] tiles: conflict-free B-fragment reads
constexpr int kWarpsW = 4, kRowsW = 16 * kWarpsW;
constexpr size_t kMaxSmem = 227 * 1024;       // H100's opt-in shared memory per CTA
enum { kUb = 0, kVb = 1, kVt = 2, kUt = 3 };  // fragment arrays in `work`

__host__ __device__ inline int r8(const tzk_dcn_v2_args& a) { return (a.r + 7) & ~7; }
__host__ __device__ inline int r16(const tzk_dcn_v2_args& a) { return (a.r + 15) & ~15; }
__host__ __device__ inline int d8(const tzk_dcn_v2_args& a) { return (a.D + 7) & ~7; }
__host__ __device__ inline int ldx(const tzk_dcn_v2_args& a) { return d8(a) + 4; }   // conflict-free A-fragment reads
__host__ __device__ inline int ldv(const tzk_dcn_v2_args& a) { return r8(a) + 4; }
inline int64_t work_floats(const tzk_dcn_v2_args& a) { return (int64_t)8 * a.L * r8(a) * d8(a); }
__host__ __device__ inline int64_t param_floats(const tzk_dcn_v2_args& a) { return (int64_t)a.L * a.D * (2 * a.r + 1); }
// bwd_weight accumulators of one layer: dU [r16][kNB], dV^T [r16][kNB], dc [kNB]
__host__ __device__ inline int acc_floats(const tzk_dcn_v2_args& a) { return (2 * r16(a) + 1) * kNB; }

__host__ __device__ inline int tile_warps(const tzk_dcn_v2_args& a, int pass);
__host__ __device__ inline int tile_floats(const tzk_dcn_v2_args& a, int pass);
inline size_t smem_bytes(const tzk_dcn_v2_args& a, int pass) {
  if (pass < 2) return (size_t)tile_warps(a, pass) * tile_floats(a, pass) * sizeof(float);
  return ((size_t)(a.L + 1) * kRowsW * kLdn + (size_t)a.L * acc_floats(a) + kWarpsW * kNB) * sizeof(float);
}

// the descriptions the kernels cover (the Python side's Fn.cross_v2_usable states the same for whole modules)
inline int check(const tzk_dcn_v2_args& a, int pass) {
  if (a.B < 0 || a.B >= ((int64_t)1 << 31) || pass < 0 || pass > 2) return 1;
  if (a.D < 1 || a.D > kMaxD || a.L < 1 || a.L > kMaxL || a.r < 1 || a.r > kMaxR) return 1;
  if (smem_bytes(a, pass) > kMaxSmem) return 1;
  if (a.B == 0) return 0;
  if (!a.x0 || !a.wu || !a.wv || !a.bias || !a.work || ((uintptr_t)a.work & 15u) != 0 || !a.v) return 1;
  if (pass == 0) return a.y ? 0 : 1;
  if (!a.dy || !a.dv) return 1;
  return (pass == 2 || a.dx0) ? 0 : 1;
}

struct Frag { uint32_t x, y, z, w; };         // {b0 hi, b1 hi, b0 lo, b1 lo}

// fragment array q of layer l: n-tiles x k-steps x 32 lanes.  B[k][n] of the four products:
//   kUb  v = x U^T     B[k = d][n = j] = U[j][d]   N = r8, K = D8   (fwd)
//   kVb  w = v V^T     B[k = j][n = d] = V[d][j]   N = D8, K = r8   (fwd, bwd_data, bwd_weight)
//   kVt  dv = g V      B[k = d][n = j] = V[d][j]   N = r8, K = D8   (bwd_data)
//   kUt  dx += dv U    B[k = j][n = d] = U[j][d]   N = D8, K = r8   (bwd_data, bwd_weight)
__host__ __device__ inline int frag_ks(const tzk_dcn_v2_args& a, int q) { return (q == kUb || q == kVt ? d8(a) : r8(a)) / 8; }
__device__ inline const Frag* frags(const tzk_dcn_v2_args& a, int q, int l) {
  const int64_t per = (int64_t)r8(a) * d8(a) * 2;
  return reinterpret_cast<const Frag*>(a.work + ((int64_t)q * a.L + l) * per);
}

__device__ __forceinline__ void split(float x, uint32_t& hi, uint32_t& lo) {
  hi = tf32_bits(x);
  lo = tf32_bits(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma3(float (&c)[4], const uint32_t (&ah)[4], const uint32_t (&al)[4], const Frag& b) {
  const uint32_t bh[2] = {b.x, b.y}, bl[2] = {b.z, b.w};
  mma_tf32(c, al, bh);
  mma_tf32(c, ah, bl);
  mma_tf32(c, ah, bh);
}
__device__ __forceinline__ Frag ldfrag(const Frag* p) {
#ifdef TZK_CPU_SHIM
  return *p;
#else
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  return Frag{u.x, u.y, u.z, u.w};
#endif
}
// A fragment (16 x 8 at column k0) of a row-major shared-memory tile T [16][ld]
__device__ __forceinline__ void afrag(const float* T, int ld, int k0, int g, int t, uint32_t (&h)[4], uint32_t (&l)[4]) {
  split(T[g * ld + k0 + t], h[0], l[0]);
  split(T[(g + 8) * ld + k0 + t], h[1], l[1]);
  split(T[g * ld + k0 + t + 4], h[2], l[2]);
  split(T[(g + 8) * ld + k0 + t + 4], h[3], l[3]);
}

// the weights as B fragments, for the arrays in `mask`
__global__ void __launch_bounds__(256) prep_kernel(const __grid_constant__ tzk_dcn_v2_args a, int mask) {
  const int D = a.D, r = a.r;
  const int64_t per = (int64_t)r8(a) * d8(a) / 2;          // fragments (lanes included) of one layer's array
  const int64_t n = (int64_t)4 * a.L * per;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int q = (int)(i / (a.L * per));
    if (!((mask >> q) & 1)) continue;
    const int64_t rem = i % (a.L * per);
    const int l = (int)(rem / per);
    const int64_t f = rem % per;
    const int lane = (int)(f % 32), KS = frag_ks(a, q);
    const int ks = (int)(f / 32 % KS), nt = (int)(f / 32 / KS);
    const int n0 = 8 * nt + lane / 4, k0 = 8 * ks + lane % 4;
    const float* U = a.wu + (int64_t)l * r * D;
    const float* V = a.wv + (int64_t)l * D * r;
    float b[2];
    for (int h = 0; h < 2; ++h) {
      const int k = k0 + 4 * h;
      float x = 0.f;
      if (q == kUb) x = (n0 < r && k < D) ? U[n0 * D + k] : 0.f;
      else if (q == kVb) x = (n0 < D && k < r) ? V[n0 * r + k] : 0.f;
      else if (q == kVt) x = (k < D && n0 < r) ? V[k * r + n0] : 0.f;
      else x = (k < r && n0 < D) ? U[k * D + n0] : 0.f;
      b[h] = x;
    }
    uint32_t h0, l0, h1, l1;
    split(b[0], h0, l0);
    split(b[1], h1, l1);
    reinterpret_cast<Frag*>(a.work)[((int64_t)q * a.L + l) * per + f] = Frag{h0, h1, l0, l1};
  }
}

// v-tile T [16][ld] of rows b0.. of a [B, L r] array at layer l (zeros beyond B and r)
__device__ inline void load_rank_tile(const tzk_dcn_v2_args& a, const float* src, int64_t b0, int l, float* T, int lane) {
  const int R8 = r8(a), ld = ldv(a), LR = a.L * a.r;
  for (int e = lane; e < 16 * R8; e += 32) {
    const int rr = e / R8, j = e % R8;
    T[rr * ld + j] = (b0 + rr < a.B && j < a.r) ? src[(b0 + rr) * LR + l * a.r + j] : 0.f;
  }
}

// v-like accumulators [16][r8] (nt < r8 / 8) -> T and the rows' entries of dst [B, L r] at layer l
template <int NT>
__device__ inline void store_rank_tile(const tzk_dcn_v2_args& a, const float (&acc)[NT][4], float* dst, int64_t b0,
                                       int l, float* T, int g, int t) {
  const int ld = ldv(a), LR = a.L * a.r;
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int rr = g + 8 * (q >> 1), j = 8 * nt + 2 * t + (q & 1);
      T[rr * ld + j] = acc[nt][q];
      if (j < a.r && b0 + rr < a.B) dst[(b0 + rr) * LR + l * a.r + j] = acc[nt][q];
    }
  }
}

// The rank-K product of a warp's 16 rows over all D8 columns: W = T F (T [16][r8] in shared memory, F one of the
// N = D8 fragment arrays, K = r8), two n-tiles per step so that their fragment loads and MMA chains overlap.
// epi(rr, n, w) receives every element of rows rr < 16, columns n < D8 once, in a lane-private order.
template <int NT, class Epi>
__device__ __forceinline__ void rank_product(const tzk_dcn_v2_args& a, const float* T, const Frag* F, int lane,
                                             Epi&& epi) {
  const int g = lane >> 2, t = lane & 3, NTd = d8(a) / 8;
  uint32_t vh[NT][4], vl[NT][4];
#pragma unroll
  for (int ks = 0; ks < NT; ++ks)
    if (ks < NT) afrag(T, ldv(a), 8 * ks, g, t, vh[ks], vl[ks]);
  for (int nt = 0; nt < NTd; nt += 2) {
    const int n1 = nt + 1 < NTd ? nt + 1 : nt;          // an odd tail repeats the last tile (its result is dropped)
    Frag b0[NT], b1[NT];
#pragma unroll
    for (int ks = 0; ks < NT; ++ks)
      if (ks < NT) {
        b0[ks] = ldfrag(F + (nt * NT + ks) * 32 + lane);
        b1[ks] = ldfrag(F + (n1 * NT + ks) * 32 + lane);
      }
    float w0[4] = {0.f, 0.f, 0.f, 0.f}, w1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int ks = 0; ks < NT; ++ks)
      if (ks < NT) {
        mma3(w0, vh[ks], vl[ks], b0[ks]);
        mma3(w1, vh[ks], vl[ks], b1[ks]);
      }
#pragma unroll
    for (int q = 0; q < 4; ++q) epi(g + 8 * (q >> 1), 8 * nt + 2 * t + (q & 1), w0[q]);
    if (n1 != nt) {
#pragma unroll
      for (int q = 0; q < 4; ++q) epi(g + 8 * (q >> 1), 8 * n1 + 2 * t + (q & 1), w1[q]);
    }
  }
}

// Warps per CTA of the per-sample kernels: 4 when their tiles fit in shared memory, else 2 or 1.  The warps of a CTA
// take adjacent 16-row tiles and go through the layers together, so each weight fragment is fetched from L2 once for
// all of them.
__host__ __device__ inline int tile_floats(const tzk_dcn_v2_args& a, int) {
  return 16 * ldx(a) + 16 * ldv(a);
}
__host__ __device__ inline int tile_warps(const tzk_dcn_v2_args& a, int pass) {
  const int64_t per = (int64_t)tile_floats(a, pass) * 4;
  return 4 * per <= (int64_t)kMaxSmem ? 4 : 2 * per <= (int64_t)kMaxSmem ? 2 : 1;
}

// dynamic shared memory: smem_bytes(a, 0), tile_warps(a, 0) warps.  CTA g takes the 16 nw-row groups g, g + grid, ..
template <int NT>
__global__ void __launch_bounds__(128, 1) fwd_kernel(const __grid_constant__ tzk_dcn_v2_args a) {
  TZK_DYN_SMEM(float, smem);
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int D = a.D, D8 = d8(a), LD = ldx(a), KSd = D8 / 8;
  float* X = smem + warp * tile_floats(a, 0);
  float* T = X + 16 * LD;
  for (int64_t base = (int64_t)blockIdx.x * 16 * nw; base < a.B; base += (int64_t)gridDim.x * 16 * nw) {
    const int64_t b0 = base + 16 * warp;
    const int rows = a.B - b0 >= 16 ? 16 : a.B - b0 > 0 ? (int)(a.B - b0) : 0;
    const float* x0 = a.x0 + b0 * D;
    for (int e = lane; e < 16 * D8; e += 32) {
      const int rr = e / D8, c = e % D8;
      X[rr * LD + c] = (rr < rows && c < D) ? x0[rr * D + c] : 0.f;
    }
    for (int l = 0; l < a.L; ++l) {
      __syncthreads();
      // v = x_l U_l^T
      const Frag* ub = frags(a, kUb, l);
      float acc[NT][4];
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll 2
      for (int ks = 0; ks < KSd; ++ks) {
        Frag b[NT];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
          if (nt < NT) b[nt] = ldfrag(ub + (nt * KSd + ks) * 32 + lane);
        uint32_t ah[4], al[4];
        afrag(X, LD, 8 * ks, g, t, ah, al);
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
          if (nt < NT) mma3(acc[nt], ah, al, b[nt]);
      }
      store_rank_tile<NT>(a, acc, a.v, b0, l, T, g, t);
      __syncwarp();
      // w = v V_l^T + c_l;  x_l <- x0 * w + x_l
      const float* c = a.bias + (int64_t)l * D;
      rank_product<NT>(a, T, frags(a, kVb, l), lane, [&](int rr, int n, float w) {
        if (rr < rows && n < D) X[rr * LD + n] += __ldg(x0 + rr * D + n) * (w + __ldg(c + n));
      });
      __syncwarp();
    }
    for (int e = lane; e < rows * D; e += 32) a.y[b0 * D + e] = X[(e / D) * LD + e % D];
    __syncwarp();
  }
}

// dynamic shared memory: smem_bytes(a, 1), tile_warps(a, 1) warps; tiles as fwd_kernel.  dx lives in shared memory,
// dx0 accumulates in its output rows (each element owned by one lane) and x0 is read where it is needed.
template <int NT>
__global__ void __launch_bounds__(128, 1) bwd_data_kernel(const __grid_constant__ tzk_dcn_v2_args a) {
  TZK_DYN_SMEM(float, smem);
  const int nw = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int D = a.D, D8 = d8(a), LD = ldx(a), KSd = D8 / 8;
  float* DX = smem + warp * tile_floats(a, 1);
  float* T = DX + 16 * LD;
  for (int64_t base = (int64_t)blockIdx.x * 16 * nw; base < a.B; base += (int64_t)gridDim.x * 16 * nw) {
    const int64_t b0 = base + 16 * warp;
    const int rows = a.B - b0 >= 16 ? 16 : a.B - b0 > 0 ? (int)(a.B - b0) : 0;
    const float* x0 = a.x0 + b0 * D;
    float* dx0 = a.dx0 + b0 * D;
    for (int e = lane; e < 16 * D8; e += 32) {
      const int rr = e / D8, c = e % D8;
      DX[rr * LD + c] = (rr < rows && c < D) ? a.dy[(b0 + rr) * D + c] : 0.f;
    }
    for (int l = a.L - 1; l >= 0; --l) {
      __syncthreads();
      load_rank_tile(a, a.v, b0, l, T, lane);
      __syncwarp();
      // w_l = V_l v_l + c_l;  dx0 += dx_{l+1} * w_l
      const float* c = a.bias + (int64_t)l * D;
      const bool first = l == a.L - 1;
      rank_product<NT>(a, T, frags(a, kVb, l), lane, [&](int rr, int n, float w) {
        if (rr < rows && n < D) {
          const float p = DX[rr * LD + n] * (w + __ldg(c + n));
          dx0[rr * D + n] = first ? p : dx0[rr * D + n] + p;
        }
      });
      // dv_l = (dx_{l+1} * x0) V_l
      {
        const Frag* vt = frags(a, kVt, l);
        float acc[NT][4];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll 2
        for (int ks = 0; ks < KSd; ++ks) {
          Frag b[NT];
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) b[nt] = ldfrag(vt + (nt * KSd + ks) * 32 + lane);
          uint32_t ah[4], al[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int rr = g + 8 * (q & 1), k = 8 * ks + t + 4 * (q >> 1);
            const float xv = (rr < rows && k < D) ? __ldg(x0 + rr * D + k) : 0.f;
            split(DX[rr * LD + k] * xv, ah[q], al[q]);
          }
#pragma unroll
          for (int nt = 0; nt < NT; ++nt) mma3(acc[nt], ah, al, b[nt]);
        }
        __syncwarp();
        store_rank_tile<NT>(a, acc, a.dv, b0, l, T, g, t);
        __syncwarp();
      }
      // dx_l = dx_{l+1} + dv_l U_l
      rank_product<NT>(a, T, frags(a, kUt, l), lane, [&](int rr, int n, float w) { DX[rr * LD + n] += w; });
      __syncwarp();
    }
    for (int e = lane; e < rows * D; e += 32) dx0[e] += DX[(e / D) * LD + e % D];
    __syncwarp();
  }
}

// this warp's A operand of the rank product over K = r8 for its 16 rows from a [B, L r] array S at layer l, in
// fragment order, all k-steps loaded before any is used
template <int NT>
__device__ __forceinline__ void aload_rank(const tzk_dcn_v2_args& a, const float* S, int64_t rb, int l, int g, int t,
                                           float (&x)[NT][4]) {
  const int64_t LR = (int64_t)a.L * a.r;
#pragma unroll
  for (int ks = 0; ks < NT; ++ks)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t row = rb + g + 8 * (q & 1);
      const int k = 8 * ks + t + 4 * (q >> 1);
      x[ks][q] = (row < a.B && k < a.r) ? __ldg(S + row * LR + (int64_t)l * a.r + k) : 0.f;
    }
}

// acc[q] (+)= the rank product of the warp's 16 rows (A operand x) with the column block's four n-tiles of F
template <int NT>
__device__ __forceinline__ void block_product(const tzk_dcn_v2_args& a, const float (&x)[NT][4], const Frag* F, int c0,
                                              int lane, float (&acc)[4][4]) {
  const int nq = d8(a) / 8 - c0 / 8;                   // n-tiles of the block inside D8
#pragma unroll
  for (int ks = 0; ks < NT; ++ks) {
    uint32_t h[4], lo[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) split(x[ks][e], h[e], lo[e]);
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (q < nq) mma3(acc[q], h, lo, ldfrag(F + ((c0 / 8 + q) * NT + ks) * 32 + lane));
  }
}

// dynamic shared memory: smem_bytes(a, 2).  grid (ceil(D / kNB), chunks), kWarpsW warps; partials [chunks][P]
template <int NT>
__global__ void __launch_bounds__(kWarpsW * 32, 1) bwd_weight_kernel(const __grid_constant__ tzk_dcn_v2_args a,
                                                                  float* __restrict__ partials) {
  TZK_DYN_SMEM(float, smem);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
  const int D = a.D, L = a.L, r = a.r, MT = r16(a) / 16, AF = acc_floats(a);
  const int c0 = blockIdx.x * kNB;
  float* X = smem;                                   // [L][64][kLdn] x_l of the tile's rows, then G [64][kLdn]
  float* G = X + (size_t)L * kRowsW * kLdn;
  float* ACC = G + kRowsW * kLdn;                    // per layer: dU [r16][kNB], dV^T [r16][kNB], dc [kNB]
  float* RED = ACC + (size_t)L * AF;                 // [kWarpsW][kNB] the warps' column sums of g_l
  for (int e = tid; e < L * AF; e += blockDim.x) ACC[e] = 0.f;
  const int64_t tiles = (a.B + kRowsW - 1) / kRowsW, K = gridDim.y, k = blockIdx.y;
  const int64_t t_begin = tiles * k / K, t_end = tiles * (k + 1) / K;
  __syncthreads();
  for (int64_t tile = t_begin; tile < t_end; ++tile) {
    const int64_t rb = tile * kRowsW + 16 * warp;   // this warp's 16 rows
    // x0, dy and the running x / dx in accumulator layout: [n-tile q][rows g, g + 8 x columns 2t, 2t + 1]
    float x0f[4][4], dyf[4][4], xf[4][4];
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t row = rb + g + 8 * (e >> 1);
        const int col = c0 + 8 * q + 2 * t + (e & 1);
        const bool in = row < a.B && col < D;
        x0f[q][e] = in ? __ldg(a.x0 + row * D + col) : 0.f;
        dyf[q][e] = in ? __ldg(a.dy + row * D + col) : 0.f;
        xf[q][e] = x0f[q][e];
      }
    // x_0 .. x_{L-1} of the column block into X
    for (int j = 0; j < L; ++j) {
      float* Xj = X + (size_t)j * kRowsW * kLdn;
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int e = 0; e < 4; ++e) Xj[(16 * warp + g + 8 * (e >> 1)) * kLdn + 8 * q + 2 * t + (e & 1)] = xf[q][e];
      if (j == L - 1) break;
      float w[4][4];
#pragma unroll
      for (int q = 0; q < 4; ++q) w[q][0] = w[q][1] = w[q][2] = w[q][3] = 0.f;
      float va[NT][4];
      aload_rank<NT>(a, a.v, rb, j, g, t, va);
      block_product<NT>(a, va, frags(a, kVb, j), c0, lane, w);
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = c0 + 8 * q + 2 * t + (e & 1);
          xf[q][e] += x0f[q][e] * (w[q][e] + (col < D ? __ldg(a.bias + (int64_t)j * D + col) : 0.f));
        }
    }
    // dyf becomes dx_{l+1}: dx_L = dy
    for (int l = L - 1; l >= 0; --l) {
      float cs[4][2];                                // this warp's column sums of g_l: rows g, g + 8, then over g
#pragma unroll
      for (int q = 0; q < 4; ++q) {
#pragma unroll
        for (int e = 0; e < 4; ++e)
          G[(16 * warp + g + 8 * (e >> 1)) * kLdn + 8 * q + 2 * t + (e & 1)] = dyf[q][e] * x0f[q][e];
        cs[q][0] = dyf[q][0] * x0f[q][0] + dyf[q][2] * x0f[q][2];
        cs[q][1] = dyf[q][1] * x0f[q][1] + dyf[q][3] * x0f[q][3];
      }
#pragma unroll
      for (int o = 4; o < 32; o <<= 1)
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          cs[q][0] += __shfl_xor_sync(0xffffffffu, cs[q][0], o);
          cs[q][1] += __shfl_xor_sync(0xffffffffu, cs[q][1], o);
        }
      if (g == 0) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          RED[warp * kNB + 8 * q + 2 * t] = cs[q][0];
          RED[warp * kNB + 8 * q + 2 * t + 1] = cs[q][1];
        }
      }
      if (l > 0) {                                    // dx_l = dx_{l+1} + dv_l U_l[:, cols]
        float w[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q) w[q][0] = w[q][1] = w[q][2] = w[q][3] = 0.f;
        float da[NT][4];
        aload_rank<NT>(a, a.dv, rb, l, g, t, da);
        block_product<NT>(a, da, frags(a, kUt, l), c0, lane, w);
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int e = 0; e < 4; ++e) dyf[q][e] += w[q][e];
      }
      __syncthreads();
      // dU_l[:, cols] += dv_l^T x_l and dV_l^T[:, cols] += v_l^T g_l over the tile's 64 rows; warp w owns jobs w, w + 4, ..
      const float* Xl = X + (size_t)l * kRowsW * kLdn;
      float* acc_l = ACC + (size_t)l * AF;
      for (int job = warp; job < 2 * MT; job += kWarpsW) {
        const int kind = job / MT, mt = job % MT;     // kind 0: dU (dv, x_l), 1: dV^T (v, g_l)
        const float* S = kind == 0 ? a.dv : a.v;
        const float* Tb = kind == 0 ? Xl : G;
        float* out = acc_l + kind * r16(a) * kNB;
        float c[4][4];
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int e = 0; e < 4; ++e) c[q][e] = out[(16 * mt + g + 8 * (e >> 1)) * kNB + 8 * q + 2 * t + (e & 1)];
#pragma unroll 2
        for (int ks = 0; ks < kRowsW / 8; ++ks) {
          // A[m = j][k = row]: S[row][l r + j]
          uint32_t ah[4], al[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int j = 16 * mt + g + 8 * (e & 1);
            const int64_t row = tile * kRowsW + 8 * ks + t + 4 * (e >> 1);
            split((row < a.B && j < r) ? __ldg(S + row * L * r + (int64_t)l * r + j) : 0.f, ah[e], al[e]);
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            // B[k = row][n = col]: Tb[row][col]
            Frag b;
            split(Tb[(8 * ks + t) * kLdn + 8 * q + g], b.x, b.z);
            split(Tb[(8 * ks + t + 4) * kLdn + 8 * q + g], b.y, b.w);
            mma3(c[q], ah, al, b);
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q)
#pragma unroll
          for (int e = 0; e < 4; ++e) out[(16 * mt + g + 8 * (e >> 1)) * kNB + 8 * q + 2 * t + (e & 1)] = c[q][e];
      }
      if (tid < kNB) {                                // dc_l[cols] += the warps' column sums, warps in order
        float s = acc_l[2 * r16(a) * kNB + tid];
        for (int w = 0; w < kWarpsW; ++w) s += RED[w * kNB + tid];
        acc_l[2 * r16(a) * kNB + tid] = s;
      }
      __syncthreads();
    }
  }
  // this chunk's share of dU [L][r][D] | dV [L][D][r] | dc [L][D], columns c0 .. c0 + kNB
  float* row = partials + (int64_t)k * param_floats(a);
  float* pU = row;
  float* pV = row + (int64_t)L * r * D;
  float* pc = pV + (int64_t)L * D * r;
  for (int e = tid; e < L * r * kNB; e += blockDim.x) {
    const int l = e / (r * kNB), j = e / kNB % r, cc = e % kNB, col = c0 + cc;
    if (col >= D) continue;
    const float* acc_l = ACC + (size_t)l * AF;
    pU[((int64_t)l * r + j) * D + col] = acc_l[j * kNB + cc];
    pV[((int64_t)l * D + col) * r + j] = acc_l[(r16(a) + j) * kNB + cc];
  }
  for (int e = tid; e < L * kNB; e += blockDim.x) {
    const int l = e / kNB, cc = e % kNB, col = c0 + cc;
    if (col < D) pc[(int64_t)l * D + col] = ACC[(size_t)l * AF + 2 * r16(a) * kNB + cc];
  }
}

// ---- launchers (return 0, or 1 on arguments outside the cover) --------------------------------------------------------
inline void prep(const tzk_dcn_v2_args& a, int mask, cudaStream_t stream) {
  const int64_t n = (int64_t)2 * a.L * r8(a) * d8(a);
  const int64_t blocks = (n + 255) / 256;
  TZK_LAUNCH((prep_kernel), (unsigned)(blocks < 1024 ? blocks : 1024), 256, 0, stream, a, mask);
}

template <class K>
inline void launch_tiles(K kernel, const tzk_dcn_v2_args& a, int pass, int grid, cudaStream_t stream) {
  const size_t smem = smem_bytes(a, pass);
  tzk_batch_sum::opt_in_smem(kernel, smem);
  TZK_LAUNCH((kernel), grid, 32 * tile_warps(a, pass), smem, stream, a);
}
template <class K>
inline void launch_weight(K kernel, const tzk_dcn_v2_args& a, int chunks, float* partials, cudaStream_t stream) {
  const size_t smem = smem_bytes(a, 2);
  tzk_batch_sum::opt_in_smem(kernel, smem);
  TZK_LAUNCH((kernel), dim3((unsigned)((a.D + kNB - 1) / kNB), (unsigned)chunks), kWarpsW * 32, smem, stream, a,
             partials);
}
// the kernels are instantiated per rank tile count r8 / 8, so their fragment arrays fit the rank
#define TZK_DCN_V2_RANK_SWITCH(a, fn, kernel, ...)                   \
  switch (r8(a) / 8) {                                                \
    case 1: fn(kernel<1>, __VA_ARGS__); break;                        \
    case 2: fn(kernel<2>, __VA_ARGS__); break;                        \
    case 3: fn(kernel<3>, __VA_ARGS__); break;                        \
    case 4: fn(kernel<4>, __VA_ARGS__); break;                        \
    case 5: fn(kernel<5>, __VA_ARGS__); break;                        \
    case 6: fn(kernel<6>, __VA_ARGS__); break;                        \
    case 7: fn(kernel<7>, __VA_ARGS__); break;                        \
    default: fn(kernel<8>, __VA_ARGS__); break;                       \
  }

inline int fwd(const tzk_dcn_v2_args& a, int grid, cudaStream_t stream) {
  if (check(a, 0) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  prep(a, 1 << kUb | 1 << kVb, stream);
  TZK_DCN_V2_RANK_SWITCH(a, launch_tiles, fwd_kernel, a, 0, grid, stream);
  return 0;
}

inline int bwd_data(const tzk_dcn_v2_args& a, int grid, cudaStream_t stream) {
  if (check(a, 1) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  prep(a, 1 << kVb | 1 << kVt | 1 << kUt, stream);
  TZK_DCN_V2_RANK_SWITCH(a, launch_tiles, bwd_data_kernel, a, 1, grid, stream);
  return 0;
}

// partials: chunks * param_floats(a) floats; dparams: param_floats(a) floats
inline int bwd_weight(const tzk_dcn_v2_args& a, int chunks, float* partials, float* dparams, cudaStream_t stream) {
  if (check(a, 2) != 0 || chunks < 1 || !partials || !dparams) return 1;
  if (a.B > 0) {
    prep(a, 1 << kVb | 1 << kUt, stream);
    TZK_DCN_V2_RANK_SWITCH(a, launch_weight, bwd_weight_kernel, a, chunks, partials, stream);
  }
  tzk_batch_sum::reduce(partials, a.B > 0 ? chunks : 0, param_floats(a), 1, dparams, stream);
  return 0;
}
}  // namespace tzk_dcn_v2
