// tzk_tower_bwd2.cuh — backward of the narrow tower layers (K, N <= 64) without shared-memory tiles and without
// barriers in the row loop (second implementation behind tzk_small_linear_bwd; TZK_SMALL_LINEAR_BWD=1 selects the
// tile kernel of tzk_tower.cu again).
//
//   small_linear_dx_rows_kernel   dx = (dy * [y > 0]) @ W         one thread per row, W broadcast from shared memory,
//                                                                 32 accumulators per pass, 16-B row stores
//   small_linear_dw_tiles_kernel  dW = dz^T @ x, db = colsum(dz)  32-row tiles through two shared-memory stages, the next
//                                                                 tile's global loads in flight under the arithmetic
//                                                                 of the current one (default)
//   small_linear_dw_kernel        the same, TZK_SMALL_LINEAR_DW=0:  a thread owns an NB x KB block of dW, loops over its
//                                                                 CTA's rows with U rows of independent 16-B loads in
//                                                                 flight; lanes of a warp share a dz row (broadcast)
//                                                                 and cover one x row (coalesced); row groups of a
//                                                                 CTA are folded in shared memory in a fixed order,
//                                                                 CTAs by a fixed-order reduction kernel.
// Plain CUDA (no PTX): the includer provides TZK_DYN_SMEM(type, name) and TZK_LAUNCH((kernel), grid, block, smem,
// stream, args...) — nvcc in libtzk.so, g++ + tests/native/cuda_cpu_shim.h in tests/test_tower_bwd2_cpu.py,
// which runs this very source on the host against float64.
#pragma once
#include <stdint.h>
#include <stdlib.h>

namespace tzk_bwd2 {
constexpr int kThreads = 128;
constexpr int kSms = 132;   // H100 SXM

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- dx -------------------------------------------------------------------------------------------------------
template <int KP>
__global__ void __launch_bounds__(kThreads, 5)
small_linear_dx_rows_kernel(const float* __restrict__ w, const float* __restrict__ y, int64_t ld_y,
                            const float* __restrict__ dy, int64_t ld_dy, int64_t M, int K, int N, int relu,
                            float* __restrict__ dx, int64_t ld_dx) {
  constexpr int KH = KP < 32 ? KP : 32;     // outputs per pass
  TZK_DYN_SMEM(float, sm);
  float* Ws = sm;                           // [N][KP]: row n of W, zero beyond K
  const int tid = threadIdx.x;
  for (int i = tid; i < N * KP; i += kThreads) {
    const int n = i / KP, k = i - n * KP;
    Ws[i] = k < K ? __ldg(w + (int64_t)n * K + k) : 0.f;
  }
  __syncthreads();
  const bool vec_in = (N & 3) == 0 && (ld_dy & 3) == 0 && aligned16(dy) && (!relu || ((ld_y & 3) == 0 && aligned16(y)));
  const bool vec_out = (K & 3) == 0 && (ld_dx & 3) == 0 && aligned16(dx);
  for (int64_t row = (int64_t)blockIdx.x * kThreads + tid; row < M; row += (int64_t)gridDim.x * kThreads) {
    const float* dr = dy + row * ld_dy;
    const float* yr = relu ? y + row * ld_y : nullptr;
    float* xr = dx + row * ld_dx;
#pragma unroll 1
    for (int k0 = 0; k0 < KP; k0 += KH) {   // the second pass re-reads the row from L1
      if (k0 >= K) break;
      float acc[KH];
#pragma unroll
      for (int k = 0; k < KH; ++k) acc[k] = 0.f;
      if (vec_in) {
        for (int n0 = 0; n0 < N; n0 += 4) {
          float4 d = *reinterpret_cast<const float4*>(dr + n0);
          if (yr) {
            const float4 m = *reinterpret_cast<const float4*>(yr + n0);
            d.x = m.x > 0.f ? d.x : 0.f; d.y = m.y > 0.f ? d.y : 0.f;
            d.z = m.z > 0.f ? d.z : 0.f; d.w = m.w > 0.f ? d.w : 0.f;
          }
          const float dv[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
          for (int nn = 0; nn < 4; ++nn) {
            const float4* wr = reinterpret_cast<const float4*>(Ws + (n0 + nn) * KP + k0);
#pragma unroll
            for (int k4 = 0; k4 < KH / 4; ++k4) {
              const float4 w4 = wr[k4];
              acc[k4 * 4 + 0] = fmaf(dv[nn], w4.x, acc[k4 * 4 + 0]);
              acc[k4 * 4 + 1] = fmaf(dv[nn], w4.y, acc[k4 * 4 + 1]);
              acc[k4 * 4 + 2] = fmaf(dv[nn], w4.z, acc[k4 * 4 + 2]);
              acc[k4 * 4 + 3] = fmaf(dv[nn], w4.w, acc[k4 * 4 + 3]);
            }
          }
        }
      } else {
#pragma unroll 4
        for (int n = 0; n < N; ++n) {
          float dv = dr[n];
          if (yr && !(yr[n] > 0.f)) dv = 0.f;
          const float4* wr = reinterpret_cast<const float4*>(Ws + n * KP + k0);
#pragma unroll
          for (int k4 = 0; k4 < KH / 4; ++k4) {
            const float4 w4 = wr[k4];
            acc[k4 * 4 + 0] = fmaf(dv, w4.x, acc[k4 * 4 + 0]);
            acc[k4 * 4 + 1] = fmaf(dv, w4.y, acc[k4 * 4 + 1]);
            acc[k4 * 4 + 2] = fmaf(dv, w4.z, acc[k4 * 4 + 2]);
            acc[k4 * 4 + 3] = fmaf(dv, w4.w, acc[k4 * 4 + 3]);
          }
        }
      }
      if (vec_out) {
#pragma unroll
        for (int k4 = 0; k4 < KH / 4; ++k4)
          if (k0 + k4 * 4 < K)
            *reinterpret_cast<float4*>(xr + k0 + k4 * 4) =
                make_float4(acc[k4 * 4], acc[k4 * 4 + 1], acc[k4 * 4 + 2], acc[k4 * 4 + 3]);
      } else {
#pragma unroll
        for (int k = 0; k < KH; ++k)
          if (k0 + k < K) xr[k0 + k] = acc[k];
      }
    }
  }
}

// ---- dW, db ---------------------------------------------------------------------------------------------------
// Threads of a row group: t = tn * TK + tk owns dW[n0 .. n0+NB) x [k0 .. k0+KB), n0 = tn * NB, k0 = tk * KB; lanes run
// over tk first, so one warp-wide load of x covers whole rows and the dz loads are broadcasts.  A CTA owns
// `rows_per_cta` consecutive rows; row group g takes rows g, g + RG, ... of them.
template <int NB, int KB, int U>
__global__ void __launch_bounds__(kThreads)
small_linear_dw_kernel(const float* __restrict__ x, int64_t ld_x, const float* __restrict__ y, int64_t ld_y,
                       const float* __restrict__ dy, int64_t ld_dy, int64_t M, int K, int N, int relu,
                       int rows_per_cta, float* __restrict__ partial) {
  TZK_DYN_SMEM(float, red);                      // [RG][N * K + N]
  const int TN = (N + NB - 1) / NB, TK = (K + KB - 1) / KB, T = TN * TK;
  const int RG = kThreads / T;
  const int tid = threadIdx.x, g = tid / T, t = tid - g * T;
  const int tn = t / TK, tk = t - tn * TK;
  const int n0 = tn * NB, k0 = tk * KB;
  const bool va = NB == 4 && (N & 3) == 0 && (ld_dy & 3) == 0 && aligned16(dy) &&
                  (!relu || ((ld_y & 3) == 0 && aligned16(y)));
  const bool vb = (KB & 3) == 0 && (K & 3) == 0 && (ld_x & 3) == 0 && aligned16(x);
  float acc[NB][KB], accB[NB];
#pragma unroll
  for (int i = 0; i < NB; ++i) {
    accB[i] = 0.f;
#pragma unroll
    for (int j = 0; j < KB; ++j) acc[i][j] = 0.f;
  }
  const int64_t row_begin = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t row_end = row_begin + rows_per_cta < M ? row_begin + rows_per_cta : M;
  if (g < RG) {
    for (int64_t r0 = row_begin + g; r0 < row_end; r0 += (int64_t)RG * U) {
      float a[U][NB], b[U][KB];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t r = r0 + (int64_t)u * RG;
        const bool ok = r < row_end;
        if (va) {
          float4 d = make_float4(0.f, 0.f, 0.f, 0.f);
          if (ok) {
            d = *reinterpret_cast<const float4*>(dy + r * ld_dy + n0);
            if (relu) {
              const float4 m = *reinterpret_cast<const float4*>(y + r * ld_y + n0);
              d.x = m.x > 0.f ? d.x : 0.f; d.y = m.y > 0.f ? d.y : 0.f;
              d.z = m.z > 0.f ? d.z : 0.f; d.w = m.w > 0.f ? d.w : 0.f;
            }
          }
          a[u][0] = d.x;
          if (NB > 1) { a[u][1 % NB] = d.y; a[u][2 % NB] = d.z; a[u][3 % NB] = d.w; }
        } else {
#pragma unroll
          for (int i = 0; i < NB; ++i) {
            float v = 0.f;
            if (ok && n0 + i < N) {
              v = __ldg(dy + r * ld_dy + n0 + i);
              if (relu && !(__ldg(y + r * ld_y + n0 + i) > 0.f)) v = 0.f;
            }
            a[u][i] = v;
          }
        }
        if (vb) {
#pragma unroll
          for (int j4 = 0; j4 < KB / 4; ++j4) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok && k0 + j4 * 4 < K) v = *reinterpret_cast<const float4*>(x + r * ld_x + k0 + j4 * 4);
            b[u][j4 * 4 + 0] = v.x; b[u][j4 * 4 + 1] = v.y; b[u][j4 * 4 + 2] = v.z; b[u][j4 * 4 + 3] = v.w;
          }
        } else {
#pragma unroll
          for (int j = 0; j < KB; ++j) b[u][j] = (ok && k0 + j < K) ? __ldg(x + r * ld_x + k0 + j) : 0.f;
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
#pragma unroll
        for (int i = 0; i < NB; ++i) {
          accB[i] += a[u][i];
#pragma unroll
          for (int j = 0; j < KB; ++j) acc[i][j] = fmaf(a[u][i], b[u][j], acc[i][j]);
        }
      }
    }
  }
  // fold the row groups in order g = 0, 1, ...: every (n, k) is owned by exactly one thread of each group
  const int total = N * K + N;
  if (g < RG) {
    float* mine = red + g * total;
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      if (n0 + i >= N) continue;
#pragma unroll
      for (int j = 0; j < KB; ++j)
        if (k0 + j < K) mine[(n0 + i) * K + k0 + j] = acc[i][j];
      if (tk == 0) mine[N * K + n0 + i] = accB[i];
    }
  }
  __syncthreads();
  float* p = partial + (int64_t)blockIdx.x * total;
  for (int i = tid; i < total; i += kThreads) {
    float s = red[i];
    for (int q = 1; q < RG; ++q) s += red[q * total + i];
    p[i] = s;
  }
}

// ---- dW, db: row tiles through shared memory, global loads of tile i+1 in flight under the arithmetic of tile i --------
// A CTA owns `rows_per_cta` consecutive rows and walks them in tiles of kDwRows rows.  Every thread fetches its share
// of the NEXT tile (x rows and dz = dy * [y > 0] rows, 16-B chunks, zero beyond K / N / the CTA's last row) into
// registers, then does the arithmetic of the current tile out of shared memory, then parks the registers in the other
// shared-memory stage: one barrier per tile, and the whole tile's global requests are in flight together instead of
// U rows per thread.  Inside a tile, thread t = tn * KC + tk of row group g owns the 4 x 4 block
// dW[4 tn .. 4 tn + 4) x [4 tk .. 4 tk + 4) and takes rows g, g + RG, ... of the tile (two 16-B shared-memory loads per
// 16 FFMA; the dz chunk is a broadcast, the x chunks of neighbouring lanes are contiguous).  Row groups are folded in
// shared memory in the order g = 0, 1, ..., CTAs by small_linear_reduce2_kernel in CTA order: deterministic.
constexpr int kDwThreads = 256;
constexpr int kDwRows = 32;

template <int KP, int NP>
__global__ void __launch_bounds__(kDwThreads)
small_linear_dw_tiles_kernel(const float* __restrict__ x, int64_t ld_x, const float* __restrict__ y, int64_t ld_y,
                             const float* __restrict__ dy, int64_t ld_dy, int64_t M, int K, int N, int relu,
                             int rows_per_cta, float* __restrict__ partial) {
  constexpr int R = kDwRows;
  constexpr int KC = KP / 4, NC = NP / 4;                           // 16-B chunks per padded row
  constexpr int XQ = (R * KC + kDwThreads - 1) / kDwThreads;        // chunks of the x tile per thread
  constexpr int DQ = (R * NC + kDwThreads - 1) / kDwThreads;        // chunks of the dz tile per thread
  constexpr int T = KC * NC;                                        // threads per row group (<= 256)
  constexpr int RG = kDwThreads / T;                                // row groups
  constexpr int STAGE = R * (KP + NP);                              // floats per stage: x tile, then dz tile
  TZK_DYN_SMEM(float, sm);
  const int tid = threadIdx.x, g = tid / T, t = tid - g * T;
  const int tn = t / KC, tk = t - tn * KC;
  const bool vx = (K & 3) == 0 && (ld_x & 3) == 0 && aligned16(x);
  const bool vd = (N & 3) == 0 && (ld_dy & 3) == 0 && aligned16(dy) && (!relu || ((ld_y & 3) == 0 && aligned16(y)));
  const int64_t row_begin = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t row_end = row_begin + rows_per_cta < M ? row_begin + rows_per_cta : M;
  const int n_tiles = row_begin < row_end ? (int)((row_end - row_begin + R - 1) / R) : 0;

  float4 xr[XQ], dr[DQ];
  auto fetch = [&](int tile) {
    const int64_t r0 = row_begin + (int64_t)tile * R;
#pragma unroll
    for (int q = 0; q < XQ; ++q) {
      const int idx = tid + q * kDwThreads;
      const int r = idx / KC, c = (idx - r * KC) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < R * KC && r0 + r < row_end && c < K) {
        const float* p = x + (r0 + r) * ld_x + c;
        if (vx) {
          v = *reinterpret_cast<const float4*>(p);
        } else {
          v.x = __ldg(p);
          if (c + 1 < K) v.y = __ldg(p + 1);
          if (c + 2 < K) v.z = __ldg(p + 2);
          if (c + 3 < K) v.w = __ldg(p + 3);
        }
      }
      xr[q] = v;
    }
#pragma unroll
    for (int q = 0; q < DQ; ++q) {
      const int idx = tid + q * kDwThreads;
      const int r = idx / NC, c = (idx - r * NC) * 4;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (idx < R * NC && r0 + r < row_end && c < N) {
        const float* p = dy + (r0 + r) * ld_dy + c;
        const float* m = relu ? y + (r0 + r) * ld_y + c : nullptr;
        if (vd) {
          v = *reinterpret_cast<const float4*>(p);
          if (m) {
            const float4 mv = *reinterpret_cast<const float4*>(m);
            v.x = mv.x > 0.f ? v.x : 0.f; v.y = mv.y > 0.f ? v.y : 0.f;
            v.z = mv.z > 0.f ? v.z : 0.f; v.w = mv.w > 0.f ? v.w : 0.f;
          }
        } else {
          v.x = (!m || __ldg(m) > 0.f) ? __ldg(p) : 0.f;
          if (c + 1 < N) v.y = (!m || __ldg(m + 1) > 0.f) ? __ldg(p + 1) : 0.f;
          if (c + 2 < N) v.z = (!m || __ldg(m + 2) > 0.f) ? __ldg(p + 2) : 0.f;
          if (c + 3 < N) v.w = (!m || __ldg(m + 3) > 0.f) ? __ldg(p + 3) : 0.f;
        }
      }
      dr[q] = v;
    }
  };
  auto park = [&](float* stage) {
    float4* xs = reinterpret_cast<float4*>(stage);
    float4* ds = reinterpret_cast<float4*>(stage + R * KP);
#pragma unroll
    for (int q = 0; q < XQ; ++q)
      if (tid + q * kDwThreads < R * KC) xs[tid + q * kDwThreads] = xr[q];
#pragma unroll
    for (int q = 0; q < DQ; ++q)
      if (tid + q * kDwThreads < R * NC) ds[tid + q * kDwThreads] = dr[q];
  };

  float acc[4][4], accB[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    accB[i] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  }
  if (n_tiles > 0) {
    fetch(0);
    park(sm);
  }
  __syncthreads();
  for (int i = 0; i < n_tiles; ++i) {
    const float* stage = sm + (i & 1) * STAGE;
    if (i + 1 < n_tiles) fetch(i + 1);
    if (g < RG) {
      const float4* xs = reinterpret_cast<const float4*>(stage) + tk;
      const float4* ds = reinterpret_cast<const float4*>(stage + R * KP) + tn;
#pragma unroll 4
      for (int r = g; r < R; r += RG) {       // rows beyond the CTA's last one are zeros in shared memory
        const float4 a4 = ds[r * NC], b4 = xs[r * KC];
        const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
        for (int ii = 0; ii < 4; ++ii) {
          accB[ii] += a[ii];
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[ii][j] = fmaf(a[ii], b[j], acc[ii][j]);
        }
      }
    }
    if (i + 1 < n_tiles) park(sm + ((i + 1) & 1) * STAGE);
    __syncthreads();
  }
  // fold the row groups in the order g = 0, 1, ... (the stages are free: every thread is past the last barrier)
  const int total = N * K + N;
  if (g < RG) {
    float* mine = sm + g * total;
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const int n = tn * 4 + ii;
      if (n >= N) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (tk * 4 + j < K) mine[n * K + tk * 4 + j] = acc[ii][j];
      if (tk == 0) mine[N * K + n] = accB[ii];
    }
  }
  __syncthreads();
  float* p = partial + (int64_t)blockIdx.x * total;
  for (int i = tid; i < total; i += kDwThreads) {
    float s = sm[i];
    for (int q = 1; q < RG; ++q) s += sm[q * total + i];
    p[i] = s;
  }
}

// shared memory of the tile kernel: two stages, or the fold area if that is larger (tiny layers: many row groups)
inline size_t dw_tiles_smem(int KP, int NP, int K, int N) {
  const size_t stages = (size_t)2 * kDwRows * (KP + NP);
  const size_t fold = (size_t)(kDwThreads / ((KP / 4) * (NP / 4))) * ((size_t)N * K + N);
  return (stages > fold ? stages : fold) * sizeof(float);
}

// out[i] = sum over CTAs (ascending) of partial[c][i]; 8 interleaved partial sums per output folded in a fixed order
__global__ void __launch_bounds__(256)
small_linear_reduce2_kernel(const float* __restrict__ partial, int n_parts, int NK, int N, float* __restrict__ dw,
                            float* __restrict__ db) {
  __shared__ float red[8][32];
  const int o = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + o;
  const int total = NK + N;
  float s = 0.f;
  if (i < total)
    for (int c = g; c < n_parts; c += 8) s += partial[(int64_t)c * total + i];
  red[g][o] = s;
  __syncthreads();
  if (g == 0 && i < total) {
    float r = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) r += red[k][o];
    if (i < NK) dw[i] = r;
    else if (db) db[i - NK] = r;
  }
}

struct Shape { int nb, kb, t; };
// block shape of the row-group kernel (TZK_SMALL_LINEAR_DW=0): 16-B loads on both sides when the sizes allow it, at most
// 128 threads per row group
inline Shape pick(int K, int N) {
  const int nb = (N % 4 == 0) ? 4 : 1;
  int kb = 4;
  int t = ((N + nb - 1) / nb) * ((K + kb - 1) / kb);
  if (t > kThreads) { kb = 8; t = ((N + nb - 1) / nb) * ((K + kb - 1) / kb); }
  return {nb, kb, t};
}
inline int dw_grid(int64_t M) {
  const int64_t want = (M + 31) / 32;   // at least 32 rows per CTA
  return (int)(want < kSms * 4 ? (want < 1 ? 1 : want) : kSms * 4);
}

inline size_t workspace_bytes(int64_t M, int K, int N) { return (size_t)dw_grid(M) * ((size_t)N * K + N) * sizeof(float); }

// Switches of code paths that have not been through a GPU validation pass yet: `name`=0/1 decides; unset, TZK_EXPERIMENTAL=1
// turns them all on (scripts/gpu_call_n1.sh); otherwise they stay off.  A validated path gets its default flipped here.
inline bool unvalidated_switch(const char* name) {
  const char* e = getenv(name);
  if (e && (e[0] == '0' || e[0] == '1')) return e[0] == '1';
  const char* x = getenv("TZK_EXPERIMENTAL");
  return x && x[0] == '1';
}

// The dW tile kernel (default); TZK_SMALL_LINEAR_DW=0: the
// row-group dW kernel (straight from global memory, U rows in flight per thread).  Read per call.
inline bool use_dw_tiles() {
  const char* e = getenv("TZK_SMALL_LINEAR_DW");
  return !(e && e[0] == '0');
}

// the tile kernel pads K and N to its compiled sizes, so every K, N <= 64 is covered; the row-group kernel needs its
// mapping to fit 128 threads (otherwise the caller keeps the tile kernel of tzk_tower.cu)
inline bool supported(int K, int N) {
  return K >= 1 && N >= 1 && K <= 64 && N <= 64 && (use_dw_tiles() || pick(K, N).t <= kThreads);
}

// dz = dy * (relu ? y > 0 : 1); dx = dz @ W (skipped when dx is NULL); dW = dz^T @ x; db = colsum(dz) (db nullable).
// Returns 0, or 1 bad argument / 2 workspace too small / 3 launch failure.
inline int run(const float* x, int64_t ld_x, const float* w, const float* y, int64_t ld_y, const float* dy,
               int64_t ld_dy, int64_t M, int32_t K, int32_t N, int32_t relu, float* dx, int64_t ld_dx, float* dw,
               float* db, void* workspace, size_t workspace_bytes_, cudaStream_t st) {

  if (M < 1 || K < 1 || N < 1 || K > 64 || N > 64 || !x || !w || !dy || !dw || (relu && !y)) return 1;
  if (workspace_bytes_ < workspace_bytes(M, K, N)) return 2;
  const Shape s = pick(K, N);
  const bool tiles = use_dw_tiles() || s.t > kThreads;   // (the row-group kernel does not cover e.g. 64 x 30)
  if (dx) {
    const int KP = K <= 16 ? 16 : (K <= 32 ? 32 : 64);
    const size_t smem = (size_t)N * KP * sizeof(float);
    const int64_t ctas = (M + kThreads - 1) / kThreads;
    const int grid = (int)(ctas < kSms * 10 ? ctas : kSms * 10);
    if (KP == 16) TZK_LAUNCH((small_linear_dx_rows_kernel<16>), grid, kThreads, smem, st, w, y, ld_y, dy, ld_dy, M, K, N, relu, dx, ld_dx);
    else if (KP == 32) TZK_LAUNCH((small_linear_dx_rows_kernel<32>), grid, kThreads, smem, st, w, y, ld_y, dy, ld_dy, M, K, N, relu, dx, ld_dx);
    else TZK_LAUNCH((small_linear_dx_rows_kernel<64>), grid, kThreads, smem, st, w, y, ld_y, dy, ld_dy, M, K, N, relu, dx, ld_dx);
    if (cudaGetLastError() != cudaSuccess) return 3;
  }
  const int grid = dw_grid(M);
  const int rows_per_cta = (int)((M + grid - 1) / grid);
  float* partial = static_cast<float*>(workspace);
  if (tiles) {
    const int KP = K <= 16 ? 16 : (K <= 32 ? 32 : 64);
    const int NP = N <= 4 ? 4 : (N <= 16 ? 16 : (N <= 32 ? 32 : 64));
    const size_t smem = dw_tiles_smem(KP, NP, K, N);      // <= 32 KB
#define TZK_DWT(KP_, NP_)                                                                                              \
  TZK_LAUNCH((small_linear_dw_tiles_kernel<KP_, NP_>), grid, kDwThreads, smem, st, x, ld_x, y, ld_y, dy, ld_dy, M, K, N, \
             relu, rows_per_cta, partial)
#define TZK_DWT_N(KP_)                                                                                                 \
  do {                                                                                                                 \
    if (NP == 4) TZK_DWT(KP_, 4);                                                                                      \
    else if (NP == 16) TZK_DWT(KP_, 16);                                                                               \
    else if (NP == 32) TZK_DWT(KP_, 32);                                                                               \
    else TZK_DWT(KP_, 64);                                                                                             \
  } while (0)
    if (KP == 16) TZK_DWT_N(16);
    else if (KP == 32) TZK_DWT_N(32);
    else TZK_DWT_N(64);
#undef TZK_DWT_N
#undef TZK_DWT
  } else {
    const int RG = kThreads / s.t;
    const size_t smem = (size_t)RG * ((size_t)N * K + N) * sizeof(float);
#define TZK_DW(NB, KB, U)                                                                                            \
  TZK_LAUNCH((small_linear_dw_kernel<NB, KB, U>), grid, kThreads, smem, st, x, ld_x, y, ld_y, dy, ld_dy, M, K, N, relu, \
             rows_per_cta, partial)
    if (s.nb == 4 && s.kb == 4) TZK_DW(4, 4, 8);
    else if (s.nb == 4) TZK_DW(4, 8, 4);
    else if (s.kb == 4) TZK_DW(1, 4, 8);
    else TZK_DW(1, 8, 8);
#undef TZK_DW
  }
  if (cudaGetLastError() != cudaSuccess) return 3;
  const int total = N * K + N;
  TZK_LAUNCH((small_linear_reduce2_kernel), (total + 31) / 32, 256, 0, st, partial, grid, N * K, N, dw, db);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
}  // namespace tzk_bwd2
