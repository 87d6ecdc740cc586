// tzk_tower_tail.cuh — the tail of a rank tower in ONE pass over the batch, forward AND backward:
//
//     h = relu(y1 @ W1^T + b1)        last Perceptron of the final MLP      (tzrec/modules/mlp.py:20-84; K, N <= 64)
//     z = h @ w2^T + b2               output Linear(N, 1)                   (tzrec/models/rank_model.py:133-179)
//     loss = mean BCE-with-logits(z, label)                                (tzrec/models/rank_model.py:181-262)
//
// and, in the same kernel, d loss / d {y1, W1, b1, w2, b2}.  On DLRM-Criteo (64 -> 32 -> 1, B = 65536) the unfused
// chain is 18 launches of latency-bound kernels around 24 MB of data; here every row is read once.
//
// A CTA walks tiles of 128 rows, thread r <-> row r of the tile:
//   phase 1 (a row per thread, W1 broadcast from shared memory): h, z, the row's loss term, dz = (sigmoid(z) - y) / M,
//           dh = dz * w2 * [h > 0], dy1 = dh @ W1 (stored to global); the row of y1, dh, dz * h and dz go to shared memory;
//   phase 2 (the tile as a small GEMM, like small_linear_dw_tiles_kernel): thread (tn, tk) adds dh^T y1 over the tile's
//           rows into its 4 x 4 block(s) of dW1; threads 0..N-1 add the columns of dh (db1) and dz * h (dw2); thread 0
//           adds dz (db2) and the loss terms — all in row order.
// The per-CTA sums leave as one vector [N K | N | N | 1 | 1] = dW1, db1, dw2, db2, loss; tower_tail_reduce_kernel folds
// the CTAs in CTA order: deterministic.
//
// Masked mode (kMask; y1 the output of a ReLU layer): the kernel stores dZ = dy1 * [y1 > 0], the gradient of that
// layer's pre-activation, in place of dy1, and per 128-row tile the K column sums of dZ, in act_bwd_colsum_kernel's
// order at 64 columns (tzk_dense.cu): its 128-row slabs are these tiles, so colsum_final_kernel folds them into the
// layer's bias gradient with act_bwd_colsum's bits.  The separate ReLU-backward pass over [M, K] is not needed.
//
// Plain CUDA (no PTX): the includer provides TZK_DYN_SMEM / TZK_LAUNCH (nvcc: tzk_tower.cu; g++ +
// tests/native/cuda_cpu_shim.h: tests/test_tower_tail_cpu.py runs this source on the host against float64).
#pragma once
#include <stdint.h>

namespace tzk_tail {
constexpr int kRows = 128;       // rows per tile = threads per CTA
constexpr int kMaxCtas = 132 * 4;   // 4 CTAs per H100 SM

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

inline int out_len(int K, int N) { return N * K + 2 * N + 2; }
inline int grid_for(int64_t M) {
  const int64_t t = (M + kRows - 1) / kRows;
  return (int)(t < 1 ? 1 : (t < kMaxCtas ? t : kMaxCtas));
}
inline int64_t tiles(int64_t M) { return (M + kRows - 1) / kRows; }
// workspace: the per-CTA sums [grid][out_len], then (masked mode) the per-tile column sums of dZ [tiles][K]
inline size_t colsum_offset(int64_t M, int K, int N) { return (size_t)grid_for(M) * out_len(K, N); }
inline size_t workspace_bytes(int64_t M, int K, int N) {
  return (colsum_offset(M, K, N) + (size_t)tiles(M) * K) * sizeof(float);
}
// shared memory: W1 [NP][KP] | b1 [NP] | w2 [NP] | y1 tile [R][KP + 4] | dh tile [R][NP] | dz*h tile [R][NP] | dz [R] | l [R]
// | masked mode: dZ tile [R][KP + 4]
inline size_t smem_bytes(int KP, int NP, bool mask) {
  return ((size_t)NP * KP + 2 * NP + (size_t)(mask ? 2 : 1) * kRows * (KP + 4) + 2 * (size_t)kRows * NP + 2 * kRows) *
         sizeof(float);
}

template <int KP, int NP, bool kMask>
__global__ void __launch_bounds__(kRows)
tower_tail_bce_kernel(const float* __restrict__ y1, int64_t ld_y, const float* __restrict__ w1,
                      const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                      const float* __restrict__ labels, int64_t M, int K, int N, float inv_m, int rows_per_cta,
                      float* __restrict__ logits, float* __restrict__ dy1, int64_t ld_dy, float* __restrict__ partial,
                      float* __restrict__ zsum) {
  constexpr int R = kRows, KC = KP / 4, NC = NP / 4, XS = KP + 4;
  constexpr int NB = (KC * NC + R - 1) / R;          // 4 x 4 blocks of dW1 per thread
  TZK_DYN_SMEM(float, sm);
  float* Ws = sm;                        // [NP][KP], zero beyond N / K
  float* b1s = Ws + NP * KP;             // [NP]
  float* w2s = b1s + NP;                 // [NP]
  float* Xs = w2s + NP;                  // [R][XS]
  float* Dh = Xs + R * XS;               // [R][NP]
  float* Hg = Dh + R * NP;               // [R][NP]
  float* Dz = Hg + R * NP;               // [R]
  float* Ls = Dz + R;                    // [R]
  float* Zs = Ls + R;                    // [R][XS], masked mode
  const int tid = threadIdx.x;
  for (int i = tid; i < NP * KP; i += R) {
    const int n = i / KP, k = i - n * KP;
    Ws[i] = (n < N && k < K) ? __ldg(w1 + (int64_t)n * K + k) : 0.f;
  }
  for (int n = tid; n < NP; n += R) {
    b1s[n] = (n < N && b1) ? __ldg(b1 + n) : 0.f;
    w2s[n] = n < N ? __ldg(w2 + n) : 0.f;
  }
  const float b2v = b2 ? __ldg(b2) : 0.f;
  const bool vin = (K & 3) == 0 && (ld_y & 3) == 0 && aligned16(y1);
  const bool vout = (K & 3) == 0 && (ld_dy & 3) == 0 && aligned16(dy1);
  float acc[NB][4][4], accv = 0.f, accw = 0.f, accz = 0.f, accl = 0.f;   // dW1 blocks; db1[tid]; dw2[tid]; db2; loss
#pragma unroll
  for (int q = 0; q < NB; ++q)
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[q][i][j] = 0.f;
  const int64_t row_begin = (int64_t)blockIdx.x * rows_per_cta;
  const int64_t row_end = row_begin + rows_per_cta < M ? row_begin + rows_per_cta : M;
  __syncthreads();
  for (int64_t t0 = row_begin; t0 < row_end; t0 += R) {
    const int64_t row = t0 + tid;
    const bool live = row < row_end;
    // ---- phase 1: this thread's row ------------------------------------------------------------------------------
    float* xr = Xs + tid * XS;
#pragma unroll
    for (int c = 0; c < KC; ++c) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (live && 4 * c < K) {
        const float* p = y1 + row * ld_y + 4 * c;
        if (vin) {
          v = *reinterpret_cast<const float4*>(p);
        } else {
          v.x = __ldg(p);
          if (4 * c + 1 < K) v.y = __ldg(p + 1);
          if (4 * c + 2 < K) v.z = __ldg(p + 2);
          if (4 * c + 3 < K) v.w = __ldg(p + 3);
        }
      }
      *reinterpret_cast<float4*>(xr + 4 * c) = v;
    }
    float h[NP];
#pragma unroll
    for (int n = 0; n < NP; ++n) h[n] = b1s[n];
#pragma unroll 2
    for (int c = 0; c < KC; ++c) {
      const float4 x4 = *reinterpret_cast<const float4*>(xr + 4 * c);
#pragma unroll
      for (int n = 0; n < NP; ++n) {
        const float4 w4 = *reinterpret_cast<const float4*>(Ws + n * KP + 4 * c);
        h[n] = fmaf(x4.x, w4.x, h[n]);
        h[n] = fmaf(x4.y, w4.y, h[n]);
        h[n] = fmaf(x4.z, w4.z, h[n]);
        h[n] = fmaf(x4.w, w4.w, h[n]);
      }
    }
    float z = b2v;
#pragma unroll
    for (int n = 0; n < NP; ++n) {
      h[n] = h[n] > 0.f ? h[n] : 0.f;
      z = fmaf(h[n], w2s[n], z);
    }
    float dz = 0.f, lt = 0.f;
    if (live) {
      const float y = __ldg(labels + row);
      const float e = expf(-fabsf(z));
      lt = fmaxf(z, 0.f) - z * y + log1pf(e);
      const float sig = z >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
      dz = (sig - y) * inv_m;
      logits[row] = z;
    }
    Dz[tid] = dz;
    Ls[tid] = lt;
#pragma unroll
    for (int n = 0; n < NP; ++n) {
      Hg[tid * NP + n] = dz * h[n];
      h[n] = h[n] > 0.f ? dz * w2s[n] : 0.f;      // h now holds dh
      Dh[tid * NP + n] = h[n];
    }
#pragma unroll 2
    for (int c = 0; c < KC; ++c) {
      float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int n = 0; n < NP; ++n) {
        const float4 w4 = *reinterpret_cast<const float4*>(Ws + n * KP + 4 * c);
        a.x = fmaf(h[n], w4.x, a.x);
        a.y = fmaf(h[n], w4.y, a.y);
        a.z = fmaf(h[n], w4.z, a.z);
        a.w = fmaf(h[n], w4.w, a.w);
      }
      if constexpr (kMask) {                      // act_bwd_colsum's predicate: !(y1 > 0), NaN included, gives +0
        const float4 y4 = *reinterpret_cast<const float4*>(xr + 4 * c);
        a.x = y4.x > 0.f ? a.x : 0.f;
        a.y = y4.y > 0.f ? a.y : 0.f;
        a.z = y4.z > 0.f ? a.z : 0.f;
        a.w = y4.w > 0.f ? a.w : 0.f;
        *reinterpret_cast<float4*>(Zs + tid * XS + 4 * c) = a;     // dead rows and columns past K: y1 = 0, so +0
      }
      if (live && 4 * c < K) {
        float* p = dy1 + row * ld_dy + 4 * c;
        if (vout) {
          *reinterpret_cast<float4*>(p) = a;
        } else {
          p[0] = a.x;
          if (4 * c + 1 < K) p[1] = a.y;
          if (4 * c + 2 < K) p[2] = a.z;
          if (4 * c + 3 < K) p[3] = a.w;
        }
      }
    }
    __syncthreads();
    // ---- phase 2: the tile's contribution to dW1, db1, dw2, db2, loss (rows in order; dead rows are zeros) ---------
#pragma unroll
    for (int q = 0; q < NB; ++q) {
      const int blk = tid + q * R;
      if (blk < KC * NC) {
        const int tn = blk / KC, tk = blk - tn * KC;
        const float* dp = Dh + 4 * tn;
        const float* xp = Xs + 4 * tk;
#pragma unroll 4
        for (int r = 0; r < R; ++r) {
          const float4 a4 = *reinterpret_cast<const float4*>(dp + r * NP);
          const float4 b4 = *reinterpret_cast<const float4*>(xp + r * XS);
          const float a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[q][i][j] = fmaf(a[i], b[j], acc[q][i][j]);
        }
      }
    }
    if (tid < NP) {
      for (int r = 0; r < R; ++r) {
        accv += Dh[r * NP + tid];
        accw += Hg[r * NP + tid];
      }
    }
    if (tid == 0) {
      for (int r = 0; r < R; ++r) {
        accz += Dz[r];
        accl += Ls[r];
      }
    }
    if constexpr (kMask) {
      // column c on thread R - KP + c (past the db1 / dw2 threads, NP <= 64 <= R - KP + c): act_bwd_colsum_kernel's
      // sums at 64 columns, rows r0, r0 + 4, .. for r0 = 0 .. 3 from +0, then the four in r0 order.  Its slab stops at
      // M; the dead rows here add +0, which changes no sum (a sum that starts at +0 is never -0).
      const int c = tid - (R - KP);
      if (c >= 0 && c < K) {
        float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
        for (int r = 0; r < R; r += 4)
#pragma unroll
          for (int j = 0; j < 4; ++j) s[j] += Zs[(r + j) * XS + c];
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) v += s[j];
        zsum[t0 / R * K + c] = v;
      }
    }
    __syncthreads();
  }
  // ---- this CTA's sums: [N K | N | N | 1 | 1] -------------------------------------------------------------------------
  float* out = partial + (int64_t)blockIdx.x * (N * K + 2 * N + 2);
#pragma unroll
  for (int q = 0; q < NB; ++q) {
    const int blk = tid + q * R;
    if (blk < KC * NC) {
      const int tn = blk / KC, tk = blk - tn * KC;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (4 * tn + i < N && 4 * tk + j < K) out[(4 * tn + i) * K + 4 * tk + j] = acc[q][i][j];
    }
  }
  if (tid < N) {
    out[N * K + tid] = accv;
    out[N * K + N + tid] = accw;
  }
  if (tid == 0) {
    out[N * K + 2 * N] = accz;
    out[N * K + 2 * N + 1] = accl;
  }
}

// out[i] = sum over CTAs (ascending) of partial[c][i]; the last element (the loss sum) is scaled by inv_m
__global__ void __launch_bounds__(256)
tower_tail_reduce_kernel(const float* __restrict__ partial, int n_parts, int len, float inv_m, float* __restrict__ out) {
  __shared__ float red[8][32];
  const int o = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + o;
  float s = 0.f;
  if (i < len)
    for (int c = g; c < n_parts; c += 8) s += partial[(int64_t)c * len + i];
  red[g][o] = s;
  __syncthreads();
  if (g == 0 && i < len) {
    float r = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) r += red[k][o];
    out[i] = i == len - 1 ? r * inv_m : r;
  }
}

inline bool supported(int K, int N) { return K >= 1 && N >= 1 && K <= 64 && N <= 64; }

// out: [N K + 2 N + 2] = dW1 (row-major [N][K]), db1, dw2, db2, loss.  mask: masked mode, dy1 receives dZ and the
// workspace at colsum_offset() the per-tile column sums [tiles(M)][K].  Returns 0, or 1 bad argument / 2 workspace too
// small / 3 launch failure.
inline int run(const float* y1, int64_t ld_y, const float* w1, const float* b1, const float* w2, const float* b2,
               const float* labels, int64_t M, int32_t K, int32_t N, float* logits, float* dy1, int64_t ld_dy,
               float* out, void* workspace, size_t workspace_bytes_, cudaStream_t st, bool mask = false) {
  if (M < 1 || !supported(K, N) || !y1 || !w1 || !w2 || !labels || !logits || !dy1 || !out || ld_y < K || ld_dy < K) return 1;
  if (workspace_bytes_ < workspace_bytes(M, K, N)) return 2;
  const int KP = K <= 16 ? 16 : (K <= 32 ? 32 : 64);
  const int NP = N <= 16 ? 16 : (N <= 32 ? 32 : 64);
  const int grid = grid_for(M);
  int rows_per_cta = (int)((M + grid - 1) / grid);
  rows_per_cta = (rows_per_cta + kRows - 1) / kRows * kRows;        // whole tiles: every CTA but the last is full
  const float inv_m = 1.0f / (float)M;
  const size_t smem = smem_bytes(KP, NP, mask);
  float* partial = static_cast<float*>(workspace);
  float* zsum = partial + colsum_offset(M, K, N);
#ifdef TZK_CPU_SHIM
#define TZK_TAIL_ATTR(KP_, NP_, MASK_)
#else
#define TZK_TAIL_ATTR(KP_, NP_, MASK_)                                                                                \
  if (smem > 48 * 1024)                                                                                               \
    cudaFuncSetAttribute(tower_tail_bce_kernel<KP_, NP_, MASK_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
#endif
#define TZK_TAIL(KP_, NP_, MASK_)                                                                                     \
  do {                                                                                                                \
    TZK_TAIL_ATTR(KP_, NP_, MASK_)                                                                                    \
    TZK_LAUNCH((tower_tail_bce_kernel<KP_, NP_, MASK_>), grid, kRows, smem, st, y1, ld_y, w1, b1, w2, b2, labels, M,  \
               K, N, inv_m, rows_per_cta, logits, dy1, ld_dy, partial, zsum);                                         \
  } while (0)
#define TZK_TAIL_N(KP_, MASK_)                                                                                        \
  do {                                                                                                                \
    if (NP == 16) TZK_TAIL(KP_, 16, MASK_);                                                                           \
    else if (NP == 32) TZK_TAIL(KP_, 32, MASK_);                                                                      \
    else TZK_TAIL(KP_, 64, MASK_);                                                                                    \
  } while (0)
#define TZK_TAIL_K(MASK_)                                                                                             \
  do {                                                                                                                \
    if (KP == 16) TZK_TAIL_N(16, MASK_);                                                                              \
    else if (KP == 32) TZK_TAIL_N(32, MASK_);                                                                         \
    else TZK_TAIL_N(64, MASK_);                                                                                       \
  } while (0)
  if (mask) TZK_TAIL_K(true);
  else TZK_TAIL_K(false);
#undef TZK_TAIL_K
#undef TZK_TAIL_N
#undef TZK_TAIL
#undef TZK_TAIL_ATTR
  if (cudaGetLastError() != cudaSuccess) return 3;
  const int len = out_len(K, N);
  // (the grid that actually holds rows: CTAs past the last tile wrote zeros)
  TZK_LAUNCH((tower_tail_reduce_kernel), (len + 31) / 32, 256, 0, st, partial, grid, len, inv_m, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
}  // namespace tzk_tail
