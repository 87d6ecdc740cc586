// tzk_seq_attn.cuh — the sequence encoders of DEEP feature groups (tzrec/modules/sequence.py SelfAttentionEncoder and
// PoolingEncoder) over jagged sequence rows: sample b owns rows offsets[b] .. offsets[b + 1], of which the first
// L_b = min(len_b, max_len) are kept (max_len 0: all).
//
//   self_attn_pool_fwd  per (sample, head) work item: s_ij = (q_i sqrt(1/hd)) . k_j over the kept rows i, j < L_b,
//                       p = softmax over j, pooled[b, head] = sum_i sum_j p_ij v_j = sum_j c_j v_j (c_j = sum_i p_ij).
//                       Pass 1 walks each 64-row query tile over all key tiles with an online max / sum and writes one
//                       log-sum-exp per kept row and head (lse [N, H], 0 on cropped rows).  Pass 2 walks each key tile
//                       over all query tiles, forms c_j from p = exp(s - lse) and adds c_j v_j into the head's output.
//   self_attn_pool_bwd  from g = d pooled: u_j = g . v_j, D_i = sum_j p_ij u_j, dS_ij = p_ij (u_j - D_i),
//                       dq_i = sqrt(1/hd) sum_j dS_ij k_j, dk_j = sqrt(1/hd) sum_i dS_ij q_i, dv_j = c_j g.
//                       Pass A (query tiles outer) forms D (kept in the `dsum` workspace [N, H]) and dq; pass B (key
//                       tiles outer) forms dk, c and dv.  Cropped rows get zero gradients.
//   Scores are recomputed, never stored: no [T, T] or [N, E] attention state reaches HBM.  A CTA of 256 threads owns
//   one work item at a time (grid-stride over B H items), each thread a 4 x 4 block of the 64 x 64 score tile; q and k
//   tiles live transposed in shared memory ([hd][kLd], kLd = 68: float4 reads of 4 rows / 4 keys).  Each item writes
//   only its own outputs in a fixed order, so there are no float atomics and the bits do not depend on the grid.
//
//   jagged_pool_fwd / _bwd  one warp per sample: the sum, or the mean over max(L_b, 1), of the first L_b rows; the
//                       backward writes g (or g / max(L_b, 1)) to kept rows and 0 to cropped rows.
//
// FFMA in fp32 throughout, expf / logf at full precision.  Plain CUDA (no PTX): nvcc builds it in tzk_seq_attn.cu;
// g++ + tests/native/cuda_cpu_shim.h: tests/test_seq_encoders_cpu.py runs this source on the host against float64.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/tzk.h"
#include "tzk_batch_sum.cuh"
#include "tzk_launch.cuh"

namespace tzk_seq_attn {
constexpr int kTile = 64;                     // rows of a query or key tile
constexpr int kLd = kTile + 4;                // pitch of the transposed tiles (16-B aligned float4 reads)
constexpr int kThreads = 256;                 // 16 x 16 threads, a 4 x 4 block of the score tile each
constexpr int kMaxHd = 128;
constexpr int kPoolWarps = 8;

// shared memory (floats): Qt, Kt [hd][kLd]; P [kTile][kLd] (dS tiles; the column-sum scratch); row and column vectors
// lse, D, u, c [kTile] each; g [kMaxHd]
__host__ __device__ inline int64_t smem_floats(int hd) { return 2 * (int64_t)hd * kLd + kTile * kLd + 4 * kTile + kMaxHd; }
inline size_t smem_bytes(const tzk_seq_attn_args& a) { return (size_t)smem_floats(a.hd) * sizeof(float); }

// the descriptions the kernels cover (Fn.self_attn_pool_usable states the same for whole modules)
inline int check(const tzk_seq_attn_args& a, bool backward) {
  if (a.B < 0 || a.N < 0 || a.H < 1 || a.hd < 1 || a.hd > kMaxHd || a.max_len < 0) return 1;
  if ((int64_t)a.H * a.hd > (1 << 20) || a.B * a.H >= ((int64_t)1 << 31)) return 1;
  const int64_t E = (int64_t)a.H * a.hd;
  if (a.ldq < E || a.ldk < E || a.ldv < E) return 1;
  if (a.B == 0) return 0;
  if (!a.offsets) return 1;
  if (a.N > 0 && (!a.q || !a.k || !a.v || !a.lse)) return 1;            // no rows: empty tensors may have no storage
  if (!backward) return a.pooled ? 0 : 1;
  return (a.d_pooled && (a.N == 0 || (a.dq && a.dk && a.dv && a.dsum))) ? 0 : 1;
}

inline int check_pool(const tzk_jagged_pool_args& a, bool backward) {
  if (a.B < 0 || a.N < 0 || a.D < 1 || a.max_len < 0 || (a.mean != 0 && a.mean != 1)) return 1;
  if (a.B == 0) return 0;
  if (!a.offsets) return 1;
  return backward ? ((a.d_out && (a.N == 0 || a.d_seq)) ? 0 : 1) : (((a.N == 0 || a.seq) && a.out) ? 0 : 1);
}

struct Item {
  int64_t r0;      // first row of the sample
  int64_t len;     // its rows
  int L;           // kept rows
  int nt;          // 64-row tiles over the kept rows
  int col0;        // first column of the head
};

__device__ inline Item item_of(const tzk_seq_attn_args& a, int64_t b, int h) {
  Item it;
  it.r0 = a.offsets[b];
  it.len = a.offsets[b + 1] - it.r0;
  const int64_t L = (a.max_len > 0 && it.len > a.max_len) ? a.max_len : it.len;
  it.L = (int)L;
  it.nt = (it.L + kTile - 1) / kTile;
  it.col0 = h * a.hd;
  return it;
}

// rows t0 .. t0 + 63 of the head's columns of src (row stride ld), times `scale`, transposed into T [hd][kLd]; rows at
// or beyond L are zeros
__device__ inline void load_tile_t(float* T, const float* src, int64_t ld, const Item& it, int t0, int hd, float scale) {
  for (int e = threadIdx.x; e < kTile * hd; e += kThreads) {
    const int r = e / hd, d = e % hd;
    T[d * kLd + r] = (t0 + r < it.L) ? src[(it.r0 + t0 + r) * ld + it.col0 + d] * scale : 0.f;
  }
}

// u_j = g . v_j for the 64 keys of the tile at t0 (0 beyond L): four lanes per key over d = p, p + 4, ..
__device__ inline void load_u(float* u, const float* g, const tzk_seq_attn_args& a, const Item& it, int t0) {
  const int j = threadIdx.x >> 2, p = threadIdx.x & 3;
  float s = 0.f;
  if (t0 + j < it.L) {
    const float* v = a.v + (it.r0 + t0 + j) * a.ldv + it.col0;
    for (int d = p; d < a.hd; d += 4) s = fmaf(g[d], v[d], s);
  }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  if (p == 0) u[j] = s;
}

// s[r][c] = Qt[:, 4 ty + r] . Kt[:, 4 tx + c]; threads whose rows or keys are all beyond the tile's valid counts skip
__device__ inline void scores(float (&s)[4][4], const float* Qt, const float* Kt, int hd, int ty, int tx, int nq,
                              int nk) {
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) s[r][c] = 0.f;
  if (4 * ty >= nq || 4 * tx >= nk) return;
  for (int d = 0; d < hd; ++d) {
    const float4 qa = *reinterpret_cast<const float4*>(Qt + d * kLd + 4 * ty);
    const float4 kb = *reinterpret_cast<const float4*>(Kt + d * kLd + 4 * tx);
    const float qv[4] = {qa.x, qa.y, qa.z, qa.w}, kv[4] = {kb.x, kb.y, kb.z, kb.w};
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) s[r][c] = fmaf(qv[r], kv[c], s[r][c]);
  }
}

// sum / max over the 16 threads of a score-tile row (lanes tx = 0..15 of one half warp)
__device__ inline float row_sum(float x) {
  for (int m = 8; m >= 1; m >>= 1) x += __shfl_xor_sync(0xffffffffu, x, m);
  return x;
}
__device__ inline float row_max(float x) {
  for (int m = 8; m >= 1; m >>= 1) x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, m));
  return x;
}

// c_j of the key tile: the column sums `cacc` of the 16 thread rows, added in ty order (P as scratch)
__device__ inline void column_sums(float* c, float* P, const float (&cacc)[4], int ty, int tx) {
  __syncthreads();
#pragma unroll
  for (int q = 0; q < 4; ++q) P[ty * kTile + 4 * tx + q] = cacc[q];
  __syncthreads();
  if (threadIdx.x < kTile) {
    float s = 0.f;
    for (int y = 0; y < 16; ++y) s += P[y * kTile + threadIdx.x];
    c[threadIdx.x] = s;
  }
  __syncthreads();
}

struct Smem {
  float *Qt, *Kt, *P, *lse, *D, *u, *c, *g;
  __device__ explicit Smem(float* base, int hd) {
    Qt = base;
    Kt = Qt + hd * kLd;
    P = Kt + hd * kLd;
    lse = P + kTile * kLd;
    D = lse + kTile;
    u = D + kTile;
    c = u + kTile;
    g = c + kTile;
  }
};

__global__ void __launch_bounds__(kThreads, 2) self_attn_pool_fwd_kernel(const __grid_constant__ tzk_seq_attn_args a) {
  TZK_DYN_SMEM(float, smem);
  Smem S(smem, a.hd);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, hd = a.hd;
  const float scale = sqrtf(1.f / (float)hd);
  const int64_t items = a.B * a.H, E = (int64_t)a.H * hd;
  for (int64_t w = blockIdx.x; w < items; w += gridDim.x) {
    const int64_t b = w / a.H;
    const int h = (int)(w % a.H);
    const Item it = item_of(a, b, h);
    int qcur = -1, kcur = -1;
    // pass 1: lse of every kept row
    for (int qi = 0; qi < it.nt; ++qi) {
      if (qcur != qi) {
        __syncthreads();
        load_tile_t(S.Qt, a.q, a.ldq, it, qi * kTile, hd, scale);
        qcur = qi;
      }
      float m[4], l[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) m[r] = -INFINITY, l[r] = 0.f;
      for (int kj = 0; kj < it.nt; ++kj) {
        if (kcur != kj) {
          __syncthreads();
          load_tile_t(S.Kt, a.k, a.ldk, it, kj * kTile, hd, 1.f);
          kcur = kj;
        }
        __syncthreads();
        const int nq = it.L - qi * kTile, nk = it.L - kj * kTile;
        float s[4][4];
        scores(s, S.Qt, S.Kt, hd, ty, tx, nq, nk);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          float mx = -INFINITY;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            if (4 * tx + c >= nk) s[r][c] = -INFINITY;
            mx = fmaxf(mx, s[r][c]);
          }
          const float mn = fmaxf(m[r], row_max(mx));        // finite: tile kj holds at least one kept key
          float e = 0.f;
#pragma unroll
          for (int c = 0; c < 4; ++c) e += expf(s[r][c] - mn);
          l[r] = l[r] * expf(m[r] - mn) + row_sum(e);
          m[r] = mn;
        }
      }
      if (tx == 0)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = qi * kTile + 4 * ty + r;
          if (i < it.L) a.lse[(it.r0 + i) * a.H + h] = m[r] + logf(l[r]);
        }
    }
    for (int64_t i = it.L + tid; i < it.len; i += kThreads) a.lse[(it.r0 + i) * a.H + h] = 0.f;
    __syncthreads();                          // the lse rows are read back below
    // pass 2: c_j per key tile, then pooled += c_j v_j
    float acc = 0.f;
    for (int kj = 0; kj < it.nt; ++kj) {
      if (kcur != kj) {
        __syncthreads();
        load_tile_t(S.Kt, a.k, a.ldk, it, kj * kTile, hd, 1.f);
        kcur = kj;
      }
      const int nk = it.L - kj * kTile;
      float cacc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int qi = 0; qi < it.nt; ++qi) {
        __syncthreads();
        if (qcur != qi) {
          load_tile_t(S.Qt, a.q, a.ldq, it, qi * kTile, hd, scale);
          qcur = qi;
        }
        const int nq = it.L - qi * kTile;
        if (tid < kTile) S.lse[tid] = tid < nq ? a.lse[(it.r0 + qi * kTile + tid) * a.H + h] : 0.f;
        __syncthreads();
        float s[4][4];
        scores(s, S.Qt, S.Kt, hd, ty, tx, nq, nk);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const bool row_ok = 4 * ty + r < nq;
          const float ls = S.lse[4 * ty + r];
#pragma unroll
          for (int c = 0; c < 4; ++c) cacc[c] += (row_ok && 4 * tx + c < nk) ? expf(s[r][c] - ls) : 0.f;
        }
      }
      column_sums(S.c, S.P, cacc, ty, tx);
      if (tid < hd) {
        const int n = nk < kTile ? nk : kTile;
        const float* v = a.v + (it.r0 + kj * kTile) * a.ldv + it.col0 + tid;
        for (int j = 0; j < n; ++j) acc = fmaf(S.c[j], v[j * a.ldv], acc);
      }
    }
    if (tid < hd) a.pooled[b * E + it.col0 + tid] = acc;
    __syncthreads();
  }
}

// MT: head columns per thread in the dq / dk products (hd <= 16 MT), so the accumulators take only the registers hd
// needs
template <int MT>
__global__ void __launch_bounds__(kThreads, 1)
    self_attn_pool_bwd_kernel(const __grid_constant__ tzk_seq_attn_args a) {
  TZK_DYN_SMEM(float, smem);
  Smem S(smem, a.hd);
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15, hd = a.hd;
  const float scale = sqrtf(1.f / (float)hd);
  const int64_t items = a.B * a.H, E = (int64_t)a.H * hd;
  for (int64_t w = blockIdx.x; w < items; w += gridDim.x) {
    const int64_t b = w / a.H;
    const int h = (int)(w % a.H);
    const Item it = item_of(a, b, h);
    __syncthreads();
    if (tid < hd) S.g[tid] = a.d_pooled[b * E + it.col0 + tid];
    __syncthreads();
    int qcur = -1, kcur = -1;
    // loads key tile kj and its u_j once per change of tile
    auto key_tile = [&](int kj) {
      if (kcur == kj) return;
      __syncthreads();
      load_tile_t(S.Kt, a.k, a.ldk, it, kj * kTile, hd, 1.f);
      load_u(S.u, S.g, a, it, kj * kTile);
      kcur = kj;
    };
    auto query_tile = [&](int qi) {         // the q tile and its lse / D rows (D only once pass A has written it)
      __syncthreads();
      if (qcur != qi) {
        load_tile_t(S.Qt, a.q, a.ldq, it, qi * kTile, hd, scale);
        qcur = qi;
      }
      const int nq = it.L - qi * kTile;
      if (tid < kTile) S.lse[tid] = tid < nq ? a.lse[(it.r0 + qi * kTile + tid) * a.H + h] : 0.f;
    };
    // pass A: per query tile D_i, then dq_i
    for (int qi = 0; qi < it.nt; ++qi) {
      query_tile(qi);
      const int nq = it.L - qi * kTile;
      float dacc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int kj = 0; kj < it.nt; ++kj) {
        key_tile(kj);
        __syncthreads();
        const int nk = it.L - kj * kTile;
        float s[4][4];
        scores(s, S.Qt, S.Kt, hd, ty, tx, nq, nk);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float ls = S.lse[4 * ty + r];
#pragma unroll
          for (int c = 0; c < 4; ++c)
            if (4 * tx + c < nk) dacc[r] = fmaf(expf(s[r][c] - ls), S.u[4 * tx + c], dacc[r]);
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) dacc[r] = row_sum(dacc[r]);
      __syncthreads();
      if (tx == 0)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = 4 * ty + r;
          S.D[i] = dacc[r];
          if (i < nq) a.dsum[(it.r0 + qi * kTile + i) * a.H + h] = dacc[r];
        }
      float acc[4][MT];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int mm = 0; mm < MT; ++mm) acc[r][mm] = 0.f;
      for (int kj = 0; kj < it.nt; ++kj) {
        key_tile(kj);
        __syncthreads();
        const int nk = it.L - kj * kTile;
        float s[4][4];
        scores(s, S.Qt, S.Kt, hd, ty, tx, nq, nk);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float ls = S.lse[4 * ty + r], Di = S.D[4 * ty + r];
          const bool row_ok = 4 * ty + r < nq;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int j = 4 * tx + c;
            S.P[(4 * ty + r) * kLd + j] = (row_ok && j < nk) ? expf(s[r][c] - ls) * (S.u[j] - Di) : 0.f;
          }
        }
        __syncthreads();
        if (4 * ty < nq) {
          const int n = nk < kTile ? nk : kTile;
          for (int j = 0; j < n; ++j) {
            float ds[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) ds[r] = S.P[(4 * ty + r) * kLd + j];
#pragma unroll
            for (int mm = 0; mm < MT; ++mm) {
              const int d = tx + 16 * mm;
              if (d < hd) {
                const float kv = S.Kt[d * kLd + j];
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[r][mm] = fmaf(ds[r], kv, acc[r][mm]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = 4 * ty + r;
        if (i >= nq) continue;
        float* dst = a.dq + (it.r0 + qi * kTile + i) * E + it.col0;
#pragma unroll
        for (int mm = 0; mm < MT; ++mm)
          if (tx + 16 * mm < hd) dst[tx + 16 * mm] = scale * acc[r][mm];
      }
    }
    // cropped rows: zero gradients
    for (int64_t e = (int64_t)it.L * hd + tid; e < it.len * hd; e += kThreads) {
      const int64_t off = (it.r0 + e / hd) * E + it.col0 + e % hd;
      a.dq[off] = 0.f;
      a.dk[off] = 0.f;
      a.dv[off] = 0.f;
    }
    // pass B: per key tile dk_j, c_j and dv_j
    for (int kj = 0; kj < it.nt; ++kj) {
      key_tile(kj);
      const int nk = it.L - kj * kTile;
      float acc[4][MT];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int mm = 0; mm < MT; ++mm) acc[r][mm] = 0.f;
      float cacc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int qi = 0; qi < it.nt; ++qi) {
        query_tile(qi);
        const int nq = it.L - qi * kTile;
        if (tid < kTile) S.D[tid] = tid < nq ? a.dsum[(it.r0 + qi * kTile + tid) * a.H + h] : 0.f;
        __syncthreads();
        float s[4][4];
        scores(s, S.Qt, S.Kt, hd, ty, tx, nq, nk);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int i = 4 * ty + r;
          const float ls = S.lse[i], Di = S.D[i];
          const bool row_ok = i < nq;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int j = 4 * tx + c;
            const float p = (row_ok && j < nk) ? expf(s[r][c] - ls) : 0.f;
            cacc[c] += p;
            S.P[j * kLd + i] = p * (S.u[j] - Di);        // dS transposed: [key][query]
          }
        }
        __syncthreads();
        if (4 * ty < nk) {
          const int n = nq < kTile ? nq : kTile;
          for (int i = 0; i < n; ++i) {
            float ds[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) ds[r] = S.P[(4 * ty + r) * kLd + i];
#pragma unroll
            for (int mm = 0; mm < MT; ++mm) {
              const int d = tx + 16 * mm;
              if (d < hd) {
                const float qv = S.Qt[d * kLd + i];
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[r][mm] = fmaf(ds[r], qv, acc[r][mm]);
              }
            }
          }
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int j = 4 * ty + r;
        if (j >= nk) continue;
        float* dst = a.dk + (it.r0 + kj * kTile + j) * E + it.col0;
#pragma unroll
        for (int mm = 0; mm < MT; ++mm)
          if (tx + 16 * mm < hd) dst[tx + 16 * mm] = acc[r][mm];     // Qt carries the scale already
      }
      column_sums(S.c, S.P, cacc, ty, tx);
      const int n = nk < kTile ? nk : kTile;
      for (int e = tid; e < n * hd; e += kThreads) {
        const int j = e / hd, d = e % hd;
        a.dv[(it.r0 + kj * kTile + j) * E + it.col0 + d] = S.c[j] * S.g[d];
      }
    }
  }
}

__global__ void __launch_bounds__(kPoolWarps * 32) jagged_pool_fwd_kernel(const __grid_constant__ tzk_jagged_pool_args a) {
  const int lane = threadIdx.x & 31;
  for (int64_t b = (int64_t)blockIdx.x * kPoolWarps + (threadIdx.x >> 5); b < a.B; b += (int64_t)gridDim.x * kPoolWarps) {
    const int64_t r0 = a.offsets[b], len = a.offsets[b + 1] - r0;
    const int64_t L = (a.max_len > 0 && len > a.max_len) ? a.max_len : len;
    const float cnt = (float)(L > 1 ? L : 1);
    for (int d = lane; d < a.D; d += 32) {
      float s = 0.f;
      for (int64_t i = 0; i < L; ++i) s += a.seq[(r0 + i) * a.D + d];
      a.out[b * a.D + d] = a.mean ? s / cnt : s;
    }
  }
}

__global__ void __launch_bounds__(kPoolWarps * 32) jagged_pool_bwd_kernel(const __grid_constant__ tzk_jagged_pool_args a) {
  const int lane = threadIdx.x & 31;
  for (int64_t b = (int64_t)blockIdx.x * kPoolWarps + (threadIdx.x >> 5); b < a.B; b += (int64_t)gridDim.x * kPoolWarps) {
    const int64_t r0 = a.offsets[b], len = a.offsets[b + 1] - r0;
    const int64_t L = (a.max_len > 0 && len > a.max_len) ? a.max_len : len;
    const float cnt = (float)(L > 1 ? L : 1);
    for (int d = lane; d < a.D; d += 32) {
      const float g = a.mean ? a.d_out[b * a.D + d] / cnt : a.d_out[b * a.D + d];
      for (int64_t i = 0; i < len; ++i) a.d_seq[(r0 + i) * a.D + d] = i < L ? g : 0.f;
    }
  }
}

// ---- launchers (return 0, or 1 on arguments outside the cover) --------------------------------------------------------
inline int fwd(const tzk_seq_attn_args& a, int grid, cudaStream_t stream) {
  if (check(a, false) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  const size_t smem = smem_bytes(a);
  tzk_batch_sum::opt_in_smem(self_attn_pool_fwd_kernel, smem);
  TZK_LAUNCH((self_attn_pool_fwd_kernel), grid, kThreads, smem, stream, a);
  return 0;
}

template <int MT>
inline void launch_bwd(const tzk_seq_attn_args& a, int grid, size_t smem, cudaStream_t stream) {
  tzk_batch_sum::opt_in_smem(self_attn_pool_bwd_kernel<MT>, smem);
  TZK_LAUNCH((self_attn_pool_bwd_kernel<MT>), grid, kThreads, smem, stream, a);
}

inline int bwd(const tzk_seq_attn_args& a, int grid, cudaStream_t stream) {
  if (check(a, true) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  const size_t smem = smem_bytes(a);
  const int mt = (a.hd + 15) / 16;
  if (mt <= 1) launch_bwd<1>(a, grid, smem, stream);
  else if (mt <= 2) launch_bwd<2>(a, grid, smem, stream);
  else if (mt <= 4) launch_bwd<4>(a, grid, smem, stream);
  else launch_bwd<8>(a, grid, smem, stream);
  return 0;
}

inline int pool_fwd(const tzk_jagged_pool_args& a, int grid, cudaStream_t stream) {
  if (check_pool(a, false) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  TZK_LAUNCH((jagged_pool_fwd_kernel), grid, kPoolWarps * 32, 0, stream, a);
  return 0;
}

inline int pool_bwd(const tzk_jagged_pool_args& a, int grid, cudaStream_t stream) {
  if (check_pool(a, true) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  TZK_LAUNCH((jagged_pool_bwd_kernel), grid, kPoolWarps * 32, 0, stream, a);
  return 0;
}
}  // namespace tzk_seq_attn
