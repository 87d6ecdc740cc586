// tzk_tdm.cuh — TDM's multi-window DIN attention (tzrec/modules/sequence.py MultiWindowDINEncoder) over jagged
// sequence rows: sample b owns rows offsets[b] .. offsets[b + 1] of seq [N, C].
//
//   fwd  per row t of sample b at position p = t - offsets[b] < S (S = sum of the window lengths):
//          x_t = [k_t, q k_t, q]  (q zero-padded from Dq to C)
//          h = act(W_l h + b_l) for the 1..3 attention layers (ReLU or one-slope PReLU), z_t = lin_w . h + lin_b,
//          a_t = PReLU_active(z_t)
//        out[b] = [window_0 .. window_{L-1}, q], window_w = sum over its rows of a_t k_t / max(min(len - cum_w, W_w), 1)
//        One warp per sample; rows in groups of kRows, every layer's output unit j on lane j and j + 32.  Rows at
//        p >= S never contribute (the reference crops them).  z [N] is the only saved state (0 on rows p >= S).
//   bwd  d_seq, d_query and every parameter gradient from d_out.  Each CTA owns the contiguous samples
//        [B g / G, B (g + 1) / G) and walks their rows in tiles of kWarpsBwd * kRows: every warp recomputes its rows'
//        hidden layers, back-propagates them from the saved z, writes d_seq and leaves d_u, the layer inputs and the
//        rows' d_query shares in shared memory; then each thread adds the tile's rows in order into its own entries of
//        the CTA's parameter-gradient row, and thread c into column c of the running d_query.
//        tzk_batch_sum::reduce adds the CTA rows in CTA order: the bits depend only on the grid.
//
// Weights, biases and slopes live in shared memory, transposed to [K][Hs] with an odd row pitch Hs = H | 1, so lanes
// over output units and lanes over input units both read without bank conflicts.  FFMA in fp32 throughout.
// Plain CUDA (no PTX): nvcc builds it in tzk_tdm.cu; g++ + tests/native/cuda_cpu_shim.h: tests/test_tdm_cpu.py runs
// this source on the host against float64.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/tzk.h"
#include "tzk_batch_sum.cuh"
#include "tzk_launch.cuh"

namespace tzk_tdm {
constexpr int kRows = 4;                      // rows of one warp's group (a float4 per input unit)
constexpr int kWarpsFwd = 8, kWarpsBwd = 4;
constexpr int kMaxC = 128, kMaxH = 64, kMaxS = 256;
constexpr int kMaxLayers = TZK_TDM_MAX_LAYERS, kMaxWindows = TZK_TDM_MAX_WINDOWS;
constexpr size_t kMaxSmem = 227 * 1024;       // H100's opt-in shared memory per CTA

__host__ __device__ inline int pad4(int n) { return (n + 3) & ~3; }
__host__ __device__ inline int in_dim(const tzk_tdm_args& a, int l) { return l == 0 ? 3 * a.C : a.hidden[l - 1]; }
__host__ __device__ inline int pitch(const tzk_tdm_args& a, int l) { return a.hidden[l] | 1; }
__host__ __device__ inline int h_last(const tzk_tdm_args& a) { return a.hidden[a.n_layers - 1]; }
__host__ __device__ inline int window_sum(const tzk_tdm_args& a) {
  int s = 0;
  for (int w = 0; w < a.L; ++w) s += a.windows[w];
  return s;
}
__host__ __device__ inline int slope_n(const tzk_tdm_args& a) { return a.act == TZK_TDM_PRELU ? 1 : 0; }

// parameters in shared memory: per layer W^T [K][Hs], b [H], slope [1]; then lin_w [H_last], lin_b, act_w
__host__ __device__ inline int params_smem_floats(const tzk_tdm_args& a) {
  int n = 0;
  for (int l = 0; l < a.n_layers; ++l) n += in_dim(a, l) * pitch(a, l) + a.hidden[l] + 1;
  return pad4(n + h_last(a) + 2);
}
// parameter gradients (dparams, and one partials row per CTA): per layer dW [H][K] (the weight's layout), db [H],
// dslope [PReLU only]; then d lin_w [H_last], d lin_b, d act_w
__host__ __device__ inline int64_t param_floats(const tzk_tdm_args& a) {
  int64_t n = 0;
  for (int l = 0; l < a.n_layers; ++l) n += (int64_t)a.hidden[l] * in_dim(a, l) + a.hidden[l] + slope_n(a);
  return n + h_last(a) + 2;
}
// per-warp buffers: xs [3C][kRows], then per layer u [H][kRows] and h [H][kRows]; fwd adds a [S]; bwd adds dh
// [kMaxH][kRows], dq [kRows][C] and the row scalars (d z, d act_w, d slope per layer, sample)
__host__ __device__ inline int layers_floats(const tzk_tdm_args& a) {
  int n = 3 * a.C * kRows;
  for (int l = 0; l < a.n_layers; ++l) n += 2 * a.hidden[l] * kRows;
  return n;
}
constexpr int kRowScalars = (2 + kMaxLayers + 1) * kRows;
__host__ __device__ inline int warp_floats(const tzk_tdm_args& a, bool backward) {
  return layers_floats(a) + (backward ? kMaxH * kRows + kRows * a.C + kRowScalars : pad4(window_sum(a)));
}
inline size_t smem_bytes(const tzk_tdm_args& a, bool backward) {
  size_t f = params_smem_floats(a) + kMaxS;                       // + the window of every position
  f += backward ? (size_t)pad4((int)param_floats(a)) + (size_t)kWarpsBwd * warp_floats(a, true)
                : (size_t)kWarpsFwd * warp_floats(a, false);
  return f * sizeof(float);
}

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// the descriptions the kernels cover (the Python side's Fn.multiwindow_din_usable states the same for whole modules)
inline int check(const tzk_tdm_args& a, bool backward) {
  if (a.B < 0 || a.B >= ((int64_t)1 << 31) || a.N < 0 || a.N >= ((int64_t)1 << 31)) return 1;
  if (a.C < 4 || a.C > kMaxC || a.C % 4 != 0 || a.Dq < 1 || a.Dq > a.C) return 1;
  if (a.n_layers < 1 || a.n_layers > kMaxLayers || (a.act != TZK_TDM_RELU && a.act != TZK_TDM_PRELU)) return 1;
  for (int l = 0; l < a.n_layers; ++l)
    if (a.hidden[l] < 1 || a.hidden[l] > kMaxH) return 1;
  if (a.L < 1 || a.L > kMaxWindows) return 1;
  for (int w = 0; w < a.L; ++w)
    if (a.windows[w] < 1 || a.windows[w] > kMaxS) return 1;
  if (window_sum(a) > kMaxS || smem_bytes(a, backward) > kMaxSmem) return 1;
  if (a.B == 0) return 0;
  if (!aligned16(a.seq) || !a.offsets || !a.query || !a.lin_w || !a.lin_b || !a.act_w) return 1;
  if (a.N > 0 && (!a.seq || !a.z)) return 1;                     // all-zero lengths: no rows
  for (int l = 0; l < a.n_layers; ++l)
    if (!a.w[l] || !a.b[l] || (a.act == TZK_TDM_PRELU && !a.slope[l])) return 1;
  if (!backward) return a.out ? 0 : 1;
  return (a.d_out && aligned16(a.d_seq) && (a.N == 0 || a.d_seq) && a.d_query) ? 0 : 1;
}

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

// offset of layer l's parameters in shared memory (W^T [K][Hs], then b [H], then the slope)
__host__ __device__ inline int layer_off(const tzk_tdm_args& a, int l) {
  int n = 0;
  for (int m = 0; m < l; ++m) n += in_dim(a, m) * pitch(a, m) + a.hidden[m] + 1;
  return n;
}

struct Smem {                     // shared-memory carve-up, identical in both kernels up to `tail`
  float* base;
  float* lin_w;
  float* lin_b;
  float* act_w;
  int* win;                       // [kMaxS] window of position p
  float* tail;
  __device__ float* wt(const tzk_tdm_args& a, int l) const { return base + layer_off(a, l); }
  __device__ float* bias(const tzk_tdm_args& a, int l) const { return wt(a, l) + in_dim(a, l) * pitch(a, l); }
  __device__ float slope(const tzk_tdm_args& a, int l) const { return bias(a, l)[a.hidden[l]]; }
};

__device__ inline Smem carve(const tzk_tdm_args& a, float* base) {
  Smem s;
  s.base = base;
  s.lin_w = base + layer_off(a, a.n_layers);
  s.lin_b = s.lin_w + h_last(a);
  s.act_w = s.lin_b + 1;
  float* p = base + params_smem_floats(a);
  s.win = reinterpret_cast<int*>(p);
  s.tail = p + kMaxS;
  return s;
}

// every thread of the CTA: the parameters into shared memory (weights transposed), and the position -> window table
__device__ inline void load_params(const tzk_tdm_args& a, const Smem& s) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int l = 0; l < a.n_layers; ++l) {
    const int K = in_dim(a, l), H = a.hidden[l], Hs = pitch(a, l);
    float* wt = s.wt(a, l);
    float* bias = s.bias(a, l);
    for (int e = tid; e < H * K; e += nt) {
      const int j = e / K, i = e % K;
      wt[i * Hs + j] = a.w[l][e];
    }
    for (int j = tid; j < H; j += nt) bias[j] = a.b[l][j];
    if (tid == 0) bias[H] = a.act == TZK_TDM_PRELU ? a.slope[l][0] : 0.f;
  }
  for (int j = tid; j < h_last(a); j += nt) s.lin_w[j] = a.lin_w[j];
  if (tid == 0) {
    s.lin_b[0] = a.lin_b[0];
    s.act_w[0] = a.act_w[0];
  }
  if (tid == 0) {
    int p = 0;
    for (int w = 0; w < a.L; ++w)
      for (int r = 0; r < a.windows[w]; ++r) s.win[p++] = w;
  }
}

struct Warp {                     // one warp's buffers: xs [3C][kRows], then per layer u [H][kRows] (pre-activations;
  float* xs;                      // bwd: overwritten by d u) and h [H][kRows] (outputs), then `extra`
  float* extra;
  __device__ float* u(const tzk_tdm_args& a, int l) const {
    float* p = xs + 3 * a.C * kRows;
    for (int m = 0; m < l; ++m) p += 2 * a.hidden[m] * kRows;
    return p;
  }
  __device__ float* h(const tzk_tdm_args& a, int l) const { return u(a, l) + a.hidden[l] * kRows; }
};

__device__ inline Warp carve_warp(const tzk_tdm_args& a, float* base) {
  Warp w;
  w.xs = base;
  w.extra = base + layers_floats(a);
  return w;
}

// xs[i][r] = x_i of row r: rows[r] < 0 (no row) gives zeros.  q of row r: query row qb[r] (zero-padded to C).
__device__ inline void stage_x(const tzk_tdm_args& a, const Warp& w, const int64_t (&rows)[kRows],
                               const int64_t (&qb)[kRows], int lane) {
  const int C = a.C;
  const int r = lane % kRows;                      // the same row on every pass (kRows divides 32)
  const int64_t row = r == 0 ? rows[0] : r == 1 ? rows[1] : r == 2 ? rows[2] : rows[3];
  const int64_t qrow = r == 0 ? qb[0] : r == 1 ? qb[1] : r == 2 ? qb[2] : qb[3];
  static_assert(kRows == 4 && 32 % kRows == 0, "stage_x picks one of four rows per lane");
  for (int e = lane; e < C * kRows; e += 32) {
    const int c = e / kRows;
    float k = 0.f, q = 0.f;
    if (row >= 0) {
      k = a.seq[row * C + c];
      q = c < a.Dq ? a.query[qrow * a.Dq + c] : 0.f;
    }
    w.xs[c * kRows + r] = k;
    w.xs[(C + c) * kRows + r] = q * k;
    w.xs[(2 * C + c) * kRows + r] = q;
  }
  __syncwarp();
}

// the attention layers for the warp's kRows rows: u = W in + b, h = act(u); lane j owns units j and j + 32
__device__ inline void mlp_fwd(const tzk_tdm_args& a, const Smem& s, const Warp& w, int lane) {
  const float* in = w.xs;
  for (int l = 0; l < a.n_layers; ++l) {
    const int K = in_dim(a, l), H = a.hidden[l], Hs = pitch(a, l);
    const float* wt = s.wt(a, l);
    const bool v0 = lane < H, v1 = lane + 32 < H;
    float4 c0 = make_float4(0.f, 0.f, 0.f, 0.f), c1 = c0;
    for (int i = 0; i < K; ++i) {
      const float4 x = ld4(in + i * kRows);
      const float w0 = v0 ? wt[i * Hs + lane] : 0.f;
      const float w1 = v1 ? wt[i * Hs + lane + 32] : 0.f;
      c0.x += w0 * x.x; c0.y += w0 * x.y; c0.z += w0 * x.z; c0.w += w0 * x.w;
      c1.x += w1 * x.x; c1.y += w1 * x.y; c1.z += w1 * x.z; c1.w += w1 * x.w;
    }
    const float sl = s.slope(a, l);
    const bool prelu = a.act == TZK_TDM_PRELU;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
      const int j = lane + 32 * half;
      if (j >= H) break;
      const float bj = s.bias(a, l)[j];
      float4 u = half ? c1 : c0;
      u.x += bj; u.y += bj; u.z += bj; u.w += bj;
      float4 h;
      h.x = u.x > 0.f ? u.x : (prelu ? sl * u.x : 0.f);
      h.y = u.y > 0.f ? u.y : (prelu ? sl * u.y : 0.f);
      h.z = u.z > 0.f ? u.z : (prelu ? sl * u.z : 0.f);
      h.w = u.w > 0.f ? u.w : (prelu ? sl * u.w : 0.f);
      st4(w.u(a, l) + j * kRows, u);
      st4(w.h(a, l) + j * kRows, h);
    }
    __syncwarp();
    in = w.h(a, l);
  }
}

// z of row r = lin_w . h_last + lin_b, the same bits on every lane (xor butterfly)
__device__ inline float score(const tzk_tdm_args& a, const Smem& s, const Warp& w, int r, int lane) {
  const int H = h_last(a);
  const float* h = w.h(a, a.n_layers - 1);
  float v = 0.f;
  for (int j = lane; j < H; j += 32) v += s.lin_w[j] * h[j * kRows + r];
  return warp_sum(v) + s.lin_b[0];
}

__device__ __forceinline__ float prelu1(float z, float slope) { return z > 0.f ? z : slope * z; }

// dynamic shared memory: smem_bytes(a, false)
__global__ void __launch_bounds__(kWarpsFwd * 32) fwd_kernel(const __grid_constant__ tzk_tdm_args a) {
  TZK_DYN_SMEM(float, smem);
  const Smem s = carve(a, smem);
  const int lane = threadIdx.x % 32, wid = threadIdx.x / 32;
  const Warp w = carve_warp(a, s.tail + wid * warp_floats(a, false));
  float* as = w.extra;                                   // a_t of the sample's positions
  load_params(a, s);
  __syncthreads();
  const int C = a.C, L = a.L, S = window_sum(a);
  const int64_t OC = (int64_t)(L + 1) * C;
  for (int64_t b = (int64_t)blockIdx.x * kWarpsFwd + wid; b < a.B; b += (int64_t)gridDim.x * kWarpsFwd) {
    const int64_t row0 = a.offsets[b], len = a.offsets[b + 1] - row0;
    const int n = (int)(len < S ? len : S);
    for (int p0 = 0; p0 < n; p0 += kRows) {
      int64_t rows[kRows], qb[kRows];
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        rows[r] = p0 + r < n ? row0 + p0 + r : -1;
        qb[r] = b;
      }
      stage_x(a, w, rows, qb, lane);
      mlp_fwd(a, s, w, lane);
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const float z = score(a, s, w, r, lane);
        if (p0 + r < n && lane == r) {
          a.z[row0 + p0 + r] = z;
          as[p0 + r] = prelu1(z, s.act_w[0]);
        }
      }
      __syncwarp();
    }
    for (int64_t p = n + lane; p < len; p += 32) a.z[row0 + p] = 0.f;
    float* o = a.out + b * OC;
    for (int c = 4 * lane; c < C; c += 128) {
      for (int wi = 0, cum = 0; wi < L; cum += a.windows[wi], ++wi) {
        const int W = a.windows[wi];
        const int end = cum + W < n ? cum + W : n;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int p = cum; p < end; ++p) {
          const float4 k = ld4(a.seq + (row0 + p) * C + c);
          const float at = as[p];
          acc.x += at * k.x; acc.y += at * k.y; acc.z += at * k.z; acc.w += at * k.w;
        }
        const int64_t m = len - cum < W ? len - cum : W;
        const float cnt = (float)(m > 1 ? m : 1);
        st4(o + wi * C + c, make_float4(acc.x / cnt, acc.y / cnt, acc.z / cnt, acc.w / cnt));
      }
      float4 q;
      q.x = c + 0 < a.Dq ? a.query[b * a.Dq + c + 0] : 0.f;
      q.y = c + 1 < a.Dq ? a.query[b * a.Dq + c + 1] : 0.f;
      q.z = c + 2 < a.Dq ? a.query[b * a.Dq + c + 2] : 0.f;
      q.w = c + 3 < a.Dq ? a.query[b * a.Dq + c + 3] : 0.f;
      st4(o + L * C + c, q);
    }
    __syncwarp();
  }
}

// dynamic shared memory: smem_bytes(a, true).  partials: gridDim.x rows of param_floats(a).
__global__ void __launch_bounds__(kWarpsBwd * 32) bwd_kernel(const __grid_constant__ tzk_tdm_args a,
                                                             float* __restrict__ partials) {
  TZK_DYN_SMEM(float, smem);
  const Smem s = carve(a, smem);
  const int tid = threadIdx.x, lane = tid % 32, wid = tid / 32;
  const int64_t P = param_floats(a);
  float* acc = s.tail;
  float* wbase = s.tail + pad4((int)P);
  const int wf = warp_floats(a, true);
  const Warp w = carve_warp(a, wbase + wid * wf);
  float* dh = w.extra;                                   // [kMaxH][kRows] d h of the layer below
  const int C = a.C, L = a.L, S = window_sum(a), nl = a.n_layers, Dq = a.Dq;
  const bool prelu = a.act == TZK_TDM_PRELU;
  const int64_t OC = (int64_t)(L + 1) * C;
  load_params(a, s);
  for (int64_t e = tid; e < P; e += blockDim.x) acc[e] = 0.f;
  __syncthreads();
  const int64_t G = gridDim.x, g = blockIdx.x;
  const int64_t b0 = a.B * g / G, b1 = a.B * (g + 1) / G;
  const int64_t r_begin = a.offsets[b0], r_end = a.offsets[b1];
  float q_acc = 0.f;                                     // thread c < C: column c of d query of sample `cur`
  int64_t cur = b0;
  const float slope_act = s.act_w[0];
  constexpr int kTile = kWarpsBwd * kRows;
  for (int64_t t0 = r_begin; t0 < r_end; t0 += kTile) {
    float* dq = dh + kMaxH * kRows;                     // [kRows][C] this warp's rows' d query shares
    float* rs = dq + kRows * C;                          // row scalars: d z, d act_w, d slope_l, sample
    int64_t rows[kRows], qb[kRows];
    int win[kRows];
    float cnt[kRows];
    bool any = false;
#pragma unroll
    for (int r = 0; r < kRows; ++r) {
      const int64_t t = t0 + wid * kRows + r;
      rows[r] = -1;
      qb[r] = -1;
      win[r] = 0;
      cnt[r] = 1.f;
      if (t < r_end) {
        int64_t lo = b0, hi = b1;                        // the sample of row t: offsets[lo] <= t < offsets[lo + 1]
        while (hi - lo > 1) {
          const int64_t mid = (lo + hi) / 2;
          if (a.offsets[mid] <= t) lo = mid; else hi = mid;
        }
        qb[r] = lo;
        const int64_t p = t - a.offsets[lo];
        if (p < S) {
          rows[r] = t;
          win[r] = s.win[p];
          int cum = 0;
          for (int wi = 0; wi < win[r]; ++wi) cum += a.windows[wi];
          const int64_t len = a.offsets[lo + 1] - a.offsets[lo], W = a.windows[win[r]];
          const int64_t m = len - cum < W ? len - cum : W;
          cnt[r] = (float)(m > 1 ? m : 1);
          any = true;
        } else {
          for (int c = 4 * lane; c < C; c += 128) st4(a.d_seq + t * C + c, make_float4(0.f, 0.f, 0.f, 0.f));
        }
      }
    }
#pragma unroll
    for (int r = 0; r < kRows; ++r)
      if (lane == r) reinterpret_cast<int*>(rs)[(2 + kMaxLayers) * kRows + r] = (int)(qb[r] - b0);
    if (any) {
      stage_x(a, w, rows, qb, lane);
      mlp_fwd(a, s, w, lane);
      // d z of every row: d a = sum_c g_c k_c, g = d_out[window] / cnt; the pooling's d k = a g
      float dz[kRows];
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        float da = 0.f, z = 0.f;
        if (rows[r] >= 0) {
          z = a.z[rows[r]];
          const float* go = a.d_out + qb[r] * OC + win[r] * C;
          for (int c = lane; c < C; c += 32) da += go[c] / cnt[r] * w.xs[c * kRows + r];
          da = warp_sum(da);
        }
        dz[r] = z > 0.f ? da : slope_act * da;
        if (lane == 0) {
          rs[r] = dz[r];
          rs[kRows + r] = z > 0.f ? 0.f : z * da;
        }
      }
      // d h of the last layer = d z lin_w, then layer by layer: d u = d h act'(u) (into u), d slope, d h below
      for (int j = lane; j < h_last(a); j += 32)
        st4(dh + j * kRows, make_float4(dz[0] * s.lin_w[j], dz[1] * s.lin_w[j], dz[2] * s.lin_w[j], dz[3] * s.lin_w[j]));
      __syncwarp();
      for (int l = nl - 1; l >= 0; --l) {
        const int H = a.hidden[l], Hs = pitch(a, l);
        const float sl = s.slope(a, l);
        float ds[kRows] = {0.f, 0.f, 0.f, 0.f};
        for (int j = lane; j < H; j += 32) {
          const float4 u = ld4(w.u(a, l) + j * kRows), d = ld4(dh + j * kRows);
          float4 du;
          du.x = u.x > 0.f ? d.x : sl * d.x;
          du.y = u.y > 0.f ? d.y : sl * d.y;
          du.z = u.z > 0.f ? d.z : sl * d.z;
          du.w = u.w > 0.f ? d.w : sl * d.w;
          ds[0] += u.x > 0.f ? 0.f : u.x * d.x;
          ds[1] += u.y > 0.f ? 0.f : u.y * d.y;
          ds[2] += u.z > 0.f ? 0.f : u.z * d.z;
          ds[3] += u.w > 0.f ? 0.f : u.w * d.w;
          st4(w.u(a, l) + j * kRows, du);
        }
        if (prelu) {
#pragma unroll
          for (int r = 0; r < kRows; ++r) {
            const float v = warp_sum(ds[r]);
            if (lane == 0) rs[(2 + l) * kRows + r] = v;
          }
        }
        __syncwarp();
        const float* wt = s.wt(a, l);
        if (l > 0) {
          const int K = a.hidden[l - 1];
          for (int i = lane; i < K; i += 32) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int j = 0; j < H; ++j) {
              const float wv = wt[i * Hs + j];
              const float4 du = ld4(w.u(a, l) + j * kRows);
              v.x += wv * du.x; v.y += wv * du.y; v.z += wv * du.z; v.w += wv * du.w;
            }
            st4(dh + i * kRows, v);
          }
          __syncwarp();
        } else {
          // d x = W1^T d u: column c gets d k (x block 0, and q times block 1) and its d query share (k times block
          // 1, plus block 2)
          for (int c = lane; c < C; c += 32) {
            float4 va = make_float4(0.f, 0.f, 0.f, 0.f), vb = va, vc = va;
            for (int j = 0; j < H; ++j) {
              const float4 du = ld4(w.u(a, 0) + j * kRows);
              const float wa = wt[c * Hs + j], wb = wt[(C + c) * Hs + j], wc = wt[(2 * C + c) * Hs + j];
              va.x += wa * du.x; va.y += wa * du.y; va.z += wa * du.z; va.w += wa * du.w;
              vb.x += wb * du.x; vb.y += wb * du.y; vb.z += wb * du.z; vb.w += wb * du.w;
              vc.x += wc * du.x; vc.y += wc * du.y; vc.z += wc * du.z; vc.w += wc * du.w;
            }
            const float dxa[kRows] = {va.x, va.y, va.z, va.w}, dxb[kRows] = {vb.x, vb.y, vb.z, vb.w},
                        dxc[kRows] = {vc.x, vc.y, vc.z, vc.w};
#pragma unroll
            for (int r = 0; r < kRows; ++r) {
              float share = 0.f;
              if (rows[r] >= 0) {
                const float k = w.xs[c * kRows + r], q = w.xs[(2 * C + c) * kRows + r];
                const float at = prelu1(a.z[rows[r]], slope_act);
                const float gc = a.d_out[qb[r] * OC + win[r] * C + c] / cnt[r];
                a.d_seq[rows[r] * C + c] = at * gc + dxa[r] + q * dxb[r];
                share = k * dxb[r] + dxc[r];
              }
              dq[r * C + c] = share;
            }
          }
        }
      }
    } else {
      for (int e = lane; e < kRows * C; e += 32) dq[e] = 0.f;
      for (int e = lane; e < layers_floats(a); e += 32) w.xs[e] = 0.f;
      if (lane < (2 + kMaxLayers) * kRows) rs[lane] = 0.f;
    }
    __syncthreads();
    // this tile's rows, in order (warp by warp, then row), into the CTA's parameter-gradient row
    int off = 0;
    for (int l = 0; l < nl; ++l) {
      const int K = in_dim(a, l), H = a.hidden[l], HK = H * K;
      const int n = HK + H + slope_n(a);
      const float* ul[kWarpsBwd];
      const float* xl[kWarpsBwd];
#pragma unroll
      for (int ww = 0; ww < kWarpsBwd; ++ww) {
        const Warp o = carve_warp(a, wbase + ww * wf);
        ul[ww] = o.u(a, l);
        xl[ww] = l == 0 ? o.xs : o.h(a, l - 1);
      }
      for (int e = tid; e < n; e += blockDim.x) {
        float v = acc[off + e];
        if (e < HK) {
          const int j = e / K, i = e - j * K;
#pragma unroll
          for (int ww = 0; ww < kWarpsBwd; ++ww) {
            const float4 du = ld4(ul[ww] + j * kRows), x = ld4(xl[ww] + i * kRows);
            v += du.x * x.x; v += du.y * x.y; v += du.z * x.z; v += du.w * x.w;
          }
        } else if (e < HK + H) {
#pragma unroll
          for (int ww = 0; ww < kWarpsBwd; ++ww) {
            const float4 du = ld4(ul[ww] + (e - HK) * kRows);
            v += du.x; v += du.y; v += du.z; v += du.w;
          }
        } else {
#pragma unroll
          for (int ww = 0; ww < kWarpsBwd; ++ww) {
            const float* ors = wbase + ww * wf + layers_floats(a) + kMaxH * kRows + kRows * C;
            for (int r = 0; r < kRows; ++r) v += ors[(2 + l) * kRows + r];
          }
        }
        acc[off + e] = v;
      }
      off += n;
    }
    {
      const int H = h_last(a);
      for (int e = tid; e < H + 2; e += blockDim.x) {
        float v = acc[off + e];
        for (int ww = 0; ww < kWarpsBwd; ++ww) {
          const Warp o = carve_warp(a, wbase + ww * wf);
          const float* ors = o.extra + kMaxH * kRows + kRows * C;
          for (int r = 0; r < kRows; ++r) {
            if (e < H) v += ors[r] * o.h(a, nl - 1)[e * kRows + r];
            else if (e == H) v += ors[r];
            else v += ors[kRows + r];
          }
        }
        acc[off + e] = v;
      }
    }
    if (tid < C) {                                       // column tid of d query, rows in order
      for (int ww = 0; ww < kWarpsBwd; ++ww) {
        const Warp o = carve_warp(a, wbase + ww * wf);
        const float* odq = o.extra + kMaxH * kRows;
        const int* osm = reinterpret_cast<const int*>(odq + kRows * C + (2 + kMaxLayers) * kRows);
        for (int r = 0; r < kRows; ++r) {
          if (t0 + ww * kRows + r >= r_end) break;
          const int64_t rb = b0 + osm[r];
          for (; cur < rb; ++cur) {
            if (tid < Dq) a.d_query[cur * Dq + tid] = a.d_out[cur * OC + L * C + tid] + q_acc;
            q_acc = 0.f;
          }
          q_acc += odq[r * C + tid];
        }
      }
    }
    __syncthreads();
  }
  if (tid < C) {
    for (; cur < b1; ++cur) {
      if (tid < Dq) a.d_query[cur * Dq + tid] = a.d_out[cur * OC + L * C + tid] + q_acc;
      q_acc = 0.f;
    }
  }
  for (int64_t e = tid; e < P; e += blockDim.x) partials[g * P + e] = acc[e];
}

// ---- launchers (return 0, or 1 on arguments outside the cover) --------------------------------------------------------
inline int fwd(const tzk_tdm_args& a, int grid, cudaStream_t stream) {
  if (check(a, false) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  const size_t smem = smem_bytes(a, false);
  tzk_batch_sum::opt_in_smem(fwd_kernel, smem);
  TZK_LAUNCH((fwd_kernel), grid, kWarpsFwd * 32, smem, stream, a);
  return 0;
}

// CTA g owns samples [B g / grid, B (g + 1) / grid); partials: grid * param_floats(a) floats; dparams:
// param_floats(a) floats
inline int bwd(const tzk_tdm_args& a, int grid, float* partials, float* dparams, cudaStream_t stream) {
  if (check(a, true) != 0 || grid < 1 || !partials || !dparams) return 1;
  if (a.B > 0) {
    const size_t smem = smem_bytes(a, true);
    tzk_batch_sum::opt_in_smem(bwd_kernel, smem);
    TZK_LAUNCH((bwd_kernel), grid, kWarpsBwd * 32, smem, stream, a, partials);
  }
  tzk_batch_sum::reduce(partials, a.B > 0 ? grid : 0, param_floats(a), 1, dparams, stream);
  return 0;
}
}  // namespace tzk_tdm
