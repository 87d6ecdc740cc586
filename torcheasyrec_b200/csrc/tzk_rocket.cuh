// tzk_rocket.cuh — RocketLaunching's booster / light head (tzrec/models/rocket_launching.py): everything after the
// two MLPs, per sample, for the light head and optionally the booster head.
//
//   head_fwd  z_e = h_e W_e^T + b_e, p_e = softmax(z_e) for both heads (e = 0 light, 1 booster); with labels the
//             per-sample terms of the losses: the label-smoothed cross-entropy of each head, the hint term
//             sum_c (z_light - z_booster)^2 and, per similarity pair (light l, booster b, both [B, d]):
//               COSINE  <b, l> / (max(|b|, 1e-12) max(|l|, 1e-12))   (F.normalize twice, then the row sum)
//               EUCLID  sum_d (b - l)^2
//             One warp per sample: every dot product is a fixed xor butterfly, so each lane holds the same bits.
//             The CTA's per-sample terms are added warp by warp in order into one partials row; finish_kernel adds
//             the rows in CTA order and applies the means (CE / B, hint / (B C), cosine -0.1 / B) and EUCLID's sqrt.
//   head_bwd  the gradients of those losses for the upstream gradients dlosses (a device array): d logits from the
//             saved probs and logits, then dh = dz W, dlight of every pair and the CTA's dW / db rows in a shared
//             memory accumulator.  The CTA walks tiles of kTile samples; each thread owns fixed accumulator entries
//             and adds the tile's samples in order.  tzk_batch_sum::reduce adds the CTA rows in CTA order.
//
// The backward of COSINE follows torch's autograd of F.normalize: with cl = max(|l|, eps), cb = max(|b|, eps),
//   d sim / d l = b / (cb cl) - [|l| >= eps] <b, l> / (cb cl^2 |l|) l
// so an all-zero light row gets b / (cb eps), as torch gives at the clamp.  pair_stats keeps the two coefficients.
// EUCLID's gradient is (l - b) / loss, NaN at loss 0 as torch's (0 times infinity).
//
// fp32 throughout.  Plain CUDA (no PTX): nvcc builds it in tzk_rocket.cu; g++ + tests/native/cuda_cpu_shim.h:
// tests/test_rocket_cpu.py runs this source on the host against float64.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/tzk.h"
#include "tzk_batch_sum.cuh"
#include "tzk_launch.cuh"

namespace tzk_rocket {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxC = TZK_ROCKET_MAX_CLASSES;
constexpr int kMaxPairs = TZK_ROCKET_MAX_PAIRS;
constexpr int kMaxWidth = 1024;
constexpr int kMaxLoss = 3 + kMaxPairs;      // CE light, CE booster, hint, one per pair
constexpr int kTile = 32;                    // samples per backward step
constexpr float kNormEps = 1e-12f;           // F.normalize's eps
constexpr size_t kBwdStaticSmem = 2 * kTile * kMaxC * sizeof(float);   // head_bwd_kernel's s_dz

__host__ __device__ inline int n_losses(const tzk_rocket_args& a) { return 3 + a.n_pairs; }
__host__ __device__ inline int n_heads(const tzk_rocket_args& a) { return a.has_booster ? 2 : 1; }
inline bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }
inline bool width_ok(int w) { return w >= 4 && w <= kMaxWidth && w % 4 == 0; }

// floats of one backward partials row (and of dparams): dW_light [C, H_l] | db_light [C] | dW_booster | db_booster
inline int64_t param_floats(const tzk_rocket_args& a) {
  int64_t P = 0;
  for (int e = 0; e < n_heads(a); ++e) P += (int64_t)a.C * (a.head[e].H + 1);
  return P;
}

// the descriptions the kernels cover (the Python side's rocket_head_usable states the same for whole models)
inline int check(const tzk_rocket_args& a, bool backward) {
  if (a.B < 0 || a.B >= ((int64_t)1 << 31) || a.C < 2 || a.C > kMaxC) return 1;
  if ((a.has_booster != 0 && a.has_booster != 1) || a.n_pairs < 0 || a.n_pairs > kMaxPairs) return 1;
  if (a.sim != TZK_ROCKET_COSINE && a.sim != TZK_ROCKET_EUCLID) return 1;
  if (!(a.eps >= 0.f && a.eps <= 1.f)) return 1;
  if (a.n_pairs > 0 && !a.has_booster) return 1;
  const bool live = a.B > 0;
  if (backward && live && !a.labels) return 1;
  for (int e = 0; e < n_heads(a); ++e) {
    const tzk_rocket_head& h = a.head[e];
    if (!width_ok(h.H) || !aligned16(h.h) || !aligned16(h.w)) return 1;
    if (live && (!h.h || !h.w || !h.b || !h.logits || !h.probs)) return 1;
    if (backward && live && !h.dh) return 1;
  }
  if (live && a.labels == nullptr && a.n_pairs > 0) return 1;
  for (int k = 0; k < a.n_pairs; ++k) {
    const tzk_rocket_pair& p = a.pair[k];
    if (!width_ok(p.d) || !aligned16(p.light) || !aligned16(p.booster)) return 1;
    if (live && (!p.light || !p.booster)) return 1;
    if (backward && live && !p.dlight) return 1;
  }
  if (live && a.n_pairs > 0 && a.sim == TZK_ROCKET_COSINE && !a.pair_stats) return 1;
  return 0;
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ float dot4(const float4& x, const float4& y) {
  return x.x * y.x + x.y * y.y + x.z * y.z + x.w * y.w;
}
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// One warp per sample.  partials [gridDim.x][n_losses] when labels are given.
__global__ void __launch_bounds__(kThreads) head_fwd_kernel(const __grid_constant__ tzk_rocket_args a,
                                                            float* __restrict__ partials) {
  __shared__ float s_acc[kWarps][kMaxLoss];
  const int lane = threadIdx.x % 32, w = threadIdx.x / 32;
  const int C = a.C, nh = n_heads(a), NL = n_losses(a);
  const bool with_loss = a.labels != nullptr;
  float acc[kMaxLoss];
#pragma unroll
  for (int j = 0; j < kMaxLoss; ++j) acc[j] = 0.f;
  for (int64_t b = (int64_t)blockIdx.x * kWarps + w; b < a.B; b += (int64_t)gridDim.x * kWarps) {
    float z[2][kMaxC];
    int y = 0;
    if (with_loss) {
      const float lab = a.labels[b];
      y = (lab >= 0.f && lab < (float)C) ? (int)lab : -1;
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      if (e >= nh) break;
      const tzk_rocket_head& hd = a.head[e];
      const int H = hd.H;
      float s[kMaxC];
#pragma unroll
      for (int c = 0; c < kMaxC; ++c) s[c] = 0.f;
      const float* hr = hd.h + b * H;
      for (int j = 4 * lane; j < H; j += 128) {
        const float4 x = ld4(hr + j);
#pragma unroll
        for (int c = 0; c < kMaxC; ++c)
          if (c < C) s[c] += dot4(x, ld4(hd.w + (int64_t)c * H + j));
      }
      float m = -INFINITY;
#pragma unroll
      for (int c = 0; c < kMaxC; ++c) {
        if (c < C) {
          s[c] = warp_sum(s[c]) + hd.b[c];
          m = fmaxf(m, s[c]);
        }
        z[e][c] = s[c];
      }
      float sum = 0.f;
#pragma unroll
      for (int c = 0; c < kMaxC; ++c)
        if (c < C) sum += expf(s[c] - m);
#pragma unroll
      for (int c = 0; c < kMaxC; ++c)
        if (c < C && lane == c) {
          hd.logits[b * C + c] = s[c];
          hd.probs[b * C + c] = expf(s[c] - m) / sum;
        }
      if (with_loss) {
        // -sum_c q_c log p_c = lse - (1 - eps) z_y - eps / C sum_c z_c
        const float lse = m + logf(sum);
        float zy = 0.f, zs = 0.f;
#pragma unroll
        for (int c = 0; c < kMaxC; ++c)
          if (c < C) {
            zs += s[c];
            if (c == y) zy = s[c];
          }
        acc[e] += (y < 0) ? NAN : lse - (1.f - a.eps) * zy - a.eps / (float)C * zs;
      }
    }
    if (!with_loss || !a.has_booster) continue;
    float hint = 0.f;
#pragma unroll
    for (int c = 0; c < kMaxC; ++c)
      if (c < C) hint += (z[0][c] - z[1][c]) * (z[0][c] - z[1][c]);
    acc[2] += hint;
#pragma unroll
    for (int k = 0; k < kMaxPairs; ++k) {
      if (k >= a.n_pairs) break;
      const tzk_rocket_pair& pr = a.pair[k];
      const int d = pr.d;
      const float* lr = pr.light + b * d;
      const float* br = pr.booster + b * d;
      float ll = 0.f, bb = 0.f, lb = 0.f;
      for (int j = 4 * lane; j < d; j += 128) {
        const float4 l = ld4(lr + j), o = ld4(br + j);
        if (a.sim == TZK_ROCKET_COSINE) {
          ll += dot4(l, l);
          bb += dot4(o, o);
          lb += dot4(l, o);
        } else {
          const float4 df = make_float4(o.x - l.x, o.y - l.y, o.z - l.z, o.w - l.w);
          lb += dot4(df, df);
        }
      }
      lb = warp_sum(lb);
      if (a.sim == TZK_ROCKET_COSINE) {
        ll = warp_sum(ll);
        bb = warp_sum(bb);
        const float nl = sqrtf(ll), cl = fmaxf(nl, kNormEps), cb = fmaxf(sqrtf(bb), kNormEps);
        acc[3 + k] += lb / (cb * cl);
        if (lane == 0) {
          float* st = a.pair_stats + ((int64_t)k * a.B + b) * 2;
          st[0] = 1.f / (cb * cl);
          st[1] = nl >= kNormEps ? lb / (cb * cl * cl * nl) : 0.f;
        }
      } else {
        acc[3 + k] += lb;
      }
    }
  }
  if (!with_loss) return;
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < kMaxLoss; ++j) s_acc[w][j] = acc[j];
  }
  __syncthreads();
  if ((int)threadIdx.x < NL) {
    float t = 0.f;
    for (int i = 0; i < kWarps; ++i) t += s_acc[i][threadIdx.x];
    partials[(int64_t)blockIdx.x * NL + threadIdx.x] = t;
  }
}

// losses[j] = the CTA-order sum of partials column j, then the loss's mean / sqrt.  G = 0 (an empty batch): the means
// are 0 / 0 = NaN, as torch's mean over no samples.  One CTA of 32 threads.
__global__ void __launch_bounds__(32) finish_kernel(const __grid_constant__ tzk_rocket_args a,
                                                    const float* __restrict__ partials, int G,
                                                    float* __restrict__ losses) {
  const int j = threadIdx.x, NL = n_losses(a);
  if (j >= NL) return;
  float s = 0.f;
  for (int g = 0; g < G; ++g) s += partials[(int64_t)g * NL + j];
  const float B = (float)a.B;
  float v;
  if (j < 2) {
    v = (j == 1 && !a.has_booster) ? 0.f : s / B;
  } else if (j == 2) {
    v = a.has_booster ? s / (B * (float)a.C) : 0.f;
  } else {
    v = a.sim == TZK_ROCKET_COSINE ? -0.1f * (s / B) : sqrtf(s);
  }
  losses[j] = v;
}

// dynamic shared memory: param_floats(a) accumulator floats
__global__ void __launch_bounds__(kThreads) head_bwd_kernel(const __grid_constant__ tzk_rocket_args a,
                                                            const float* __restrict__ dlosses,
                                                            const float* __restrict__ losses,
                                                            float* __restrict__ partials, int64_t P) {
  TZK_DYN_SMEM(float, s_acc);
  __shared__ float s_dz[2][kTile][kMaxC];
  static_assert(sizeof(s_dz) == kBwdStaticSmem, "kBwdStaticSmem is the size of s_dz");
  const int tid = threadIdx.x;
  const int C = a.C, nh = n_heads(a);
  const float B = (float)a.B;
  for (int64_t i = tid; i < P; i += kThreads) s_acc[i] = 0.f;
  // the upstream gradient of each loss, scaled as the loss's mean is
  const float g_ce0 = dlosses[0] / B, g_ce1 = a.has_booster ? dlosses[1] / B : 0.f;
  const float g_hint = a.has_booster ? dlosses[2] * (2.f / (B * (float)C)) : 0.f;
  for (int64_t t0 = (int64_t)blockIdx.x * kTile; t0 < a.B; t0 += (int64_t)gridDim.x * kTile) {
    const int nt = (int)((a.B - t0) < kTile ? (a.B - t0) : kTile);
    if (tid < nt) {                               // d logits of sample t0 + tid
      const int64_t b = t0 + tid;
      const float lab = a.labels[b];
      const int y = (lab >= 0.f && lab < (float)C) ? (int)lab : -1;
      for (int e = 0; e < nh; ++e) {
        const float* p = a.head[e].probs + b * C;
        for (int c = 0; c < C; ++c) {
          const float q = (c == y ? 1.f - a.eps : 0.f) + a.eps / (float)C;
          float dz = (y < 0) ? NAN : (e == 0 ? g_ce0 : g_ce1) * (p[c] - q);
          if (e == 0 && a.has_booster)
            dz += g_hint * (a.head[0].logits[b * C + c] - a.head[1].logits[b * C + c]);
          s_dz[e][tid][c] = dz;
        }
      }
    }
    __syncthreads();
    for (int e = 0; e < nh; ++e) {                // dh = dz W
      const tzk_rocket_head& hd = a.head[e];
      const int H = hd.H;
      for (int i = tid; i < nt * H; i += kThreads) {
        const int t = i / H, h = i % H;
        float v = 0.f;
        for (int c = 0; c < C; ++c) v += s_dz[e][t][c] * hd.w[(int64_t)c * H + h];
        hd.dh[(t0 + t) * H + h] = v;
      }
    }
    for (int k = 0; k < a.n_pairs; ++k) {         // d light of every pair
      const tzk_rocket_pair& pr = a.pair[k];
      const int d = pr.d;
      const float g = dlosses[3 + k];
      const float s_cos = g * -0.1f / B, s_euc = g / losses[3 + k];
      for (int i = tid; i < nt * d; i += kThreads) {
        const int64_t b = t0 + i / d;
        const int64_t o = b * d + i % d;
        const float l = pr.light[o], bo = pr.booster[o];
        float dl;
        if (a.sim == TZK_ROCKET_COSINE) {
          const float* st = a.pair_stats + ((int64_t)k * a.B + b) * 2;
          dl = s_cos * (st[0] * bo - st[1] * l);
        } else {
          dl = s_euc * (l - bo);
        }
        pr.dlight[o] = dl;
      }
    }
    int64_t off = 0;                              // this CTA's dW / db: each thread its own entries, samples in order
    for (int e = 0; e < nh; ++e) {
      const tzk_rocket_head& hd = a.head[e];
      const int H = hd.H;
      const int64_t n = (int64_t)C * (H + 1);
      for (int64_t i = tid; i < n; i += kThreads) {
        float v = s_acc[off + i];
        if (i < (int64_t)C * H) {
          const int c = (int)(i / H), h = (int)(i % H);
          for (int t = 0; t < nt; ++t) v += s_dz[e][t][c] * hd.h[(t0 + t) * H + h];
        } else {
          const int c = (int)(i - (int64_t)C * H);
          for (int t = 0; t < nt; ++t) v += s_dz[e][t][c];
        }
        s_acc[off + i] = v;
      }
      off += n;
    }
    __syncthreads();
  }
  for (int64_t i = tid; i < P; i += kThreads) partials[(int64_t)blockIdx.x * P + i] = s_acc[i];
}

inline size_t bwd_smem_bytes(const tzk_rocket_args& a) { return (size_t)param_floats(a) * sizeof(float); }

// ---- launchers (return 0, or 1 on arguments outside the cover) --------------------------------------------------------
// partials: grid * n_losses(a) floats; losses: n_losses(a) floats, or NULL for no losses (then labels is NULL too)
inline int head_fwd(const tzk_rocket_args& a, int grid, float* partials, float* losses, cudaStream_t stream) {
  if (check(a, false) != 0 || grid < 1) return 1;
  if ((a.labels != nullptr) != (losses != nullptr) && a.B > 0) return 1;
  if (losses && !partials) return 1;
  if (a.B > 0) TZK_LAUNCH((head_fwd_kernel), grid, kThreads, 0, stream, a, partials);
  if (losses) TZK_LAUNCH((finish_kernel), 1, 32, 0, stream, a, partials, a.B > 0 ? grid : 0, losses);
  return 0;
}

// partials: grid * param_floats(a) floats; dparams: param_floats(a) floats
inline int head_bwd(const tzk_rocket_args& a, const float* dlosses, const float* losses, int grid, float* partials,
                    float* dparams, cudaStream_t stream) {
  if (check(a, true) != 0 || grid < 1 || !dlosses || !losses || !partials || !dparams) return 1;
  const int64_t P = param_floats(a);
  if (a.B > 0) {
    const size_t smem = bwd_smem_bytes(a);
    // static + dynamic above 48 KB needs the opt-in, so a dynamic size just under 48 KB does too
    tzk_batch_sum::opt_in_smem(head_bwd_kernel, smem + kBwdStaticSmem);
    TZK_LAUNCH((head_bwd_kernel), grid, kThreads, smem, stream, a, dlosses, losses, partials, P);
  }
  tzk_batch_sum::reduce(partials, a.B > 0 ? grid : 0, P, 1, dparams, stream);
  return 0;
}
}  // namespace tzk_rocket
