// tzk_wukong.cuh — one WuKong layer's interaction (tzrec/modules/interaction.py:236-378) around its dense FMB MLP:
//
//   mix_fwd   per sample X [n, d]:  T = X^T W_fmb [d, k],  F = X T [n, k],  LN(F) over n*k with affine -> the FMB
//             MLP's input, per-sample (mean, rstd);  base [m = f + l, d] = residual (W_res^T X, or X when n == m) with
//             lcb = W_lcb^T X added to rows >= f — the reference's `concat(fmb, lcb) + res` for those rows.
//   out_fwd   per row r of [m, d]:  z = fmb_out + base (r < f) or base (r >= f);  LN(z) over d with affine, (mean, rstd).
//   out_bwd / mix_bwd: the exact gradients.  F and z are recomputed from X / (fmb_out, base), not stored.
//
// Weight, gamma and beta gradients are sums over the batch: every CTA accumulates its own samples (grid-stride, always
// the same samples for a given grid) in a fixed order into its row of a partials buffer, which tzk_batch_sum::reduce
// adds in CTA order (tzk_batch_sum.cuh).
//
// fp32 FFMA throughout (the reference runs fp32 with TF32 off).  Every product of the layer is a matrix of at most
// 64 x 32 x 64: too small for an MMA tile to pay for its fragment shuffles; see DESIGN.md (WuKong).
//
// Plain CUDA (no PTX): nvcc builds it in tzk_wukong.cu; g++ + tests/native/cuda_cpu_shim.h: tests/test_wukong_cpu.py
// runs this source on the host against a float64 restatement.
#pragma once
#include <math.h>
#include <stdint.h>

#include "tzk_batch_sum.cuh"
#include "tzk_launch.cuh"

namespace tzk_wukong {
constexpr int kThreads = 128;
constexpr float kEps = 1e-5f;                 // nn.LayerNorm's default eps, both norms of the layer

// shapes the kernels cover (the Python side's wukong_usable states the same)
inline bool usable(int n, int d, int k, int f, int l) {
  return n >= 1 && n <= 64 && (d == 4 || d == 8 || d == 16 || d == 32) && k >= 1 && k <= 32 && f >= 1 && l >= 1 &&
         f + l <= 64;
}

// floats of one CTA's row of weight-gradient partials: dW_fmb | dW_lcb | dW_res (projection only) | dgamma | dbeta
__host__ __device__ inline int64_t mix_params(int n, int k, int f, int l, bool proj) {
  return (int64_t)n * k * 3 + (int64_t)n * l + (proj ? (int64_t)n * (f + l) : 0);
}

constexpr int kWarps = kThreads / 32;

inline size_t mix_fwd_smem(int n, int d, int k, int f, int l, bool proj) {
  const int m = f + l;
  return sizeof(float) * ((size_t)n * k + (size_t)n * l + (proj ? (size_t)n * m : 0) + (size_t)n * d + (size_t)d * k +
                          (size_t)n * k + 2 * kWarps);
}

__global__ void __launch_bounds__(kThreads)
mix_fwd_kernel(const float* __restrict__ x, const float* __restrict__ wf, const float* __restrict__ gf,
               const float* __restrict__ bf, const float* __restrict__ wl, const float* __restrict__ wr, int64_t B,
               int n, int d, int k, int f, int l, float* __restrict__ ln_f, float* __restrict__ stats,
               float* __restrict__ base) {
  TZK_DYN_SMEM(float, sm);
  const int t = threadIdx.x, m = f + l, nk = n * k, nd = n * d, dk = d * k, md = m * d;
  const bool proj = wr != nullptr;
  float* s_wf = sm;
  float* s_wl = s_wf + nk;
  float* s_wr = s_wl + n * l;
  float* s_x = s_wr + (proj ? n * m : 0);
  float* s_t = s_x + nd;
  float* s_f = s_t + dk;
  float* s_red = s_f + nk;
  for (int e = t; e < nk; e += kThreads) s_wf[e] = wf[e];
  for (int e = t; e < n * l; e += kThreads) s_wl[e] = wl[e];
  if (proj)
    for (int e = t; e < n * m; e += kThreads) s_wr[e] = wr[e];
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    const float* xb = x + b * nd;
    for (int e = t; e < nd; e += kThreads) s_x[e] = xb[e];
    __syncthreads();
    for (int e = t; e < dk; e += kThreads) {          // T = X^T W_fmb
      const int j = e / k, c = e % k;
      float acc = 0.f;
      for (int i = 0; i < n; ++i) acc += s_x[i * d + j] * s_wf[i * k + c];
      s_t[e] = acc;
    }
    float* bb = base + b * md;
    for (int e = t; e < md; e += kThreads) {          // residual (+ lcb on rows >= f)
      const int r = e / d, j = e % d;
      float res;
      if (proj) {
        res = 0.f;
        for (int i = 0; i < n; ++i) res += s_wr[i * m + r] * s_x[i * d + j];
      } else {
        res = s_x[e];
      }
      if (r >= f) {
        float lcb = 0.f;
        for (int i = 0; i < n; ++i) lcb += s_wl[i * l + (r - f)] * s_x[i * d + j];
        res = lcb + res;
      }
      bb[e] = res;
    }
    __syncthreads();
    float part = 0.f;
    for (int e = t; e < nk; e += kThreads) {          // F = X T
      const int i = e / k, c = e % k;
      float acc = 0.f;
      for (int j = 0; j < d; ++j) acc += s_x[i * d + j] * s_t[j * k + c];
      s_f[e] = acc;
      part += acc;
    }
    float unused = 0.f;
    tzk_batch_sum::block_sum2<kWarps>(part, unused, s_red);
    const float mean = part / (float)nk;
    float sq = 0.f;
    for (int e = t; e < nk; e += kThreads) {
      const float c = s_f[e] - mean;
      sq += c * c;
    }
    tzk_batch_sum::block_sum2<kWarps>(sq, unused, s_red);
    const float rstd = 1.0f / sqrtf(sq / (float)nk + kEps);
    float* ob = ln_f + b * nk;
    for (int e = t; e < nk; e += kThreads) ob[e] = (s_f[e] - mean) * rstd * __ldg(gf + e) + __ldg(bf + e);
    if (t == 0) {
      stats[2 * b] = mean;
      stats[2 * b + 1] = rstd;
    }
  }
}

inline size_t mix_bwd_smem(int n, int d, int k, int f, int l, bool proj) {
  const int m = f + l;
  return sizeof(float) * ((size_t)n * k + (size_t)n * l + (proj ? (size_t)n * m : 0) + (size_t)n * d + 2 * (size_t)d * k +
                          2 * (size_t)n * k + (size_t)m * d + (size_t)mix_params(n, k, f, l, proj) + 2 * kWarps);
}

__global__ void __launch_bounds__(kThreads, 4)
mix_bwd_kernel(const float* __restrict__ x, const float* __restrict__ wf, const float* __restrict__ gf,
               const float* __restrict__ wl, const float* __restrict__ wr, const float* __restrict__ stats,
               const float* __restrict__ d_ln_f, const float* __restrict__ d_base, int64_t B, int n, int d, int k,
               int f, int l, float* __restrict__ dx, float* __restrict__ partials) {
  TZK_DYN_SMEM(float, sm);
  const int t = threadIdx.x, m = f + l, nk = n * k, nd = n * d, dk = d * k, md = m * d, nl = n * l, nm = n * m;
  const bool proj = wr != nullptr;
  const int P = (int)mix_params(n, k, f, l, proj);
  float* s_wf = sm;
  float* s_wl = s_wf + nk;
  float* s_wr = s_wl + nl;
  float* s_x = s_wr + (proj ? nm : 0);
  float* s_t = s_x + nd;
  float* s_dt = s_t + dk;
  float* s_f = s_dt + dk;     // xhat, then dF
  float* s_g = s_f + nk;      // d LN(F) * gamma
  float* s_db = s_g + nk;
  float* s_acc = s_db + md;   // this CTA's partials
  float* s_red = s_acc + P;
  float* a_wf = s_acc;
  float* a_wl = a_wf + nk;
  float* a_wr = a_wl + nl;
  float* a_g = a_wr + (proj ? nm : 0);
  float* a_b = a_g + nk;
  for (int e = t; e < nk; e += kThreads) s_wf[e] = wf[e];
  for (int e = t; e < nl; e += kThreads) s_wl[e] = wl[e];
  if (proj)
    for (int e = t; e < nm; e += kThreads) s_wr[e] = wr[e];
  for (int e = t; e < P; e += kThreads) s_acc[e] = 0.f;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    __syncthreads();
    for (int e = t; e < nd; e += kThreads) s_x[e] = x[b * nd + e];
    for (int e = t; e < md; e += kThreads) s_db[e] = d_base[b * md + e];
    __syncthreads();
    for (int e = t; e < dk; e += kThreads) {          // T = X^T W_fmb (recomputed)
      const int j = e / k, c = e % k;
      float acc = 0.f;
      for (int i = 0; i < n; ++i) acc += s_x[i * d + j] * s_wf[i * k + c];
      s_t[e] = acc;
    }
    __syncthreads();
    const float mean = stats[2 * b], rstd = stats[2 * b + 1];
    float sg = 0.f, sgx = 0.f;
    for (int e = t; e < nk; e += kThreads) {          // F (recomputed) -> xhat; LayerNorm(n*k) backward sums
      const int i = e / k, c = e % k;
      float acc = 0.f;
      for (int j = 0; j < d; ++j) acc += s_x[i * d + j] * s_t[j * k + c];
      const float xh = (acc - mean) * rstd, dy = d_ln_f[b * nk + e], g = dy * __ldg(gf + e);
      a_g[e] += dy * xh;
      a_b[e] += dy;
      s_f[e] = xh;
      s_g[e] = g;
      sg += g;
      sgx += g * xh;
    }
    tzk_batch_sum::block_sum2<kWarps>(sg, sgx, s_red);
    const float mg = sg / (float)nk, mgx = sgx / (float)nk;
    for (int e = t; e < nk; e += kThreads) s_f[e] = rstd * (s_g[e] - mg - s_f[e] * mgx);
    __syncthreads();
    for (int e = t; e < dk; e += kThreads) {          // dT = X^T dF
      const int j = e / k, c = e % k;
      float acc = 0.f;
      for (int i = 0; i < n; ++i) acc += s_x[i * d + j] * s_f[i * k + c];
      s_dt[e] = acc;
    }
    for (int e = t; e < nl; e += kThreads) {          // dW_lcb = X d_base[f:]^T
      const int i = e / l, r = e % l;
      float acc = 0.f;
      for (int j = 0; j < d; ++j) acc += s_x[i * d + j] * s_db[(f + r) * d + j];
      a_wl[e] += acc;
    }
    if (proj)
      for (int e = t; e < nm; e += kThreads) {        // dW_res = X d_base^T
        const int i = e / m, r = e % m;
        float acc = 0.f;
        for (int j = 0; j < d; ++j) acc += s_x[i * d + j] * s_db[r * d + j];
        a_wr[e] += acc;
      }
    __syncthreads();
    for (int e = t; e < nk; e += kThreads) {          // dW_fmb = X dT
      const int i = e / k, c = e % k;
      float acc = 0.f;
      for (int j = 0; j < d; ++j) acc += s_x[i * d + j] * s_dt[j * k + c];
      a_wf[e] += acc;
    }
    float* dxb = dx + b * nd;
    for (int e = t; e < nd; e += kThreads) {          // dX = dF T^T + W_fmb dT^T + W_lcb d_base[f:] + d residual
      const int i = e / d, j = e % d;
      float a1 = 0.f, a2 = 0.f;
      for (int c = 0; c < k; ++c) {
        a1 += s_f[i * k + c] * s_t[j * k + c];
        a2 += s_wf[i * k + c] * s_dt[j * k + c];
      }
      float a3 = 0.f;
      for (int r = 0; r < l; ++r) a3 += s_wl[i * l + r] * s_db[(f + r) * d + j];
      float a4;
      if (proj) {
        a4 = 0.f;
        for (int r = 0; r < m; ++r) a4 += s_wr[i * m + r] * s_db[r * d + j];
      } else {
        a4 = s_db[e];
      }
      dxb[e] = ((a1 + a2) + a3) + a4;
    }
  }
  __syncthreads();
  for (int e = t; e < P; e += kThreads) partials[(int64_t)blockIdx.x * P + e] = s_acc[e];
}

template <int D>
__global__ void __launch_bounds__(kThreads)
out_fwd_kernel(const float* __restrict__ fmb, const float* __restrict__ base, const float* __restrict__ gamma,
               const float* __restrict__ beta, int64_t R, int f, int m, float* __restrict__ y,
               float* __restrict__ stats) {
  for (int64_t row = (int64_t)blockIdx.x * kThreads + threadIdx.x; row < R; row += (int64_t)gridDim.x * kThreads) {
    const int64_t b = row / m;
    const int r = (int)(row % m);
    float z[D];
    for (int j = 0; j < D; ++j) z[j] = base[row * D + j];
    if (r < f)
      for (int j = 0; j < D; ++j) z[j] = fmb[(b * f + r) * D + j] + z[j];
    float s = 0.f;
    for (int j = 0; j < D; ++j) s += z[j];
    const float mean = s / (float)D;
    float sq = 0.f;
    for (int j = 0; j < D; ++j) sq += (z[j] - mean) * (z[j] - mean);
    const float rstd = 1.0f / sqrtf(sq / (float)D + kEps);
    for (int j = 0; j < D; ++j) y[row * D + j] = (z[j] - mean) * rstd * __ldg(gamma + j) + __ldg(beta + j);
    stats[2 * row] = mean;
    stats[2 * row + 1] = rstd;
  }
}

template <int D>
__global__ void __launch_bounds__(kThreads)
out_bwd_kernel(const float* __restrict__ fmb, const float* __restrict__ base, const float* __restrict__ gamma,
               const float* __restrict__ stats, const float* __restrict__ dy, int64_t R, int f, int m,
               float* __restrict__ d_fmb, float* __restrict__ d_base, float* __restrict__ partials) {
  __shared__ float s_part[kThreads * 2 * D];
  float ag[D], ab[D];
  for (int j = 0; j < D; ++j) ag[j] = ab[j] = 0.f;
  for (int64_t row = (int64_t)blockIdx.x * kThreads + threadIdx.x; row < R; row += (int64_t)gridDim.x * kThreads) {
    const int64_t b = row / m;
    const int r = (int)(row % m);
    const float mean = stats[2 * row], rstd = stats[2 * row + 1];
    float xh[D], g[D];
    float sg = 0.f, sgx = 0.f;
    for (int j = 0; j < D; ++j) {
      float z = base[row * D + j];
      if (r < f) z = fmb[(b * f + r) * D + j] + z;
      xh[j] = (z - mean) * rstd;
      const float dv = dy[row * D + j];
      g[j] = dv * __ldg(gamma + j);
      ag[j] += dv * xh[j];
      ab[j] += dv;
      sg += g[j];
      sgx += g[j] * xh[j];
    }
    const float mg = sg / (float)D, mgx = sgx / (float)D;
    for (int j = 0; j < D; ++j) {
      const float dz = rstd * (g[j] - mg - xh[j] * mgx);
      d_base[row * D + j] = dz;
      if (r < f) d_fmb[(b * f + r) * D + j] = dz;
    }
  }
  for (int j = 0; j < D; ++j) {
    s_part[threadIdx.x * 2 * D + j] = ag[j];
    s_part[threadIdx.x * 2 * D + D + j] = ab[j];
  }
  __syncthreads();
  if (threadIdx.x < 2 * D) {
    float acc = 0.f;
    for (int q = 0; q < kThreads; ++q) acc += s_part[q * 2 * D + threadIdx.x];
    partials[(int64_t)blockIdx.x * 2 * D + threadIdx.x] = acc;
  }
}

// ---- launchers (return 0, or 1 on unsupported arguments) -------------------------------------------------------------
inline int mix_fwd(const float* x, const float* wf, const float* gf, const float* bf, const float* wl, const float* wr,
                   int64_t B, int n, int d, int k, int f, int l, int grid, float* ln_f, float* stats, float* base,
                   cudaStream_t stream) {
  if (!usable(n, d, k, f, l) || grid < 1) return 1;
  if (B == 0) return 0;
  const size_t smem = mix_fwd_smem(n, d, k, f, l, wr != nullptr);
  tzk_batch_sum::opt_in_smem(mix_fwd_kernel, smem);
  TZK_LAUNCH((mix_fwd_kernel), grid, kThreads, smem, stream, x, wf, gf, bf, wl, wr, B, n, d, k, f, l, ln_f, stats,
             base);
  return 0;
}

// partials: grid * mix_params(...) floats; dparams: mix_params(...) floats (dW_fmb | dW_lcb | dW_res | dgamma | dbeta)
inline int mix_bwd(const float* x, const float* wf, const float* gf, const float* wl, const float* wr,
                   const float* stats, const float* d_ln_f, const float* d_base, int64_t B, int n, int d, int k, int f,
                   int l, int grid, float* dx, float* partials, float* dparams, cudaStream_t stream) {
  if (!usable(n, d, k, f, l) || grid < 1) return 1;
  if (B > 0) {
    const size_t smem = mix_bwd_smem(n, d, k, f, l, wr != nullptr);
    tzk_batch_sum::opt_in_smem(mix_bwd_kernel, smem);
    TZK_LAUNCH((mix_bwd_kernel), grid, kThreads, smem, stream, x, wf, gf, wl, wr, stats, d_ln_f, d_base, B, n, d, k,
               f, l, dx, partials);
  }
  tzk_batch_sum::reduce(partials, B > 0 ? grid : 0, mix_params(n, k, f, l, wr != nullptr), 1, dparams, stream);
  return 0;
}

inline int out_fwd(const float* fmb, const float* base, const float* gamma, const float* beta, int64_t B, int d, int f,
                   int l, int grid, float* y, float* stats, cudaStream_t stream) {
  if (!(d == 4 || d == 8 || d == 16 || d == 32) || f < 1 || l < 1 || grid < 1) return 1;
  const int64_t R = B * (f + l);
  if (R == 0) return 0;
  const int m = f + l;
  switch (d) {
    case 4: TZK_LAUNCH((out_fwd_kernel<4>), grid, kThreads, 0, stream, fmb, base, gamma, beta, R, f, m, y, stats); break;
    case 8: TZK_LAUNCH((out_fwd_kernel<8>), grid, kThreads, 0, stream, fmb, base, gamma, beta, R, f, m, y, stats); break;
    case 16: TZK_LAUNCH((out_fwd_kernel<16>), grid, kThreads, 0, stream, fmb, base, gamma, beta, R, f, m, y, stats); break;
    default: TZK_LAUNCH((out_fwd_kernel<32>), grid, kThreads, 0, stream, fmb, base, gamma, beta, R, f, m, y, stats); break;
  }
  return 0;
}

// partials: grid * 2 d floats; dparams: 2 d floats (dgamma | dbeta)
inline int out_bwd(const float* fmb, const float* base, const float* gamma, const float* stats, const float* dy,
                   int64_t B, int d, int f, int l, int grid, float* d_fmb, float* d_base, float* partials,
                   float* dparams, cudaStream_t stream) {
  if (!(d == 4 || d == 8 || d == 16 || d == 32) || f < 1 || l < 1 || grid < 1) return 1;
  const int64_t R = B * (f + l);
  const int m = f + l;
  if (R > 0) {
    switch (d) {
      case 4: TZK_LAUNCH((out_bwd_kernel<4>), grid, kThreads, 0, stream, fmb, base, gamma, stats, dy, R, f, m, d_fmb, d_base, partials); break;
      case 8: TZK_LAUNCH((out_bwd_kernel<8>), grid, kThreads, 0, stream, fmb, base, gamma, stats, dy, R, f, m, d_fmb, d_base, partials); break;
      case 16: TZK_LAUNCH((out_bwd_kernel<16>), grid, kThreads, 0, stream, fmb, base, gamma, stats, dy, R, f, m, d_fmb, d_base, partials); break;
      default: TZK_LAUNCH((out_bwd_kernel<32>), grid, kThreads, 0, stream, fmb, base, gamma, stats, dy, R, f, m, d_fmb, d_base, partials); break;
    }
  }
  tzk_batch_sum::reduce(partials, R > 0 ? grid : 0, 2 * d, 1, dparams, stream);
  return 0;
}
}  // namespace tzk_wukong
