// tzk_masknet.cuh — the element-wise stages of MaskNet's parallel mask blocks (tzrec/modules/masknet.py:77-85 and
// 142-155) around its GEMMs, for nb blocks of input width E (padded to a row pitch Ep, a multiple of 4) and FFN width H:
//
//   mask_fwd  per sample e [E]:  LN(e) over E with affine (ln_emb), per-sample (mean, rstd);  for every block i
//             v_i = LN(e) * (m_i + b2_i), m_i [Ep] the mask generator's second GEMM without its bias.  LN(e) and the
//             biased mask are never stored.  Pad columns [E, Ep) of v are written as 0.
//   mask_bwd  dv [B, nb Ep] -> dm_i = dv_i * LN(e), de_ln = LayerNorm-backward of sum_i dv_i * (m_i + b2_i), and the
//             batch sums db2_i = sum dm_i, dgamma_ln, dbeta_ln.  LN(e) is recomputed from e and the saved (mean, rstd).
//   ffn_fwd   per (sample, block):  y = ReLU(LN_H(z_i + b3_i) with affine), written into the block's column slot of
//             hidden [B, nb H] (the reference's concat), (mean, rstd) saved.
//   ffn_bwd   the exact gradient: ReLU mask (y > 0), LayerNorm backward into dz_i, batch sums dgamma_i, dbeta_i, db3_i.
//
// One CTA of 128 threads per row (grid-stride over rows); thread t owns columns t + 128 j, so every per-column batch
// sum is accumulated by one thread in a fixed order (registers, or shared memory for the nb-dependent db2), written as
// the CTA's row of a partials buffer, and reduce_kernel adds the rows in CTA order.  No float atomics: the result
// depends only on the grid, which the host derives from B and the SM count, so a replayed graph gives the eager bits.
//
// fp32 FFMA throughout.  Plain CUDA (no PTX): the includer provides TZK_DYN_SMEM / TZK_LAUNCH (nvcc: tzk_masknet.cu;
// g++ + tests/native/cuda_cpu_shim.h: tests/test_masknet_cpu.py runs this source on the host against a float64
// restatement).
#pragma once
#include <math.h>
#include <stdint.h>

namespace tzk_masknet {
constexpr int kThreads = 128;
constexpr int kWarps = kThreads / 32;
constexpr int kVpt = 8;                       // columns per thread: widths up to kThreads * kVpt
constexpr int kMaxWidth = kThreads * kVpt;    // 1024
constexpr int kMaxBlocks = 8;
constexpr float kEps = 1e-5f;                 // nn.LayerNorm's default eps, both norms of the module

inline int pad4(int n) { return (n + 3) / 4 * 4; }

// shapes the kernels cover (the Python side's masknet_usable states the same)
inline bool usable(int E, int H, int nb) {
  return E >= 1 && pad4(E) <= kMaxWidth && H >= 4 && H <= kMaxWidth && H % 4 == 0 && nb >= 1 && nb <= kMaxBlocks;
}

// sums over the CTA in a fixed order (xor butterfly in each warp, then the warps in order); every thread gets both
// totals.  Two barriers.
__device__ __forceinline__ void block_sum2(float& a, float& b, float* s_red) {
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int w = threadIdx.x / 32;
  if (threadIdx.x % 32 == 0) {
    s_red[w] = a;
    s_red[kWarps + w] = b;
  }
  __syncthreads();
  a = s_red[0];
  b = s_red[kWarps];
  for (int i = 1; i < kWarps; ++i) {
    a += s_red[i];
    b += s_red[kWarps + i];
  }
  __syncthreads();
}

// e [B, lde] (first E columns), m [B, nb Ep], b2 [nb E], gamma / beta [E] -> v [B, nb Ep], stats [B, 2]
__global__ void __launch_bounds__(kThreads)
mask_fwd_kernel(const float* __restrict__ e, int lde, const float* __restrict__ m, const float* __restrict__ b2,
                const float* __restrict__ gamma, const float* __restrict__ beta, int64_t B, int E, int Ep, int nb,
                float* __restrict__ v, float* __restrict__ stats) {
  __shared__ float s_red[2 * kWarps];
  const int t = threadIdx.x;
  const int64_t ldm = (int64_t)nb * Ep;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    float x[kVpt];
    float s = 0.f, unused = 0.f;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      x[j] = c < E ? e[b * lde + c] : 0.f;
      s += x[j];
    }
    block_sum2(s, unused, s_red);
    const float mean = s / (float)E;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      const float d = x[j] - mean;
      if (c < E) sq += d * d;
    }
    block_sum2(sq, unused, s_red);
    const float rstd = 1.0f / sqrtf(sq / (float)E + kEps);
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      if (c < E) x[j] = (x[j] - mean) * rstd * __ldg(gamma + c) + __ldg(beta + c);
    }
    for (int i = 0; i < nb; ++i) {
      const float* mi = m + b * ldm + (int64_t)i * Ep;
      float* vi = v + b * ldm + (int64_t)i * Ep;
#pragma unroll
      for (int j = 0; j < kVpt; ++j) {
        const int c = t + j * kThreads;
        if (c < E) vi[c] = x[j] * (mi[c] + __ldg(b2 + i * E + c));
        else if (c < Ep) vi[c] = 0.f;
      }
    }
    if (t == 0) {
      stats[2 * b] = mean;
      stats[2 * b + 1] = rstd;
    }
  }
}

// -> dm [B, nb Ep], de [B, Ep] (pad columns 0), partials row per CTA: db2 [nb E] | dgamma [E] | dbeta [E]
__global__ void __launch_bounds__(kThreads)
mask_bwd_kernel(const float* __restrict__ e, int lde, const float* __restrict__ m, const float* __restrict__ b2,
                const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ stats,
                const float* __restrict__ dv, int64_t B, int E, int Ep, int nb, float* __restrict__ dm,
                float* __restrict__ de, float* __restrict__ partials) {
  TZK_DYN_SMEM(float, s_db2);               // [nb][Ep]: column c of every block is thread (c % kThreads)'s alone
  __shared__ float s_red[2 * kWarps];
  const int t = threadIdx.x;
  const int64_t ldm = (int64_t)nb * Ep;
  for (int i = 0; i < nb; ++i)
    for (int c = t; c < E; c += kThreads) s_db2[i * Ep + c] = 0.f;
  float ag[kVpt], ab[kVpt];
#pragma unroll
  for (int j = 0; j < kVpt; ++j) ag[j] = ab[j] = 0.f;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    const float mean = stats[2 * b], rstd = stats[2 * b + 1];
    float xh[kVpt], ln[kVpt], g[kVpt];
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      xh[j] = c < E ? (e[b * lde + c] - mean) * rstd : 0.f;
      ln[j] = c < E ? xh[j] * __ldg(gamma + c) + __ldg(beta + c) : 0.f;
      g[j] = 0.f;
    }
    for (int i = 0; i < nb; ++i) {
      const float* mi = m + b * ldm + (int64_t)i * Ep;
      const float* dvi = dv + b * ldm + (int64_t)i * Ep;
      float* dmi = dm + b * ldm + (int64_t)i * Ep;
#pragma unroll
      for (int j = 0; j < kVpt; ++j) {
        const int c = t + j * kThreads;
        if (c < E) {
          const float d = dvi[c];
          const float dmask = d * ln[j];
          dmi[c] = dmask;
          s_db2[i * Ep + c] += dmask;
          g[j] += d * (mi[c] + __ldg(b2 + i * E + c));
        } else if (c < Ep) {
          dmi[c] = 0.f;
        }
      }
    }
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      ag[j] += g[j] * xh[j];
      ab[j] += g[j];
      g[j] = c < E ? g[j] * __ldg(gamma + c) : 0.f;
      sg += g[j];
      sgx += g[j] * xh[j];
    }
    block_sum2(sg, sgx, s_red);
    const float mg = sg / (float)E, mgx = sgx / (float)E;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      if (c < E) de[b * Ep + c] = rstd * (g[j] - mg - xh[j] * mgx);
      else if (c < Ep) de[b * Ep + c] = 0.f;
    }
  }
  const int64_t P = (int64_t)(nb + 2) * E;
  float* out = partials + (int64_t)blockIdx.x * P;
  for (int i = 0; i < nb; ++i)
    for (int c = t; c < E; c += kThreads) out[i * E + c] = s_db2[i * Ep + c];
#pragma unroll
  for (int j = 0; j < kVpt; ++j) {
    const int c = t + j * kThreads;
    if (c < E) {
      out[(int64_t)nb * E + c] = ag[j];
      out[(int64_t)(nb + 1) * E + c] = ab[j];
    }
  }
}

// z [B, nb H] (GEMM outputs, no bias), b3 / gamma / beta [nb H] -> y [B, nb H], stats [B, nb, 2]; blockIdx.y = block
__global__ void __launch_bounds__(kThreads)
ffn_fwd_kernel(const float* __restrict__ z, const float* __restrict__ b3, const float* __restrict__ gamma,
               const float* __restrict__ beta, int64_t B, int H, int nb, float* __restrict__ y,
               float* __restrict__ stats) {
  __shared__ float s_red[2 * kWarps];
  const int t = threadIdx.x, i = blockIdx.y;
  const int64_t ld = (int64_t)nb * H;
  const float* b3i = b3 + i * H;
  const float* gi = gamma + i * H;
  const float* bi = beta + i * H;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    const float* zr = z + b * ld + (int64_t)i * H;
    float x[kVpt];
    float s = 0.f, unused = 0.f;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      x[j] = c < H ? zr[c] + __ldg(b3i + c) : 0.f;
      s += x[j];
    }
    block_sum2(s, unused, s_red);
    const float mean = s / (float)H;
    float sq = 0.f;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      const float d = x[j] - mean;
      if (c < H) sq += d * d;
    }
    block_sum2(sq, unused, s_red);
    const float rstd = 1.0f / sqrtf(sq / (float)H + kEps);
    float* yr = y + b * ld + (int64_t)i * H;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      if (c < H) yr[c] = fmaxf((x[j] - mean) * rstd * __ldg(gi + c) + __ldg(bi + c), 0.f);
    }
    if (t == 0) {
      stats[2 * (b * nb + i)] = mean;
      stats[2 * (b * nb + i) + 1] = rstd;
    }
  }
}

// dy [B, nb H] -> dz [B, nb H], partials [nb][gridDim.x][3 H] = dgamma | dbeta | db3 of block blockIdx.y
__global__ void __launch_bounds__(kThreads)
ffn_bwd_kernel(const float* __restrict__ z, const float* __restrict__ b3, const float* __restrict__ gamma,
               const float* __restrict__ beta, const float* __restrict__ stats, const float* __restrict__ dy,
               int64_t B, int H, int nb, float* __restrict__ dz, float* __restrict__ partials) {
  __shared__ float s_red[2 * kWarps];
  const int t = threadIdx.x, i = blockIdx.y;
  const int64_t ld = (int64_t)nb * H;
  const float* b3i = b3 + i * H;
  const float* gi = gamma + i * H;
  const float* bi = beta + i * H;
  float ag[kVpt], ab[kVpt], az[kVpt];
#pragma unroll
  for (int j = 0; j < kVpt; ++j) ag[j] = ab[j] = az[j] = 0.f;
  for (int64_t b = blockIdx.x; b < B; b += gridDim.x) {
    const int64_t o = b * ld + (int64_t)i * H;
    const float mean = stats[2 * (b * nb + i)], rstd = stats[2 * (b * nb + i) + 1];
    float xh[kVpt], g[kVpt];
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      xh[j] = g[j] = 0.f;
      if (c < H) {
        xh[j] = (z[o + c] + __ldg(b3i + c) - mean) * rstd;
        const float yv = xh[j] * __ldg(gi + c) + __ldg(bi + c);
        const float d = yv > 0.f ? dy[o + c] : 0.f;
        ag[j] += d * xh[j];
        ab[j] += d;
        g[j] = d * __ldg(gi + c);
      }
      sg += g[j];
      sgx += g[j] * xh[j];
    }
    block_sum2(sg, sgx, s_red);
    const float mg = sg / (float)H, mgx = sgx / (float)H;
#pragma unroll
    for (int j = 0; j < kVpt; ++j) {
      const int c = t + j * kThreads;
      if (c < H) {
        const float d = rstd * (g[j] - mg - xh[j] * mgx);
        dz[o + c] = d;
        az[j] += d;
      }
    }
  }
  float* out = partials + ((int64_t)i * gridDim.x + blockIdx.x) * 3 * H;
#pragma unroll
  for (int j = 0; j < kVpt; ++j) {
    const int c = t + j * kThreads;
    if (c < H) {
      out[c] = ag[j];
      out[H + c] = ab[j];
      out[2 * H + c] = az[j];
    }
  }
}

// out[s, e] = sum over the G rows of partials [S][G][P], in row order; blockIdx.y = s
__global__ void __launch_bounds__(256) reduce_kernel(const float* __restrict__ partials, int G, int P,
                                                     float* __restrict__ out) {
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= P) return;
  const float* p = partials + (int64_t)blockIdx.y * G * P;
  float acc = 0.f;
  for (int g = 0; g < G; ++g) acc += p[(int64_t)g * P + e];
  out[(int64_t)blockIdx.y * P + e] = acc;
}

// ---- launchers (return 0, or 1 on unsupported arguments) -------------------------------------------------------------
inline size_t mask_bwd_smem(int Ep, int nb) { return sizeof(float) * (size_t)nb * Ep; }

inline int mask_fwd(const float* e, int lde, const float* m, const float* b2, const float* gamma, const float* beta,
                    int64_t B, int E, int nb, int grid, float* v, float* stats, cudaStream_t stream) {
  const int Ep = pad4(E);
  if (!usable(E, 4, nb) || lde < E || grid < 1) return 1;
  if (B == 0) return 0;
  TZK_LAUNCH((mask_fwd_kernel), grid, kThreads, 0, stream, e, lde, m, b2, gamma, beta, B, E, Ep, nb, v, stats);
  return 0;
}

// partials: grid * (nb + 2) E floats; dparams: (nb + 2) E floats (db2 [nb E] | dgamma [E] | dbeta [E])
inline int mask_bwd(const float* e, int lde, const float* m, const float* b2, const float* gamma, const float* beta,
                    const float* stats, const float* dv, int64_t B, int E, int nb, int grid, float* dm, float* de,
                    float* partials, float* dparams, cudaStream_t stream) {
  const int Ep = pad4(E);
  if (!usable(E, 4, nb) || lde < E || grid < 1) return 1;
  const int P = (nb + 2) * E;
  if (B == 0) {
    TZK_LAUNCH((reduce_kernel), dim3((P + 255) / 256, 1), 256, 0, stream, partials, 0, P, dparams);
    return 0;
  }
  TZK_LAUNCH((mask_bwd_kernel), grid, kThreads, mask_bwd_smem(Ep, nb), stream, e, lde, m, b2, gamma, beta, stats, dv,
             B, E, Ep, nb, dm, de, partials);
  TZK_LAUNCH((reduce_kernel), dim3((P + 255) / 256, 1), 256, 0, stream, partials, grid, P, dparams);
  return 0;
}

inline int ffn_fwd(const float* z, const float* b3, const float* gamma, const float* beta, int64_t B, int H, int nb,
                   int grid, float* y, float* stats, cudaStream_t stream) {
  if (!usable(1, H, nb) || grid < 1) return 1;
  if (B == 0) return 0;
  TZK_LAUNCH((ffn_fwd_kernel), dim3(grid, nb), kThreads, 0, stream, z, b3, gamma, beta, B, H, nb, y, stats);
  return 0;
}

// partials: nb * grid * 3 H floats; dparams: nb * 3 H floats (per block: dgamma [H] | dbeta [H] | db3 [H])
inline int ffn_bwd(const float* z, const float* b3, const float* gamma, const float* beta, const float* stats,
                   const float* dy, int64_t B, int H, int nb, int grid, float* dz, float* partials, float* dparams,
                   cudaStream_t stream) {
  if (!usable(1, H, nb) || grid < 1) return 1;
  const int P = 3 * H;
  if (B == 0) {
    TZK_LAUNCH((reduce_kernel), dim3((P + 255) / 256, nb), 256, 0, stream, partials, 0, P, dparams);
    return 0;
  }
  TZK_LAUNCH((ffn_bwd_kernel), dim3(grid, nb), kThreads, 0, stream, z, b3, gamma, beta, stats, dy, B, H, nb, dz,
             partials);
  TZK_LAUNCH((reduce_kernel), dim3((P + 255) / 256, nb), 256, 0, stream, partials, grid, P, dparams);
  return 0;
}
}  // namespace tzk_masknet
