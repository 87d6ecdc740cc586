// tzk_ple.cuh — the gates of one PLE extraction layer (tzrec/modules/extraction_net.py `_gate_forward`), all of them in
// one forward and one backward launch.  A layer has n_gates gates (T task gates, plus the shared gate when the layer is
// not the last); gate g reads one input x_g [B, K_g] (one of n_inputs distinct tensors: in the first layer every gate
// reads the same one) and mixes E_g of the layer's n_experts expert outputs [B, H]:
//
//   gate_fwd  per sample:  logits_g = x_g W_g^T + b_g,  p_g = softmax(logits_g),  y_g = sum_e p_{g,e} expert_{g,e}.
//             W stays in shared memory; p [B, sum E_g] is saved for the backward.  Each expert row is read once per
//             sample however many gates mix it; the reference's torch.stack is never formed.
//   gate_bwd  per sample:  s_{g,e} = <dy_g, expert_{g,e}>,  dlogit_{g,e} = p_{g,e} (s_{g,e} - sum_e' p_{g,e'} s_{g,e'}),
//             d expert = sum over the gates that mix it of p_{g,e} dy_g (in gate order, written once per element),
//             dx_i = sum over the gates reading input i of dlogit_g W_g (one write per distinct input), and the batch
//             sums dW_g = sum_b dlogit_g^T x_g, db_g = sum_b dlogit_g.
//
// One warp per sample (grid-stride over samples).  The logits are FP32 FFMA: lane l takes the columns k = l + 32 j of
// x_g and keeps one accumulator per expert (E_g <= 32); a transposing butterfly (31 shuffles) leaves logit e in lane e.
// E_g <= 32 columns is too narrow for a tensor-core tile.
//
// The backward's batch sums are owned, element by element, by one thread of the CTA: each CTA walks tiles of kTile
// samples, the warps write the tile's dlogits to shared memory, then thread t adds them into its own elements of the
// shared dW / db accumulators in sample order.  At the end each CTA writes its accumulators as one row of `partials`
// and reduce_kernel adds the rows in CTA order.  No float atomics: the result depends only on the grid, which the host
// derives from B, the shapes and the SM count, so a replayed graph gives the eager bits.
//
// Plain CUDA (no PTX): the includer provides TZK_DYN_SMEM / TZK_LAUNCH / TZK_SET_MAX_SMEM (nvcc: tzk_ple.cu; g++ +
// tests/native/cuda_cpu_shim.h: tests/test_ple_cpu.py runs this source on the host against a float64 restatement).
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/tzk.h"

namespace tzk_ple {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxGates = TZK_PLE_MAX_GATES;              // T <= 8 task gates + the shared gate
constexpr int kMaxExperts = TZK_PLE_MAX_EXPERTS;          // distinct expert tensors of a layer
constexpr int kMaxGateExperts = TZK_PLE_MAX_GATE_EXPERTS; // E_g: one logit per lane
constexpr int kMaxWidth = 1024;           // H and K_g
constexpr int kMaxWeightFloats = 20480;   // sum_g E_g K_g: W in shared memory (80 KB; the backward holds it twice)
constexpr int kTile = 16;                 // samples per backward tile

// One layer's gates, passed by value (a kernel parameter: no host-to-device copy, so the launch is graph-capturable).
struct Params {
  int64_t B;
  int H, n_experts, n_inputs, n_gates;
  int sumE, sumEK;                        // sum_g E_g, sum_g E_g K_g
  int in_dim[kMaxGates];                  // K of each distinct input
  int gate_input[kMaxGates];              // input index of gate g
  int gate_E[kMaxGates];
  int eoff[kMaxGates];                    // column of gate g in p / dlogit rows (prefix sum of E_g)
  int woff[kMaxGates];                    // offset of W_g in the weight block (prefix sum of E_g K_g)
  signed char pos[kMaxGates][kMaxExperts];   // position of expert x in gate g's list, or -1
  const float* experts[kMaxExperts];      // [B, H] each
  const float* inputs[kMaxGates];         // [B, K_i] each
  const float* weight[kMaxGates];         // [E_g, K_g]
  const float* bias[kMaxGates];           // [E_g]
  float* dx[kMaxGates];                   // backward: [B, K_i] each
};

inline size_t fwd_smem(const Params& a) {   // W | b | per warp: p
  return sizeof(float) * ((size_t)a.sumEK + a.sumE + (size_t)kWarps * a.sumE);
}
inline size_t bwd_smem(const Params& a) {
  // W | b | dW | db | dlogit tile | per warp: p, s
  return sizeof(float) * (2 * ((size_t)a.sumEK + a.sumE) + (size_t)kTile * a.sumE + 2 * (size_t)kWarps * a.sumE);
}

// sum over the warp in a fixed butterfly order; every lane gets the total
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// v[i] of every lane -> lane l returns sum over the lanes of v[l] (31 shuffles; the order is fixed)
__device__ __forceinline__ float transpose_sum(float (&v)[32], int lane) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const bool upper = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < o; ++i) {
      const float send = upper ? v[i] : v[i + o];
      const float keep = upper ? v[i + o] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return v[0];
}

// W and b of every gate into shared memory (W_g at woff[g], row pitch K_g; b_g after the weights at sumEK + eoff[g])
__device__ __forceinline__ void load_weights(const Params& a, float* sW) {
  for (int g = 0; g < a.n_gates; ++g) {
    const int n = a.gate_E[g] * a.in_dim[a.gate_input[g]];
    for (int i = threadIdx.x; i < n; i += kThreads) sW[a.woff[g] + i] = a.weight[g][i];
    for (int i = threadIdx.x; i < a.gate_E[g]; i += kThreads) sW[a.sumEK + a.eoff[g] + i] = a.bias[g][i];
  }
}

// logit e of gate g for sample b in lane e (lanes >= E_g: undefined)
__device__ __forceinline__ float gate_logit(const Params& a, const float* sW, int g, int64_t b, int lane) {
  const int K = a.in_dim[a.gate_input[g]], Eg = a.gate_E[g];
  const float* x = a.inputs[a.gate_input[g]] + b * K;
  const float* w = sW + a.woff[g];
  float acc[32];
#pragma unroll
  for (int e = 0; e < 32; ++e) acc[e] = 0.f;
  for (int k0 = 0; k0 < K; k0 += 32) {
    const int k = k0 + lane;
    const float xv = k < K ? x[k] : 0.f;
    const int kk = k < K ? k : K - 1;              // in-range read; its product is 0
#pragma unroll
    for (int e = 0; e < 32; ++e)
      if (e < Eg) acc[e] += xv * w[e * K + kk];
  }
  const float s = transpose_sum(acc, lane);
  return lane < Eg ? s + sW[a.sumEK + a.eoff[g] + lane] : 0.f;
}

// -> y [n_gates, B, H], p [B, sumE]
__global__ void __launch_bounds__(kThreads) gate_fwd_kernel(const __grid_constant__ Params a, float* __restrict__ y,
                                                            float* __restrict__ p) {
  TZK_DYN_SMEM(float, sW);                 // W | b | per warp: the current sample's p [sumE]
  load_weights(a, sW);
  __syncthreads();
  const int lane = threadIdx.x % 32, w = threadIdx.x / 32;
  float* sP = sW + a.sumEK + a.sumE + w * a.sumE;
  const int64_t B = a.B, H = a.H;
  for (int64_t b = (int64_t)blockIdx.x * kWarps + w; b < B; b += (int64_t)gridDim.x * kWarps) {
    for (int g = 0; g < a.n_gates; ++g) {
      const int Eg = a.gate_E[g];
      const float l = gate_logit(a, sW, g, b, lane);
      const float m = warp_max(lane < Eg ? l : -INFINITY);
      const float ex = lane < Eg ? expf(l - m) : 0.f;
      const float pr = ex / warp_sum(ex);
      if (lane < Eg) {
        p[b * a.sumE + a.eoff[g] + lane] = pr;
        sP[a.eoff[g] + lane] = pr;
      }
    }
    __syncwarp();
    for (int h = lane; h < H; h += 32) {
      float acc[kMaxGates];
#pragma unroll
      for (int g = 0; g < kMaxGates; ++g) acc[g] = 0.f;
      for (int x = 0; x < a.n_experts; ++x) {
        const float v = a.experts[x][b * H + h];
#pragma unroll
        for (int g = 0; g < kMaxGates; ++g) {
          const int e = g < a.n_gates ? a.pos[g][x] : -1;
          if (e >= 0) acc[g] += sP[a.eoff[g] + e] * v;
        }
      }
#pragma unroll
      for (int g = 0; g < kMaxGates; ++g)
        if (g < a.n_gates) y[(g * B + b) * H + h] = acc[g];
    }
    __syncwarp();
  }
}

// dy [n_gates, B, H], p [B, sumE] -> d_experts [n_experts, B, H], dx_i (a.dx), partials row per CTA: dW | db
__global__ void __launch_bounds__(kThreads) gate_bwd_kernel(const __grid_constant__ Params a,
                                                            const float* __restrict__ p, const float* __restrict__ dy,
                                                            float* __restrict__ d_experts,
                                                            float* __restrict__ partials) {
  TZK_DYN_SMEM(float, sW);                 // W | b | dW | db | dlogit tile [kTile][sumE] | per warp: p, s [sumE]
  float* sdW = sW + a.sumEK + a.sumE;
  float* sdb = sdW + a.sumEK;
  float* sDL = sdb + a.sumE;
  load_weights(a, sW);
  for (int i = threadIdx.x; i < a.sumEK + a.sumE; i += kThreads) sdW[i] = 0.f;    // dW and db
  __syncthreads();
  const int lane = threadIdx.x % 32, w = threadIdx.x / 32;
  float* sP = sDL + kTile * a.sumE + 2 * w * a.sumE;
  float* sS = sP + a.sumE;
  const int64_t B = a.B, H = a.H;
  for (int64_t t0 = (int64_t)blockIdx.x * kTile; t0 < B; t0 += (int64_t)gridDim.x * kTile) {
    for (int ls = w; ls < kTile; ls += kWarps) {
      const int64_t b = t0 + ls;
      float* dl = sDL + ls * a.sumE;
      if (b >= B) {
        for (int i = lane; i < a.sumE; i += 32) dl[i] = 0.f;
        continue;
      }
      for (int i = lane; i < a.sumE; i += 32) sP[i] = p[b * a.sumE + i];
      __syncwarp();
      // s_{g,e} and the expert gradients, one expert at a time (its row read once)
      for (int x = 0; x < a.n_experts; ++x) {
        float s[kMaxGates];
#pragma unroll
        for (int g = 0; g < kMaxGates; ++g) s[g] = 0.f;
        for (int h = lane; h < H; h += 32) {
          const float v = a.experts[x][b * H + h];
          float d = 0.f;
#pragma unroll
          for (int g = 0; g < kMaxGates; ++g) {
            const int e = g < a.n_gates ? a.pos[g][x] : -1;
            if (e >= 0) {
              const float dyv = dy[(g * B + b) * H + h];
              s[g] += dyv * v;
              d += sP[a.eoff[g] + e] * dyv;
            }
          }
          d_experts[((int64_t)x * B + b) * H + h] = d;
        }
#pragma unroll
        for (int g = 0; g < kMaxGates; ++g) {
          const int e = g < a.n_gates ? a.pos[g][x] : -1;
          if (e >= 0) {
            const float t = warp_sum(s[g]);
            if (lane == 0) sS[a.eoff[g] + e] = t;
          }
        }
      }
      __syncwarp();
      // softmax backward
      for (int g = 0; g < a.n_gates; ++g) {
        const int Eg = a.gate_E[g];
        const float pr = lane < Eg ? sP[a.eoff[g] + lane] : 0.f;
        const float sv = lane < Eg ? sS[a.eoff[g] + lane] : 0.f;
        const float mean = warp_sum(pr * sv);
        if (lane < Eg) dl[a.eoff[g] + lane] = pr * (sv - mean);
      }
      __syncwarp();
      // dx_i = sum over the gates reading input i of dlogit_g W_g
      for (int i = 0; i < a.n_inputs; ++i) {
        const int K = a.in_dim[i];
        for (int k = lane; k < K; k += 32) {
          float acc = 0.f;
          for (int g = 0; g < a.n_gates; ++g) {
            if (a.gate_input[g] != i) continue;
            const float* wg = sW + a.woff[g] + k;
            const float* dlg = dl + a.eoff[g];
            for (int e = 0; e < a.gate_E[g]; ++e) acc += dlg[e] * wg[e * K];
          }
          a.dx[i][b * K + k] = acc;
        }
      }
      __syncwarp();
    }
    __syncthreads();
    // the tile's batch sums: thread t owns columns k = t + kThreads j of every dW_g row and entries t + kThreads j of db
    const int n = (int)(B - t0 < kTile ? B - t0 : kTile);
    for (int g = 0; g < a.n_gates; ++g) {
      const int K = a.in_dim[a.gate_input[g]], Eg = a.gate_E[g];
      const float* x = a.inputs[a.gate_input[g]] + t0 * K;
      for (int k = threadIdx.x; k < K; k += kThreads) {
        float xs[kTile];
#pragma unroll
        for (int s = 0; s < kTile; ++s) xs[s] = s < n ? x[(int64_t)s * K + k] : 0.f;
        for (int e = 0; e < Eg; ++e) {
          float acc = sdW[a.woff[g] + e * K + k];
#pragma unroll
          for (int s = 0; s < kTile; ++s) acc += sDL[s * a.sumE + a.eoff[g] + e] * xs[s];
          sdW[a.woff[g] + e * K + k] = acc;
        }
      }
    }
    for (int i = threadIdx.x; i < a.sumE; i += kThreads) {
      float acc = sdb[i];
      for (int s = 0; s < kTile; ++s) acc += sDL[s * a.sumE + i];
      sdb[i] = acc;
    }
    __syncthreads();
  }
  float* out = partials + (int64_t)blockIdx.x * (a.sumEK + a.sumE);
  for (int i = threadIdx.x; i < a.sumEK + a.sumE; i += kThreads) out[i] = sdW[i];
}

// out[e] = sum over the G rows of partials [G][P], in row order
__global__ void __launch_bounds__(256) reduce_kernel(const float* __restrict__ partials, int G, int P,
                                                     float* __restrict__ out) {
  const int e = blockIdx.x * 256 + threadIdx.x;
  if (e >= P) return;
  float acc = 0.f;
  for (int g = 0; g < G; ++g) acc += partials[(int64_t)g * P + e];
  out[e] = acc;
}

// ---- host side -------------------------------------------------------------------------------------------------------
// Params from the C-ABI description, with the derived fields (sumE, sumEK, eoff, woff, pos); 0, or 1 when the layer is
// outside the kernels' cover: 1 <= n_gates <= 9, 1 <= n_experts <= 64, 1 <= n_inputs <= 9, 1 <= H <= 1024,
// 1 <= K_i <= 1024, 1 <= E_g <= 32 distinct experts per gate, sum_g E_g K_g <= kMaxWeightFloats.
inline int prepare(const tzk_ple_gate_args& c, Params& a) {
  if (c.B < 0 || c.n_gates < 1 || c.n_gates > kMaxGates || c.n_experts < 1 || c.n_experts > kMaxExperts ||
      c.n_inputs < 1 || c.n_inputs > kMaxGates || c.H < 1 || c.H > kMaxWidth)
    return 1;
  a.B = c.B;
  a.H = c.H;
  a.n_experts = c.n_experts;
  a.n_inputs = c.n_inputs;
  a.n_gates = c.n_gates;
  for (int x = 0; x < kMaxExperts; ++x) a.experts[x] = x < c.n_experts ? c.experts[x] : nullptr;
  for (int i = 0; i < kMaxGates; ++i) {
    const bool in = i < c.n_inputs;
    a.in_dim[i] = in ? c.in_dim[i] : 0;
    a.inputs[i] = in ? c.inputs[i] : nullptr;
    a.dx[i] = in ? c.d_inputs[i] : nullptr;
    if (in && (a.in_dim[i] < 1 || a.in_dim[i] > kMaxWidth)) return 1;
  }
  int sumE = 0;
  long sumEK = 0;
  for (int g = 0; g < kMaxGates; ++g) {
    for (int x = 0; x < kMaxExperts; ++x) a.pos[g][x] = -1;
    a.gate_input[g] = a.gate_E[g] = a.eoff[g] = a.woff[g] = 0;
    a.weight[g] = a.bias[g] = nullptr;
    if (g >= c.n_gates) continue;
    const int Eg = c.gate_num_experts[g];
    if (c.gate_input[g] < 0 || c.gate_input[g] >= c.n_inputs || Eg < 1 || Eg > kMaxGateExperts) return 1;
    for (int e = 0; e < Eg; ++e) {
      const int x = c.gate_experts[g][e];
      if (x >= c.n_experts || a.pos[g][x] >= 0) return 1;
      a.pos[g][x] = (signed char)e;
    }
    a.gate_input[g] = c.gate_input[g];
    a.gate_E[g] = Eg;
    a.weight[g] = c.weight[g];
    a.bias[g] = c.bias[g];
    a.eoff[g] = sumE;
    a.woff[g] = (int)sumEK;
    sumE += Eg;
    sumEK += (long)Eg * a.in_dim[c.gate_input[g]];
  }
  if (sumEK > kMaxWeightFloats) return 1;
  a.sumE = sumE;
  a.sumEK = (int)sumEK;
  return 0;
}

inline int gate_fwd(const Params& a, int grid, float* y, float* p, cudaStream_t stream) {
  if (grid < 1) return 1;
  if (a.B == 0) return 0;
  const size_t smem = fwd_smem(a);
  TZK_SET_MAX_SMEM(gate_fwd_kernel, smem);
  TZK_LAUNCH((gate_fwd_kernel), grid, kThreads, smem, stream, a, y, p);
  return 0;
}

// partials: grid * (sumEK + sumE) floats; dparams: sumEK + sumE floats (dW_0 | dW_1 | ... | db_0 | db_1 | ...)
inline int gate_bwd(const Params& a, const float* p, const float* dy, int grid, float* d_experts, float* partials,
                    float* dparams, cudaStream_t stream) {
  if (grid < 1) return 1;
  const int P = a.sumEK + a.sumE;
  if (a.B == 0) {
    TZK_LAUNCH((reduce_kernel), (P + 255) / 256, 256, 0, stream, partials, 0, P, dparams);
    return 0;
  }
  const size_t smem = bwd_smem(a);
  TZK_SET_MAX_SMEM(gate_bwd_kernel, smem);
  TZK_LAUNCH((gate_bwd_kernel), grid, kThreads, smem, stream, a, p, dy, d_experts, partials);
  TZK_LAUNCH((reduce_kernel), (P + 255) / 256, 256, 0, stream, partials, grid, P, dparams);
  return 0;
}
}  // namespace tzk_ple
