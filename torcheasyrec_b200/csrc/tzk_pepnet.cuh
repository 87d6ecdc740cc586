// tzk_pepnet.cuh — PEPNet's gate-neural-unit product (tzrec/modules/personalized_net.py: GateNU.forward, EPNet.forward
// and the PPNet loop body) around its GEMMs, for up to 8 segments that share the batch size B:
//
//   gate_fwd  y_s = act_s(x_s + bx_s) * (gamma_s * sigmoid(z_s + bz_s))
//             x_s: the input of the activation without its bias (EPNet: the main embedding, identity, no bias; PPNet:
//             the task's main linear as a GEMM output), z_s: the gate's second layer as a GEMM output.
//   gate_bwd  dy_s -> dx_s = dy * g * act'(a), dz_s = dy * act(a) * gamma s (1 - s), and the batch sums dbx_s = sum_b
//             dx_s, dbz_s = sum_b dz_s.  a, s and g = gamma s are recomputed from the saved x and z.
//
// Each segment is [B, N] with N % 4 == 0 and row pitches that are multiples of 4 floats (column slices of a wider
// buffer are fine), so every access is 128-bit.  blockIdx.y is the segment; a CTA of 256 threads covers R = 256 / (N/4)
// rows per step (thread t owns column quad t % (N/4) of row t / (N/4)) and walks the rows grid-stride.  In the backward
// each thread keeps its quad's batch sums in registers, the R rows of the CTA are added in row order through shared
// memory into the CTA's row of a partials buffer, and tzk_batch_sum::reduce adds the rows in CTA order
// (tzk_batch_sum.cuh).
//
// fp32 throughout.  Plain CUDA (no PTX): nvcc builds it in tzk_pepnet.cu; g++ + tests/native/cuda_cpu_shim.h:
// tests/test_pepnet_cpu.py runs this source on the host against float64.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/tzk.h"
#include "tzk_batch_sum.cuh"
#include "tzk_launch.cuh"

namespace tzk_pepnet {
constexpr int kThreads = 256;
constexpr int kMaxN = 4 * kThreads;            // N / 4 column quads per row, at most one per thread
constexpr int kMaxSegs = TZK_PEPNET_MAX_SEGS;

inline bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

// the segments the kernels cover (the Python side's pepnet_usable states the same for whole modules)
inline int check(const tzk_pepnet_gate_args& a, bool backward) {
  if (a.B < 0 || a.B >= ((int64_t)1 << 31) || a.n_segs < 1 || a.n_segs > kMaxSegs) return 1;
  for (int s = 0; s < a.n_segs; ++s) {
    const tzk_pepnet_seg& g = a.seg[s];
    if (g.N < 4 || g.N > kMaxN || g.N % 4 != 0 || (g.act != TZK_PEPNET_IDENTITY && g.act != TZK_PEPNET_RELU)) return 1;
    if (g.ldx < g.N || g.ldz < g.N || g.ldy < g.N || g.ldx % 4 || g.ldz % 4 || g.ldy % 4) return 1;
    if (!aligned16(g.x) || !aligned16(g.z) || !aligned16(g.bx) || !aligned16(g.bz)) return 1;
    if (a.B > 0 && (!g.x || !g.z || !g.bz)) return 1;
    if (!backward && (!aligned16(g.y) || (a.B > 0 && !g.y))) return 1;
    if (backward && (!aligned16(g.dy) || !aligned16(g.dx) || !aligned16(g.dz) || (a.B > 0 && (!g.dy || !g.dx || !g.dz))))
      return 1;
  }
  return 0;
}

// floats of one partials row (and of dparams): dbx_s [N_s] | dbz_s [N_s] for every segment in order
inline int64_t partial_floats(const tzk_pepnet_gate_args& a) {
  int64_t P = 0;
  for (int s = 0; s < a.n_segs; ++s) P += 2 * (int64_t)a.seg[s].N;
  return P;
}

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }

// one element: a = x + bx, h = act(a), s = sigmoid(z + bz), g = gamma s
struct Elem {
  float h, g, s, da;
};
__device__ __forceinline__ Elem elem(float x, float bx, float z, float bz, int act, float gamma) {
  Elem e;
  const float a = x + bx;
  e.h = (act == TZK_PEPNET_RELU) ? fmaxf(a, 0.f) : a;
  e.da = (act == TZK_PEPNET_RELU) ? (a > 0.f ? 1.f : 0.f) : 1.f;
  e.s = 1.0f / (1.0f + expf(-(z + bz)));
  e.g = gamma * e.s;
  return e;
}

__global__ void __launch_bounds__(kThreads) gate_fwd_kernel(const __grid_constant__ tzk_pepnet_gate_args a) {
  const tzk_pepnet_seg& g = a.seg[blockIdx.y];
  const int N4 = g.N / 4, R = kThreads / N4;
  const int t = threadIdx.x, r = t / N4, c = 4 * (t % N4);
  if (r >= R) return;
  const float4 bx = g.bx ? ld4(g.bx + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 bz = ld4(g.bz + c);
  const int act = g.act;
  const float gamma = g.gamma;
  for (int64_t b = (int64_t)blockIdx.x * R + r; b < a.B; b += (int64_t)gridDim.x * R) {
    const float4 x = ld4(g.x + b * g.ldx + c), z = ld4(g.z + b * g.ldz + c);
    const Elem e0 = elem(x.x, bx.x, z.x, bz.x, act, gamma), e1 = elem(x.y, bx.y, z.y, bz.y, act, gamma);
    const Elem e2 = elem(x.z, bx.z, z.z, bz.z, act, gamma), e3 = elem(x.w, bx.w, z.w, bz.w, act, gamma);
    st4(g.y + b * g.ldy + c, make_float4(e0.h * e0.g, e1.h * e1.g, e2.h * e2.g, e3.h * e3.g));
  }
}

// dy_s (pitch ldy) -> dx_s / dz_s, written with the pitches of x_s / z_s.
// partials [gridDim.x][P]: the CTA's dbx_s | dbz_s at the segment's offset
__global__ void __launch_bounds__(kThreads) gate_bwd_kernel(const __grid_constant__ tzk_pepnet_gate_args a,
                                                            float* __restrict__ partials, int64_t P) {
  __shared__ float4 s_sum[2][kThreads];
  const int sg = blockIdx.y;
  const tzk_pepnet_seg& g = a.seg[sg];
  const int N4 = g.N / 4, R = kThreads / N4;
  const int t = threadIdx.x, r = t / N4, c = 4 * (t % N4);
  float4 sx = make_float4(0.f, 0.f, 0.f, 0.f), sz = sx;
  if (r < R) {
    const float4 bx = g.bx ? ld4(g.bx + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 bz = ld4(g.bz + c);
    const int act = g.act;
    const float gamma = g.gamma;
    for (int64_t b = (int64_t)blockIdx.x * R + r; b < a.B; b += (int64_t)gridDim.x * R) {
      const float4 x = ld4(g.x + b * g.ldx + c), z = ld4(g.z + b * g.ldz + c), dy = ld4(g.dy + b * g.ldy + c);
      const Elem e0 = elem(x.x, bx.x, z.x, bz.x, act, gamma), e1 = elem(x.y, bx.y, z.y, bz.y, act, gamma);
      const Elem e2 = elem(x.z, bx.z, z.z, bz.z, act, gamma), e3 = elem(x.w, bx.w, z.w, bz.w, act, gamma);
      const float4 dx = make_float4(dy.x * e0.g * e0.da, dy.y * e1.g * e1.da, dy.z * e2.g * e2.da, dy.w * e3.g * e3.da);
      const float4 dz = make_float4(dy.x * e0.h * (gamma * e0.s * (1.f - e0.s)), dy.y * e1.h * (gamma * e1.s * (1.f - e1.s)),
                                    dy.z * e2.h * (gamma * e2.s * (1.f - e2.s)), dy.w * e3.h * (gamma * e3.s * (1.f - e3.s)));
      st4(g.dx + b * g.ldx + c, dx);
      st4(g.dz + b * g.ldz + c, dz);
      sx.x += dx.x; sx.y += dx.y; sx.z += dx.z; sx.w += dx.w;
      sz.x += dz.x; sz.y += dz.y; sz.z += dz.z; sz.w += dz.w;
    }
  }
  s_sum[0][t] = sx;
  s_sum[1][t] = sz;
  __syncthreads();
  if (r == 0) {                         // the CTA's R rows of this quad, in row order
    for (int k = 1; k < R; ++k) {
      const float4 ax = s_sum[0][k * N4 + t], az = s_sum[1][k * N4 + t];
      sx.x += ax.x; sx.y += ax.y; sx.z += ax.z; sx.w += ax.w;
      sz.x += az.x; sz.y += az.y; sz.z += az.z; sz.w += az.w;
    }
    int64_t off = 0;
    for (int s = 0; s < sg; ++s) off += 2 * (int64_t)a.seg[s].N;
    float* out = partials + (int64_t)blockIdx.x * P + off;
    st4(out + c, sx);
    st4(out + g.N + c, sz);
  }
}

// ---- launchers (return 0, or 1 on arguments outside the cover) --------------------------------------------------------
inline int gate_fwd(const tzk_pepnet_gate_args& a, int grid, cudaStream_t stream) {
  if (check(a, false) != 0 || grid < 1) return 1;
  if (a.B == 0) return 0;
  TZK_LAUNCH((gate_fwd_kernel), dim3(grid, a.n_segs), kThreads, 0, stream, a);
  return 0;
}

// partials: grid * partial_floats(a) floats; dparams: partial_floats(a) floats
inline int gate_bwd(const tzk_pepnet_gate_args& a, int grid, float* partials, float* dparams, cudaStream_t stream) {
  if (check(a, true) != 0 || grid < 1) return 1;
  const int64_t P = partial_floats(a);
  if (a.B > 0) TZK_LAUNCH((gate_bwd_kernel), dim3(grid, a.n_segs), kThreads, 0, stream, a, partials, P);
  tzk_batch_sum::reduce(partials, a.B > 0 ? grid : 0, P, 1, dparams, stream);
  return 0;
}
}  // namespace tzk_pepnet
