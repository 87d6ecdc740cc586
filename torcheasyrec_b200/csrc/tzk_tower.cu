// tzk_tower.cu — narrow fully-connected layers and the BCE head of the rank models (callers of the hot path:
// tzrec/modules/mlp.py:20-84 Perceptron = Linear -> ReLU, tzrec/models/rank_model.py:190-216 BCEWithLogitsLoss).
//
// A DLRM / DeepFM step runs a handful of layers whose weight matrix is at most 64 x 64 (13->64->16 bottom MLP,
// 64->32->1 top of the final MLP, every tower's Linear(64, 1)).  As library GEMMs each of them costs 3-6 launches
// forward and 6-10 backward (GEMM, split-K reduce, bias add, clamp, ReLU mask, column sums) and every launch is
// latency-bound at these sizes.  Here a layer is ONE launch forward (a thread owns a row, the weight matrix is
// broadcast from shared memory) and one (+ a tiny fixed-order reduction) backward (a CTA walks 128-row tiles: dz, dX,
// per-CTA dW / db partials).  Plain fp32 FFMA in ascending-k order (the reference runs these layers as fp32 SIMT GEMMs,
// TF32 off).  Weight / bias gradients are summed per CTA and then across CTAs in a fixed order: run-to-run deterministic.
#include <cstdlib>

#include "tzk_common.cuh"

// second backward implementation (plain CUDA, also compiled for the host by the CPU tests)
#include "tzk_launch.cuh"
#include "tzk_tower_bwd2.cuh"
#include "tzk_tower_tail.cuh"

using namespace tzk;

namespace {
constexpr int kTM = 128;  // rows per tile == threads per CTA

__device__ __forceinline__ int odd(int v) { return v | 1; }  // odd row stride: thread-per-row reads are conflict-free
constexpr int kNW = kTM / 32;  // warps per CTA
constexpr int kLU = 16;        // rows in flight per warp while a tile is loaded

// global [rows x C] (row stride ld, C <= 64) -> shared [rows x S]: a warp per row, lanes over columns, kLU rows'
// worth of independent loads issued before the first is consumed.  `mask` (nullable, row stride ld_m): values whose
// mask entry is <= 0 are stored as 0 (ReLU backward).
__device__ __forceinline__ void load_tile(float* dst, int S, const float* __restrict__ src, int64_t ld,
                                          const float* __restrict__ mask, int64_t ld_m, int rows, int C) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r0 = warp; r0 < rows; r0 += kNW * kLU) {
    float v[kLU][2], m[kLU][2];
#pragma unroll
    for (int q = 0; q < kLU; ++q) {
      const int r = r0 + q * kNW;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cc = lane + 32 * h;
        const bool ok = r < rows && cc < C;
        v[q][h] = ok ? __ldg(src + (int64_t)r * ld + cc) : 0.f;
        m[q][h] = (ok && mask) ? __ldg(mask + (int64_t)r * ld_m + cc) : 1.f;
      }
    }
#pragma unroll
    for (int q = 0; q < kLU; ++q) {
      const int r = r0 + q * kNW;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cc = lane + 32 * h;
        if (r < rows && cc < C) dst[r * S + cc] = m[q][h] > 0.f ? v[q][h] : 0.f;
      }
    }
  }
}
__device__ __forceinline__ void store_tile(float* __restrict__ dst, int64_t ld, const float* src, int S, int rows,
                                           int C) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < rows; r += kNW)
    for (int cc = lane; cc < C; cc += 32) dst[(int64_t)r * ld + cc] = src[r * S + cc];
}

// ---------------------------------------------------------------------------------------------------
// forward: y = act(x @ W^T + b)   x [M,K]  W [N,K]  y [M,N]   K, N <= 64
// One thread per row, no tile staging and no barrier after the weight matrix is in shared memory (a staged-tile
// variant with three barriers per 128 rows was slower over the four DLRM layers).  A thread reads its own row straight from global memory (the 32 rows of a warp are one
// contiguous 32*K*4-byte span, so every sector that is fetched is fully consumed through L1 over the k loop) and
// writes its own output row with 16-B stores.  Many independent warps per SM hide the load latency.
// ---------------------------------------------------------------------------------------------------
constexpr int kRowThreads = 128;
template <int NP, bool VEC>
__global__ void __launch_bounds__(kRowThreads, 5)
small_linear_fwd_rows_kernel(const float* __restrict__ x, int64_t ld_x, const float* __restrict__ w,
                             const float* __restrict__ bias, int64_t M, int K, int N, int relu,
                             float* __restrict__ y, int64_t ld_y) {
  constexpr int NH = NP < 32 ? NP : 32;   // outputs per pass: 32 accumulators keep 6 CTAs (24 warps) per SM resident
  extern __shared__ __align__(16) float sm[];
  float* Wt = sm;             // [K][NP], zero beyond N
  float* bs = Wt + K * NP;    // [NP]
  const int tid = threadIdx.x;
  for (int i = tid; i < K * NP; i += kRowThreads) Wt[i] = 0.f;
  for (int i = tid; i < NP; i += kRowThreads) bs[i] = (bias && i < N) ? __ldg(bias + i) : 0.f;
  __syncthreads();
  for (int i = tid; i < N * K; i += kRowThreads) {
    const int n = i / K, k = i - n * K;
    Wt[k * NP + n] = __ldg(w + i);
  }
  __syncthreads();
  const bool vec_out = (N & 3) == 0 && (ld_y & 3) == 0 && ((uintptr_t)y & 15) == 0;
  for (int64_t row = (int64_t)blockIdx.x * kRowThreads + tid; row < M; row += (int64_t)gridDim.x * kRowThreads) {
    const float* xr = x + row * ld_x;
    float* yr = y + row * ld_y;
#pragma unroll 1
    for (int n0 = 0; n0 < NP; n0 += NH) {   // second pass re-reads the row from L1
      if (n0 >= N) break;
      float acc[NH];
#pragma unroll
      for (int n = 0; n < NH; ++n) acc[n] = bs[n0 + n];
      if (VEC) {   // K % 4 == 0, rows 16-B aligned
        for (int k0 = 0; k0 < K; k0 += 4) {
          const float4 xv4 = *reinterpret_cast<const float4*>(xr + k0);
          const float xv[4] = {xv4.x, xv4.y, xv4.z, xv4.w};
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            const float4* wr = reinterpret_cast<const float4*>(Wt + (k0 + kk) * NP + n0);
#pragma unroll
            for (int n4 = 0; n4 < NH / 4; ++n4) {
              const float4 w4 = wr[n4];
              acc[n4 * 4 + 0] = fmaf(xv[kk], w4.x, acc[n4 * 4 + 0]);
              acc[n4 * 4 + 1] = fmaf(xv[kk], w4.y, acc[n4 * 4 + 1]);
              acc[n4 * 4 + 2] = fmaf(xv[kk], w4.z, acc[n4 * 4 + 2]);
              acc[n4 * 4 + 3] = fmaf(xv[kk], w4.w, acc[n4 * 4 + 3]);
            }
          }
        }
      } else {
#pragma unroll 4
        for (int k = 0; k < K; ++k) {
          const float xv = xr[k];
          const float4* wr = reinterpret_cast<const float4*>(Wt + k * NP + n0);
#pragma unroll
          for (int n4 = 0; n4 < NH / 4; ++n4) {
            const float4 w4 = wr[n4];
            acc[n4 * 4 + 0] = fmaf(xv, w4.x, acc[n4 * 4 + 0]);
            acc[n4 * 4 + 1] = fmaf(xv, w4.y, acc[n4 * 4 + 1]);
            acc[n4 * 4 + 2] = fmaf(xv, w4.z, acc[n4 * 4 + 2]);
            acc[n4 * 4 + 3] = fmaf(xv, w4.w, acc[n4 * 4 + 3]);
          }
        }
      }
      if (relu) {
#pragma unroll
        for (int n = 0; n < NH; ++n) acc[n] = acc[n] > 0.f ? acc[n] : 0.f;
      }
      if (vec_out) {
#pragma unroll
        for (int n4 = 0; n4 < NH / 4; ++n4)
          if (n0 + n4 * 4 < N)
            *reinterpret_cast<float4*>(yr + n0 + n4 * 4) =
                make_float4(acc[n4 * 4], acc[n4 * 4 + 1], acc[n4 * 4 + 2], acc[n4 * 4 + 3]);
      } else {
#pragma unroll
        for (int n = 0; n < NH; ++n)
          if (n0 + n < N) yr[n0 + n] = acc[n];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// backward: dz = dy * (relu ? y > 0 : 1);  dx = dz @ W;  dW = dz^T @ x;  db = colsum(dz)
// per-CTA partial dW / db -> `partial[cta][N*K + N]`, reduced in CTA order by small_linear_reduce_kernel.
// ---------------------------------------------------------------------------------------------------
template <int KP, int NP>
__global__ void __launch_bounds__(kTM)
small_linear_bwd_kernel(const float* __restrict__ x, int64_t ld_x, const float* __restrict__ w,
                        const float* __restrict__ y, int64_t ld_y, const float* __restrict__ dy, int64_t ld_dy,
                        int64_t M, int K, int N, int relu, float* __restrict__ dx, int64_t ld_dx,
                        float* __restrict__ partial) {
  // dW micro-tiles: TN x TK threads, each NB x KB outputs
  constexpr int TN = NP >= 8 ? 8 : NP;
  constexpr int TK = kTM / TN;
  constexpr int NB = NP / TN;
  constexpr int KB = KP / TK > 0 ? KP / TK : 1;
  extern __shared__ __align__(16) float sm[];
  float* Ws = sm;                  // [N][KP] (row n of W, zero beyond K)
  const int KS = odd(K), NS = odd(N);
  float* xt = Ws + N * KP;         // [kTM][KS]
  float* dzt = xt + kTM * KS;      // [kTM][NS]
  const int tid = threadIdx.x;
  for (int i = tid; i < N * KP; i += kTM) {
    const int n = i / KP, k = i - n * KP;
    Ws[i] = k < K ? __ldg(w + (int64_t)n * K + k) : 0.f;
  }
  const int tn = tid / TK, tk = tid - tn * TK;
  const int n0 = tn * NB, k0 = tk * KB;
  float accW[NB][KB];
#pragma unroll
  for (int i = 0; i < NB; ++i)
#pragma unroll
    for (int j = 0; j < KB; ++j) accW[i][j] = 0.f;
  float accB = 0.f;
  __syncthreads();
  const int64_t n_tiles = ceil_div64(M, kTM);
  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t row0 = t * kTM;
    const int rows = (int)((M - row0) < kTM ? (M - row0) : kTM);
    load_tile(xt, KS, x + row0 * ld_x, ld_x, nullptr, 0, rows, K);
    load_tile(dzt, NS, dy + row0 * ld_dy, ld_dy, relu ? y + row0 * ld_y : nullptr, ld_y, rows, N);
    __syncthreads();
    // ---- dW += dz^T x over the tile's rows (ascending), db likewise ---------------------------------
    if (k0 < K && n0 < N) {
#pragma unroll 4
      for (int r = 0; r < rows; ++r) {
        float a[NB], b[KB];
#pragma unroll
        for (int i = 0; i < NB; ++i) a[i] = (n0 + i < N) ? dzt[r * NS + n0 + i] : 0.f;
#pragma unroll
        for (int j = 0; j < KB; ++j) b[j] = (k0 + j < K) ? xt[r * KS + k0 + j] : 0.f;
#pragma unroll
        for (int i = 0; i < NB; ++i)
#pragma unroll
          for (int j = 0; j < KB; ++j) accW[i][j] = fmaf(a[i], b[j], accW[i][j]);
      }
    }
    if (tid < N) {
#pragma unroll 8
      for (int r = 0; r < rows; ++r) accB += dzt[r * NS + tid];
    }
    // ---- dx = dz @ W : one thread per row ------------------------------------------------------------
    if (dx) {
      float acc[KP];
#pragma unroll
      for (int k = 0; k < KP; ++k) acc[k] = 0.f;
      if (tid < rows) {
        const float* dr = dzt + tid * NS;
#pragma unroll 2
        for (int n = 0; n < N; ++n) {
          const float dv = dr[n];
          const float4* wr = reinterpret_cast<const float4*>(Ws + n * KP);
#pragma unroll
          for (int k4 = 0; k4 < KP / 4; ++k4) {
            const float4 w4 = wr[k4];
            acc[k4 * 4 + 0] = fmaf(dv, w4.x, acc[k4 * 4 + 0]);
            acc[k4 * 4 + 1] = fmaf(dv, w4.y, acc[k4 * 4 + 1]);
            acc[k4 * 4 + 2] = fmaf(dv, w4.z, acc[k4 * 4 + 2]);
            acc[k4 * 4 + 3] = fmaf(dv, w4.w, acc[k4 * 4 + 3]);
          }
        }
      }
      __syncthreads();  // dW / db loops are done with the x tile
      if (tid < rows) {
        float* xr = xt + tid * KS;
#pragma unroll
        for (int k = 0; k < KP; ++k)
          if (k < K) xr[k] = acc[k];
      }
      __syncthreads();
      store_tile(dx + row0 * ld_dx, ld_dx, xt, KS, rows, K);
    }
    __syncthreads();
  }
  float* p = partial + (int64_t)blockIdx.x * (N * K + N);
  if (k0 < K && n0 < N) {
#pragma unroll
    for (int i = 0; i < NB; ++i)
#pragma unroll
      for (int j = 0; j < KB; ++j)
        if (n0 + i < N && k0 + j < K) p[(n0 + i) * K + k0 + j] = accW[i][j];
  }
  if (tid < N) p[N * K + tid] = accB;
}

// out[i] = sum_c partial[c][i]: 32 outputs x 8 partial-groups per CTA; each thread adds its partials (c = g, g+8, ...)
// with 4 loads in flight, the 8 group sums are folded in a fixed order -> deterministic.
__global__ void __launch_bounds__(256)
small_linear_reduce_kernel(const float* __restrict__ partial, int n_parts, int NK, int N, float* __restrict__ dw,
                           float* __restrict__ db) {
  __shared__ float red[8][32];
  const int o = threadIdx.x & 31, g = threadIdx.x >> 5;
  const int i = blockIdx.x * 32 + o;
  const int total = NK + N;
  float s = 0.f;
  if (i < total) {
    int c = g;
    for (; c + 24 < n_parts; c += 32) {
      const float a0 = partial[(int64_t)c * total + i], a1 = partial[(int64_t)(c + 8) * total + i];
      const float a2 = partial[(int64_t)(c + 16) * total + i], a3 = partial[(int64_t)(c + 24) * total + i];
      s += a0; s += a1; s += a2; s += a3;
    }
    for (; c < n_parts; c += 8) s += partial[(int64_t)c * total + i];
  }
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

inline int pad_pow(int v, int lo) {  // smallest of {lo, 16, 32, 64} >= v
  int p = lo;
  while (p < v) p = p < 16 ? 16 : p * 2;
  return p;
}
inline int bwd_grid(int64_t M) {   // = number of weight-gradient partials; 4 CTAs (16 warps) per SM hide the tile loads
  const int64_t t = ceil_div64(M < 1 ? 1 : M, kTM);
  return (int)(t < kSmCountH100 * 4 ? t : kSmCountH100 * 4);
}

// ---------------------------------------------------------------------------------------------------
// BCE with logits, mean reduction, forward and dloss/dlogits in one pass
//   loss_i = max(z,0) - z*t + log1p(exp(-|z|))        d_i = (sigmoid(z) - t) / M
// ---------------------------------------------------------------------------------------------------
constexpr int kBceThreads = 256;
constexpr int kBcePerThread = 4;
__global__ void __launch_bounds__(kBceThreads)
bce_fwd_bwd_kernel(const float* __restrict__ z, const float* __restrict__ t, int64_t M, float inv_m,
                   float* __restrict__ dz, float* __restrict__ partial) {
  __shared__ float red[kBceThreads / 32];
  float acc = 0.f;
  const int64_t base = (int64_t)blockIdx.x * (kBceThreads * kBcePerThread);
#pragma unroll
  for (int u = 0; u < kBcePerThread; ++u) {
    const int64_t i = base + u * kBceThreads + threadIdx.x;
    if (i < M) {
      const float zi = __ldg(z + i), ti = __ldg(t + i);
      const float e = expf(-fabsf(zi));
      acc += fmaxf(zi, 0.f) - zi * ti + log1pf(e);
      const float sig = zi >= 0.f ? 1.f / (1.f + e) : e / (1.f + e);
      if (dz) dz[i] = (sig - ti) * inv_m;
    }
  }
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < kBceThreads / 32; ++k) s += red[k];
    partial[blockIdx.x] = s;
  }
}
__global__ void __launch_bounds__(256)
bce_final_kernel(const float* __restrict__ partial, int n, float inv_m, float* __restrict__ loss) {
  __shared__ float red[256];
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += 256) s += partial[i];  // fixed assignment, fixed tree below
  red[threadIdx.x] = s;
  __syncthreads();
  for (int d = 128; d >= 1; d >>= 1) {
    if (threadIdx.x < d) red[threadIdx.x] += red[threadIdx.x + d];
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[0] = red[0] * inv_m;
}
}  // namespace

static int small_linear_check(const char* who, int64_t M, int32_t K, int32_t N) {
  TZK_REQUIRE(M >= 0, "%s: negative M", who);
  TZK_REQUIRE(K >= 1 && K <= 64 && N >= 1 && N <= 64, "%s: K=%d, N=%d outside [1,64]", who, K, N);
  return 0;
}

extern "C" int tzk_small_linear_fwd(const float* x, int64_t ld_x, const float* w, const float* bias, int64_t M,
                                    int32_t K, int32_t N, int32_t relu, float* y, int64_t ld_y,
                                    tzk_stream_t stream) {
  int rc = small_linear_check("small_linear_fwd", M, K, N);
  if (rc) return rc;
  if (M == 0) return 0;
  TZK_REQUIRE(x && w && y, "small_linear_fwd: NULL argument");
  TZK_REQUIRE(ld_x >= K && ld_y >= N, "small_linear_fwd: leading dimension smaller than the row");
  const int NP = pad_pow(N, 4);
  {
    const size_t smem_r = ((size_t)K * NP + NP) * sizeof(float);
    const bool vec = (K % 4 == 0) && (ld_x % 4 == 0) && ((uintptr_t)x % 16 == 0);
    const int64_t blocks = ceil_div64(M, kRowThreads);
    const int grid_r = (int)(blocks < kSmCountH100 * 16 ? blocks : kSmCountH100 * 16);
#define TZK_SLR(NP_)                                                                                                \
  do {                                                                                                              \
    if (vec)                                                                                                        \
      small_linear_fwd_rows_kernel<NP_, true><<<grid_r, kRowThreads, smem_r, as_stream(stream)>>>(                  \
          x, ld_x, w, bias, M, K, N, relu, y, ld_y);                                                                \
    else                                                                                                            \
      small_linear_fwd_rows_kernel<NP_, false><<<grid_r, kRowThreads, smem_r, as_stream(stream)>>>(                 \
          x, ld_x, w, bias, M, K, N, relu, y, ld_y);                                                                \
  } while (0)
    switch (NP) {
      case 4: TZK_SLR(4); break;
      case 16: TZK_SLR(16); break;
      case 32: TZK_SLR(32); break;
      default: TZK_SLR(64); break;
    }
#undef TZK_SLR
    TZK_CHECK_LAUNCH("small_linear_fwd_rows_kernel");
  }
  return 0;
}

// TZK_SMALL_LINEAR_BWD=1: 128-row shared-memory tiles (small_linear_bwd_kernel); default: the barrier-free pair of
// kernels of tzk_tower_bwd2.cuh wherever its row-group mapping covers the shape.  Read per call (tests flip it).
static bool use_bwd2(int K, int N) {
  const char* e = getenv("TZK_SMALL_LINEAR_BWD");
  return !(e && e[0] == '1') && tzk_bwd2::supported(K, N);
}

extern "C" size_t tzk_small_linear_bwd_workspace_bytes(int64_t M, int32_t K, int32_t N) {
  const size_t v1 = (size_t)bwd_grid(M) * ((size_t)(N < 1 ? 1 : N) * (K < 1 ? 1 : K) + (N < 1 ? 1 : N)) * sizeof(float);
  const size_t v2 = tzk_bwd2::supported(K, N) ? tzk_bwd2::workspace_bytes(M < 1 ? 1 : M, K, N) : 0;
  return v1 > v2 ? v1 : v2;      // either path may be selected at call time
}

extern "C" int tzk_small_linear_bwd(const float* x, int64_t ld_x, const float* w, const float* y, int64_t ld_y,
                                    const float* dy, int64_t ld_dy, int64_t M, int32_t K, int32_t N, int32_t relu,
                                    float* dx, int64_t ld_dx, float* dw, float* db, void* workspace,
                                    size_t workspace_bytes, tzk_stream_t stream) {
  int rc = small_linear_check("small_linear_bwd", M, K, N);
  if (rc) return rc;
  TZK_REQUIRE(M >= 1, "small_linear_bwd: empty batch");
  TZK_REQUIRE(x && w && dy && dw && (!relu || y), "small_linear_bwd: NULL argument");
  TZK_REQUIRE(ld_x >= K && ld_dy >= N && (!relu || ld_y >= N) && (!dx || ld_dx >= K),
              "small_linear_bwd: leading dimension smaller than the row");
  TZK_REQUIRE(workspace && workspace_bytes >= tzk_small_linear_bwd_workspace_bytes(M, K, N),
              "small_linear_bwd: workspace too small");
  if (use_bwd2(K, N)) {
    rc = tzk_bwd2::run(x, ld_x, w, y, ld_y, dy, ld_dy, M, K, N, relu, dx, ld_dx, dw, db, workspace, workspace_bytes,
                       as_stream(stream));
    TZK_REQUIRE(rc == 0, "small_linear_bwd: tzk_bwd2::run failed with code %d", rc);
    return 0;
  }
  const int KP = pad_pow(K, 16), NP = pad_pow(N, 4);
  const int grid = bwd_grid(M);
  const size_t smem = ((size_t)N * KP + (size_t)kTM * (K | 1) + (size_t)kTM * (N | 1)) * sizeof(float);
  float* partial = static_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
#define TZK_SLB(KP_, NP_)                                                                                          \
  do {                                                                                                             \
    if (smem > 48 * 1024)                                                                                          \
      cudaFuncSetAttribute(small_linear_bwd_kernel<KP_, NP_>, cudaFuncAttributeMaxDynamicSharedMemorySize,         \
                           (int)smem);                                                                             \
    small_linear_bwd_kernel<KP_, NP_><<<grid, kTM, smem, st>>>(x, ld_x, w, y, ld_y, dy, ld_dy, M, K, N, relu, dx,   \
                                                               ld_dx, partial);                                    \
  } while (0)
#define TZK_SLB_N(KP_)                      \
  switch (NP) {                             \
    case 4: TZK_SLB(KP_, 4); break;         \
    case 16: TZK_SLB(KP_, 16); break;       \
    case 32: TZK_SLB(KP_, 32); break;       \
    default: TZK_SLB(KP_, 64); break;       \
  }
  switch (KP) {
    case 16: TZK_SLB_N(16) break;
    case 32: TZK_SLB_N(32) break;
    default: TZK_SLB_N(64) break;
  }
#undef TZK_SLB_N
#undef TZK_SLB
  TZK_CHECK_LAUNCH("small_linear_bwd_kernel");
  const int total = N * K + N;
  small_linear_reduce_kernel<<<(total + 31) / 32, 256, 0, st>>>(partial, grid, N * K, N, dw, db);
  TZK_CHECK_LAUNCH("small_linear_reduce_kernel");
  return 0;
}

extern "C" size_t tzk_bce_logits_workspace_bytes(int64_t M) {
  return (size_t)ceil_div64(M < 1 ? 1 : M, kBceThreads * kBcePerThread) * sizeof(float);
}

extern "C" int tzk_bce_logits_fwd_bwd(const float* logits, const float* labels, int64_t M, float* loss,
                                      float* dlogits, void* workspace, size_t workspace_bytes,
                                      tzk_stream_t stream) {
  TZK_REQUIRE(M >= 1, "bce_logits: empty batch");
  TZK_REQUIRE(logits && labels && loss, "bce_logits: NULL argument");
  TZK_REQUIRE(workspace && workspace_bytes >= tzk_bce_logits_workspace_bytes(M), "bce_logits: workspace too small");
  const int64_t nb = ceil_div64(M, kBceThreads * kBcePerThread);
  TZK_REQUIRE(nb < ((int64_t)1 << 31), "bce_logits: batch too large");
  float* partial = static_cast<float*>(workspace);
  cudaStream_t st = as_stream(stream);
  const float inv_m = 1.0f / (float)M;
  bce_fwd_bwd_kernel<<<(unsigned)nb, kBceThreads, 0, st>>>(logits, labels, M, inv_m, dlogits, partial);
  TZK_CHECK_LAUNCH("bce_fwd_bwd_kernel");
  bce_final_kernel<<<1, 256, 0, st>>>(partial, (int)nb, inv_m, loss);
  TZK_CHECK_LAUNCH("bce_final_kernel");
  return 0;
}

// ---- the tower tail in one pass: last Perceptron (K -> N, ReLU) + Linear(N, 1) + mean BCE, forward and backward ---------
extern "C" size_t tzk_tower_tail_bce_workspace_bytes(int64_t M, int32_t K, int32_t N) {
  return tzk_tail::supported(K, N) ? tzk_tail::workspace_bytes(M < 1 ? 1 : M, K, N) : 0;
}

extern "C" int tzk_tower_tail_bce(const float* y1, int64_t ld_y, const float* w1, const float* b1, const float* w2,
                                  const float* b2, const float* labels, int64_t M, int32_t K, int32_t N, float* logits,
                                  float* dy1, int64_t ld_dy, float* colsum, float* out, void* workspace,
                                  size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(M >= 1, "tower_tail_bce: empty batch");
  TZK_REQUIRE(tzk_tail::supported(K, N), "tower_tail_bce: K=%d, N=%d must be in [1, 64]", K, N);
  TZK_REQUIRE(y1 && w1 && w2 && labels && logits && dy1 && out, "tower_tail_bce: NULL argument");
  TZK_REQUIRE(ld_y >= K && ld_dy >= K, "tower_tail_bce: leading dimension smaller than the row");
  TZK_REQUIRE(workspace && workspace_bytes >= tzk_tower_tail_bce_workspace_bytes(M, K, N),
              "tower_tail_bce: workspace too small");
  const int rc = tzk_tail::run(y1, ld_y, w1, b1, w2, b2, labels, M, K, N, logits, dy1, ld_dy, out, workspace,
                               workspace_bytes, as_stream(stream), colsum != nullptr);
  TZK_REQUIRE(rc == 0, "tower_tail_bce: tzk_tail::run failed with code %d", rc);
  if (colsum) {
    colsum_final(static_cast<const float*>(workspace) + tzk_tail::colsum_offset(M, K, N), tzk_tail::tiles(M), K, colsum,
                 as_stream(stream));
    TZK_CHECK_LAUNCH("colsum_final_kernel");
  }
  return 0;
}
