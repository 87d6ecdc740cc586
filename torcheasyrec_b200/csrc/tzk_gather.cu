// tzk_gather.cu — K4 pooled gather forward and K4-nobag sequence gather (sm_90a).
//
// HBM-bound byte mover.  Layout decisions (DESIGN.md §3):
//  * a CTA owns a tile of TB consecutive samples x all F features, so its output region
//    (TB rows x sum(D) floats) is one contiguous block of HBM written with full 128-B lines, while the
//    per-feature id runs it reads (ids are key-major) are TB*8-byte contiguous runs;
//  * a bag is served by G lanes (G*4 >= D for D <= 128): one 16-B vector load per lane per row, i.e.
//    a D=16 row is one 64-B request = two full 32-B sectors;
//  * U bags per lane-group are kept in flight (offsets -> id -> row is a 3-deep dependent chain, so
//    memory-level parallelism has to come from independent bags);
//  * feature descriptors are staged once per CTA in shared memory.
#include "tzk_common.cuh"

using namespace tzk;

namespace {

struct FeatDesc {
  int64_t w_off;
  int64_t rows;
  int32_t dim;
  int32_t col;
  int32_t pool;
  int32_t stride;  // elements between consecutive rows of the table (= dim, or 2 * dim for [weight row | state row] lines)
};

constexpr int kThreads = 256;
constexpr int kTB = 32;  // samples per tile
constexpr int kU = 8;    // bags in flight per lane group

// Two phases per (sample tile x feature chunk), both with many independent requests in flight:
//   A. every thread loads the bag bounds, then the first id, of its <= kItemsPerCta/256 bags into shared memory
//      (the per-sample index lists are staged once, coalesced: ids are key-major so a tile's ids of one feature
//      are one contiguous run);
//   B. every lane group walks its bags out of shared memory and keeps kU row loads in flight before it pools /
//      stores — the offsets -> id -> row dependency chain no longer serialises one bag at a time.
constexpr int kItemsPerCta = 1024;  // bags staged per chunk (20 KB of shared memory)

struct BagStage {
  int64_t start;   // position of the bag's first id
  int64_t id0;     // first id (valid when len > 0)
};

// WTD: weighted bags (per-sample weights psw[l], fbgemm's ..._forward_weighted): out = sum_l psw[l] * row(ids[l]) in list
// order as acc = fmaf(psw[l], row, acc), the first term as psw[l0] * row — with all-ones weights every operation is exact
// and the result has the bits of the unweighted lookup
template <int G, int VEC, typename WT, bool WTD>
__device__ __forceinline__ void
pooled_gather_body(const WT* __restrict__ weights, const int64_t* __restrict__ feat_w_off,
                   const int64_t* __restrict__ feat_rows, const int32_t* __restrict__ feat_dim,
                   const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                   const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets, int F, int B,
                   float* __restrict__ out, int64_t ld_out, const int32_t* __restrict__ feat_stride,
                   const float* __restrict__ psw) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FeatDesc* fd = reinterpret_cast<FeatDesc*>(smem_raw);
  BagStage* st = reinterpret_cast<BagStage*>(smem_raw + align16((size_t)F * sizeof(FeatDesc)));
  int32_t* st_len = reinterpret_cast<int32_t*>(st + kItemsPerCta);
  float* st_w = reinterpret_cast<float*>(st_len + kItemsPerCta);   // WTD: weight of the bag's first id
  for (int f = threadIdx.x; f < F; f += kThreads) {
    fd[f].w_off = feat_w_off[f];
    fd[f].rows = feat_rows[f];
    fd[f].dim = feat_dim[f];
    fd[f].col = feat_col[f];
    fd[f].pool = feat_pool[f];
    fd[f].stride = feat_stride ? feat_stride[f] : feat_dim[f];
  }
  __syncthreads();

  constexpr int NG = kThreads / G;  // lane groups per CTA
  constexpr int FC = kItemsPerCta / kTB;  // features per chunk
  const int g = threadIdx.x / G;
  const int lane = threadIdx.x % G;
  const int n_tiles = (B + kTB - 1) / kTB;
  const int n_chunks = (F + FC - 1) / FC;

  for (int work = blockIdx.x; work < n_tiles * n_chunks; work += gridDim.x) {
    const int tile = work / n_chunks, chunk = work - tile * n_chunks;
    const int b0 = tile * kTB;
    const int f0 = chunk * FC;
    const int nf = (F - f0) < FC ? (F - f0) : FC;
    const int items = nf * kTB;
    // ---- phase A --------------------------------------------------------------------------------------
    {
      constexpr int PT = kItemsPerCta / kThreads;  // items per thread
      int64_t s[PT];
      int32_t len[PT];
#pragma unroll
      for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + k * kThreads;
        const int b = b0 + (i % kTB);
        s[k] = 0;
        len[k] = -1;
        if (i < items && b < B) {
          const int64_t bag = (int64_t)(f0 + i / kTB) * B + b;
          s[k] = __ldg(offsets + bag);
          len[k] = (int32_t)(__ldg(offsets + bag + 1) - s[k]);
        }
      }
      int64_t id0[PT];
#pragma unroll
      for (int k = 0; k < PT; ++k) id0[k] = len[k] > 0 ? __ldg(ids + s[k]) : 0;
      float w0[PT];
      if constexpr (WTD) {
#pragma unroll
        for (int k = 0; k < PT; ++k) w0[k] = len[k] > 0 ? __ldg(psw + s[k]) : 0.f;
      }
#pragma unroll
      for (int k = 0; k < PT; ++k) {
        const int i = threadIdx.x + k * kThreads;
        if (i < items) {
          st[i].start = s[k];
          st[i].id0 = id0[k];
          st_len[i] = len[k];
          if constexpr (WTD) st_w[i] = w0[k];
        }
      }
    }
    __syncthreads();
    // ---- phase B --------------------------------------------------------------------------------------
    for (int i0 = g; i0 < items; i0 += NG * kU) {
      if (VEC == 4) {
        float4 acc[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int i = i0 + u * NG;
          acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (i < items && st_len[i] > 0) {
            const FeatDesc& d = fd[f0 + i / kTB];
            int64_t id = st[i].id0;
            if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
            if (lane * 4 < d.dim) acc[u] = ld_table_f4<WT>(weights + d.w_off + id * d.stride + lane * 4);
          }
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const int i = i0 + u * NG;
          if (i >= items) continue;
          const int L = st_len[i];
          if (L < 0) continue;  // sample beyond B
          const FeatDesc d = fd[f0 + i / kTB];
          float* orow = out + (int64_t)(b0 + (i % kTB)) * ld_out + d.col;
          for (int c = lane * 4; c < d.dim; c += G * 4) {
            float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
            if (L > 0) {
              if (c == lane * 4) {
                a = acc[u];
              } else {
                int64_t id = st[i].id0;
                if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
                a = ld_table_f4<WT>(weights + d.w_off + id * d.stride + c);
              }
              const int64_t s0 = st[i].start;
              if constexpr (WTD) {
                a = f4_scale(a, st_w[i]);
                for (int l = 1; l < L; ++l) {
                  int64_t idl = __ldg(ids + s0 + l);
                  const float wl = __ldg(psw + s0 + l);
                  if ((uint64_t)idl >= (uint64_t)d.rows) idl = 0;
                  const float4 r = ld_table_f4<WT>(weights + d.w_off + idl * d.stride + c);
                  a = make_float4(fmaf(wl, r.x, a.x), fmaf(wl, r.y, a.y), fmaf(wl, r.z, a.z), fmaf(wl, r.w, a.w));
                }
              } else {
                for (int l = 1; l < L; ++l) {
                  int64_t idl = __ldg(ids + s0 + l);
                  if ((uint64_t)idl >= (uint64_t)d.rows) idl = 0;
                  a = f4_add(a, ld_table_f4<WT>(weights + d.w_off + idl * d.stride + c));
                }
              }
              if (d.pool == TZK_POOL_MEAN) a = f4_scale(a, 1.0f / (float)L);
            }
            st_stream_f4(orow + c, a);
          }
        }
      } else {
#pragma unroll 1
        for (int u = 0; u < kU; ++u) {
          const int i = i0 + u * NG;
          if (i >= items) continue;
          const int L = st_len[i];
          if (L < 0) continue;
          const FeatDesc d = fd[f0 + i / kTB];
          float* orow = out + (int64_t)(b0 + (i % kTB)) * ld_out + d.col;
          const int64_t s0 = st[i].start;
          for (int c = lane; c < d.dim; c += G) {
            float acc = 0.f;
            if (L > 0) {
              int64_t id = st[i].id0;
              if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
              acc = ld_table_f1<WT>(weights + d.w_off + id * d.stride + c);
              if constexpr (WTD) {
                acc = st_w[i] * acc;
                for (int l = 1; l < L; ++l) {
                  int64_t idl = __ldg(ids + s0 + l);
                  const float wl = __ldg(psw + s0 + l);
                  if ((uint64_t)idl >= (uint64_t)d.rows) idl = 0;
                  acc = fmaf(wl, ld_table_f1<WT>(weights + d.w_off + idl * d.stride + c), acc);
                }
              } else {
                for (int l = 1; l < L; ++l) {
                  int64_t idl = __ldg(ids + s0 + l);
                  if ((uint64_t)idl >= (uint64_t)d.rows) idl = 0;
                  acc += ld_table_f1<WT>(weights + d.w_off + idl * d.stride + c);
                }
              }
              if (d.pool == TZK_POOL_MEAN) acc = acc * (1.0f / (float)L);
            }
            orow[c] = acc;
          }
        }
      }
    }
    __syncthreads();  // the stage buffer is reused by the next (tile, chunk)
  }
}

template <int G, int VEC, typename WT>
__global__ void __launch_bounds__(kThreads)
pooled_gather_fwd_kernel(const WT* __restrict__ weights, const int64_t* __restrict__ feat_w_off,
                         const int64_t* __restrict__ feat_rows, const int32_t* __restrict__ feat_dim,
                         const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                         const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets, int F, int B,
                         float* __restrict__ out, int64_t ld_out, const int32_t* __restrict__ feat_stride) {
  pooled_gather_body<G, VEC, WT, false>(weights, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool, ids, offsets, F,
                                        B, out, ld_out, feat_stride, nullptr);
}

template <int G, int VEC, typename WT>
__global__ void __launch_bounds__(kThreads, 2)     // (up to 128 registers: the default allocation spilled)
pooled_gather_fwd_weighted_kernel(const WT* __restrict__ weights, const int64_t* __restrict__ feat_w_off,
                                  const int64_t* __restrict__ feat_rows, const int32_t* __restrict__ feat_dim,
                                  const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                                  const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets, int F, int B,
                                  float* __restrict__ out, int64_t ld_out, const int32_t* __restrict__ feat_stride,
                                  const float* __restrict__ psw) {
  pooled_gather_body<G, VEC, WT, true>(weights, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool, ids, offsets, F,
                                       B, out, ld_out, feat_stride, psw);
}

// one lane group per id position; f found by binary search over the key boundaries offsets[f*B]
template <int G, int VEC, typename WT>
__global__ void __launch_bounds__(kThreads)
seq_gather_fwd_kernel(const WT* __restrict__ weights, const int64_t* __restrict__ feat_w_off,
                      const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ ids,
                      const int64_t* __restrict__ offsets, int F, int B, int D, int64_t nnz,
                      float* __restrict__ out, int row_stride) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int64_t* key_start = reinterpret_cast<int64_t*>(smem_raw);  // [F+1]
  int64_t* w_off = key_start + (F + 1);
  int64_t* rows = w_off + F;
  for (int f = threadIdx.x; f <= F; f += kThreads) key_start[f] = offsets[(int64_t)f * B];
  for (int f = threadIdx.x; f < F; f += kThreads) {
    w_off[f] = feat_w_off[f];
    rows[f] = feat_rows[f];
  }
  __syncthreads();
  constexpr int NG = kThreads / G;
  const int lane = threadIdx.x % G;
  const int64_t stride = (int64_t)gridDim.x * NG;
  for (int64_t l = (int64_t)blockIdx.x * NG + threadIdx.x / G; l < nnz; l += stride) {
    int lo = 0, hi = F;  // largest f with key_start[f] <= l
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (key_start[mid] <= l) lo = mid; else hi = mid;
    }
    int64_t id = __ldg(ids + l);
    if ((uint64_t)id >= (uint64_t)rows[lo]) id = 0;
    const WT* src = weights + w_off[lo] + id * row_stride;
    float* dst = out + l * D;
    for (int c = lane * VEC; c < D; c += G * VEC) {
      if (VEC == 4) st_stream_f4(dst + c, ld_table_f4<WT>(src + c));
      else dst[c] = ld_table_f1<WT>(src + c);
    }
  }
}

inline int pick_lanes(int max_dim, int vec) {
  int need = (max_dim + vec - 1) / vec;
  int g = 1;
  while (g < need && g < 32) g <<= 1;
  return g;
}

}  // namespace

#define TZK_DISPATCH_G(G_, VEC_, WT_, KERNEL, ...)                                               \
  switch (G_) {                                                                                   \
    case 1: KERNEL<1, VEC_, WT_><<<grid, kThreads, smem, st>>>(__VA_ARGS__); break;               \
    case 2: KERNEL<2, VEC_, WT_><<<grid, kThreads, smem, st>>>(__VA_ARGS__); break;               \
    case 4: KERNEL<4, VEC_, WT_><<<grid, kThreads, smem, st>>>(__VA_ARGS__); break;               \
    case 8: KERNEL<8, VEC_, WT_><<<grid, kThreads, smem, st>>>(__VA_ARGS__); break;               \
    case 16: KERNEL<16, VEC_, WT_><<<grid, kThreads, smem, st>>>(__VA_ARGS__); break;             \
    default: KERNEL<32, VEC_, WT_><<<grid, kThreads, smem, st>>>(__VA_ARGS__); break;             \
  }

template <int VEC, typename WT>
static void pooled_gather_weighted_allow_smem_v(int G, size_t smem) {
  auto k = G == 1 ? pooled_gather_fwd_weighted_kernel<1, VEC, WT> : G == 2 ? pooled_gather_fwd_weighted_kernel<2, VEC, WT>
         : G == 4 ? pooled_gather_fwd_weighted_kernel<4, VEC, WT> : G == 8 ? pooled_gather_fwd_weighted_kernel<8, VEC, WT>
         : G == 16 ? pooled_gather_fwd_weighted_kernel<16, VEC, WT> : pooled_gather_fwd_weighted_kernel<32, VEC, WT>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}
template <typename WT>
static void pooled_gather_weighted_allow_smem(int G, int vec, size_t smem) {
  if (vec == 4) pooled_gather_weighted_allow_smem_v<4, WT>(G, smem);
  else pooled_gather_weighted_allow_smem_v<1, WT>(G, smem);
}

template <typename WT>
static int pooled_gather_fwd_impl(const WT* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                                  const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_pool,
                                  const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t max_dim,
                                  int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream,
                                  const int32_t* feat_stride = nullptr, const float* psw = nullptr) {
  TZK_REQUIRE(F >= 0 && B >= 0, "pooled_gather_fwd: negative F/B");
  if (F == 0 || B == 0) return 0;
  TZK_REQUIRE(weights && feat_w_off && feat_rows && feat_dim && feat_col && feat_pool && offsets && out,
              "pooled_gather_fwd: NULL argument");
  TZK_REQUIRE(max_dim >= 1, "pooled_gather_fwd: max_dim < 1");
  TZK_REQUIRE(F <= 4096, "pooled_gather_fwd: F=%d > 4096 keys per collection", F);
  const int vec = (vec_ok && ((uintptr_t)weights % (4 * sizeof(WT)) == 0) && ((uintptr_t)out % 16 == 0) &&
                   (ld_out % 4 == 0)) ? 4 : 1;
  const int G = pick_lanes(max_dim, vec);
  cudaStream_t st = as_stream(stream);
  const int n_tiles = (B + kTB - 1) / kTB;
  const int n_work = n_tiles * ((F + kItemsPerCta / kTB - 1) / (kItemsPerCta / kTB));
  int grid = n_work < kSmCountH100 * 8 ? n_work : kSmCountH100 * 8;
  size_t smem = align16((size_t)F * sizeof(FeatDesc)) + (size_t)kItemsPerCta * (sizeof(BagStage) + sizeof(int32_t));
  if (psw) {      // + the first weight of every staged bag; above 48 KB the weighted kernel opts in
    smem += (size_t)kItemsPerCta * sizeof(float);
    if (smem > 48 * 1024) pooled_gather_weighted_allow_smem<WT>(G, vec, smem);
  }
  TZK_REQUIRE(psw || smem <= 48 * 1024, "pooled_gather_fwd: F=%d keys need %zu B of shared memory (> 48 KB)", F, smem);
  if (psw) {
    if (vec == 4) {
      TZK_DISPATCH_G(G, 4, WT, pooled_gather_fwd_weighted_kernel, weights, feat_w_off, feat_rows, feat_dim, feat_col,
                     feat_pool, ids, offsets, F, B, out, ld_out, feat_stride, psw)
    } else {
      TZK_DISPATCH_G(G, 1, WT, pooled_gather_fwd_weighted_kernel, weights, feat_w_off, feat_rows, feat_dim, feat_col,
                     feat_pool, ids, offsets, F, B, out, ld_out, feat_stride, psw)
    }
  } else if (vec == 4) {
    TZK_DISPATCH_G(G, 4, WT, pooled_gather_fwd_kernel, weights, feat_w_off, feat_rows, feat_dim, feat_col,
                   feat_pool, ids, offsets, F, B, out, ld_out, feat_stride)
  } else {
    TZK_DISPATCH_G(G, 1, WT, pooled_gather_fwd_kernel, weights, feat_w_off, feat_rows, feat_dim, feat_col,
                   feat_pool, ids, offsets, F, B, out, ld_out, feat_stride)
  }
  TZK_CHECK_LAUNCH("pooled_gather_fwd");
  return 0;
}

extern "C" int tzk_pooled_gather_fwd(const float* weights, const int64_t* feat_w_off,
                                     const int64_t* feat_rows, const int32_t* feat_dim,
                                     const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                     const int64_t* offsets, int32_t F, int32_t B, int32_t max_dim,
                                     int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream) {
  return pooled_gather_fwd_impl<float>(weights, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool, ids, offsets, F,
                                       B, max_dim, vec_ok, out, ld_out, stream);
}

// FP16 tables (EmbeddingBagConfig.data_type = FP16): the arena holds halfs, pooling and the output stay fp32
extern "C" int tzk_pooled_gather_fwd_f16(const void* weights, const int64_t* feat_w_off,
                                         const int64_t* feat_rows, const int32_t* feat_dim,
                                         const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                         const int64_t* offsets, int32_t F, int32_t B, int32_t max_dim,
                                         int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream) {
  return pooled_gather_fwd_impl<__half>(static_cast<const __half*>(weights), feat_w_off, feat_rows, feat_dim, feat_col,
                                        feat_pool, ids, offsets, F, B, max_dim, vec_ok, out, ld_out, stream);
}

// the kernel stages 3 F + 1 int64 in shared memory: 49 160 B at F = 2048, above the 48 KB a launch gets by default
template <int VEC, typename WT>
static void seq_gather_allow_smem(int G, size_t smem) {
  if (smem <= 48 * 1024) return;
  auto k = G == 1 ? seq_gather_fwd_kernel<1, VEC, WT> : G == 2 ? seq_gather_fwd_kernel<2, VEC, WT>
         : G == 4 ? seq_gather_fwd_kernel<4, VEC, WT> : G == 8 ? seq_gather_fwd_kernel<8, VEC, WT>
         : G == 16 ? seq_gather_fwd_kernel<16, VEC, WT> : seq_gather_fwd_kernel<32, VEC, WT>;
  cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
}

template <typename WT>
static int seq_gather_fwd_impl(const WT* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                               const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t D, int64_t nnz,
                               float* out, tzk_stream_t stream, int32_t row_stride = 0) {
  TZK_REQUIRE(F >= 0 && B >= 0 && nnz >= 0 && D >= 1, "seq_gather_fwd: bad sizes");
  if (row_stride == 0) row_stride = D;
  TZK_REQUIRE(row_stride >= D && (D % 4 != 0 || row_stride % 4 == 0), "seq_gather_fwd: bad row stride %d for D=%d", row_stride, D);
  if (F == 0 || nnz == 0) return 0;
  TZK_REQUIRE(weights && feat_w_off && feat_rows && ids && offsets && out, "seq_gather_fwd: NULL argument");
  TZK_REQUIRE(F <= 2048, "seq_gather_fwd: F=%d > 2048", F);
  const int vec = (D % 4 == 0 && ((uintptr_t)weights % (4 * sizeof(WT)) == 0) && ((uintptr_t)out % 16 == 0)) ? 4 : 1;
  const int G = pick_lanes(D, vec);
  cudaStream_t st = as_stream(stream);
  const int NG = kThreads / G;
  int64_t blocks = ceil_div64(nnz, NG);
  int grid = blocks < kSmCountH100 * 16 ? (int)blocks : kSmCountH100 * 16;
  size_t smem = (size_t)(3 * F + 1) * sizeof(int64_t);
  if (vec == 4) seq_gather_allow_smem<4, WT>(G, smem); else seq_gather_allow_smem<1, WT>(G, smem);
  if (vec == 4) {
    TZK_DISPATCH_G(G, 4, WT, seq_gather_fwd_kernel, weights, feat_w_off, feat_rows, ids, offsets, F, B, D, nnz, out, row_stride)
  } else {
    TZK_DISPATCH_G(G, 1, WT, seq_gather_fwd_kernel, weights, feat_w_off, feat_rows, ids, offsets, F, B, D, nnz, out, row_stride)
  }
  TZK_CHECK_LAUNCH("seq_gather_fwd");
  return 0;
}

extern "C" int tzk_seq_gather_fwd(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                                  const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B,
                                  int32_t D, int64_t nnz, float* out, tzk_stream_t stream) {
  return seq_gather_fwd_impl<float>(weights, feat_w_off, feat_rows, ids, offsets, F, B, D, nnz, out, stream);
}

extern "C" int tzk_seq_gather_fwd_f16(const void* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                                      const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B,
                                      int32_t D, int64_t nnz, float* out, tzk_stream_t stream) {
  return seq_gather_fwd_impl<__half>(static_cast<const __half*>(weights), feat_w_off, feat_rows, ids, offsets, F, B, D,
                                     nnz, out, stream);
}

// Strided tables: consecutive rows of feature f's table are feat_stride[f] (>= D_f) elements apart — the interleaved
// [weight row | optimizer-state row] layout (tzk_opt_args.interleaved) keeps a row and its Adagrad accumulator in one
// 128-B line for D = 16, so the update writes whole lines.  feat_stride == NULL: dense rows.
extern "C" int tzk_pooled_gather_fwd_strided(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                                             const int32_t* feat_dim, const int32_t* feat_stride,
                                             const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                             const int64_t* offsets, int32_t F, int32_t B, int32_t max_dim,
                                             int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream) {
  return pooled_gather_fwd_impl<float>(weights, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool, ids, offsets, F,
                                       B, max_dim, vec_ok, out, ld_out, stream, feat_stride);
}

extern "C" int tzk_seq_gather_fwd_strided(const float* weights, const int64_t* feat_w_off, const int64_t* feat_rows,
                                          const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t D,
                                          int32_t row_stride, int64_t nnz, float* out, tzk_stream_t stream) {
  return seq_gather_fwd_impl<float>(weights, feat_w_off, feat_rows, ids, offsets, F, B, D, nnz, out, stream, row_stride);
}

// Weighted bags ([EXT] fbgemm TBE split_embedding_codegen_forward_weighted, per_sample_weights of the sharded lookup): one
// entry point for the three arena formats — weights_f16 selects halfs, feat_stride (nullable) strided fp32 rows.
extern "C" int tzk_pooled_gather_fwd_weighted(const void* weights, int32_t weights_f16, const int64_t* feat_w_off,
                                              const int64_t* feat_rows, const int32_t* feat_dim,
                                              const int32_t* feat_stride, const int32_t* feat_col,
                                              const int32_t* feat_pool, const int64_t* ids, const int64_t* offsets,
                                              const float* per_sample_weights, int32_t F, int32_t B, int32_t max_dim,
                                              int32_t vec_ok, float* out, int64_t ld_out, tzk_stream_t stream) {
  TZK_REQUIRE(F == 0 || B == 0 || per_sample_weights != nullptr,
              "pooled_gather_fwd_weighted: per_sample_weights is NULL");
  if (weights_f16) {
    TZK_REQUIRE(feat_stride == nullptr, "pooled_gather_fwd_weighted: strided (interleaved) tables are fp32");
    return pooled_gather_fwd_impl<__half>(static_cast<const __half*>(weights), feat_w_off, feat_rows, feat_dim, feat_col,
                                          feat_pool, ids, offsets, F, B, max_dim, vec_ok, out, ld_out, stream, nullptr,
                                          per_sample_weights);
  }
  return pooled_gather_fwd_impl<float>(static_cast<const float*>(weights), feat_w_off, feat_rows, feat_dim, feat_col,
                                       feat_pool, ids, offsets, F, B, max_dim, vec_ok, out, ld_out, stream, feat_stride,
                                       per_sample_weights);
}
