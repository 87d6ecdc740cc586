// tzk_peer.cu — the sharded sparse step over peer memory (part of libtzk.so; exchange="peer" in shard_model).
//
// The sharded sparse step without a collective call (DESIGN.md §6).  Every rank's table arena, its wire buffers and its
// published gradient live in symmetric (peer-mapped) memory of the NVSwitch domain, and the kernels read them in place:
//
//   forward   peer_pooled_gather_fwd_kernel / peer_seq_gather_fwd_kernel: the REQUESTER's gather reads each embedding
//             row straight from the owning rank's arena (owner = feat_owner + id / block, the same rule as tzk_dist.cu's
//             dest_of) — no id exchange, no row exchange, no staging, any bag length, same bits as the unsharded
//             gather.  (Replaces: bucketize -> ids all-to-all -> owner gather -> rows all-to-all -> local pooling; the
//             reference's KJTAllToAll + lookup + PooledEmbeddingsAllToAll, SURVEY.md §8 A3 / App. A.5-A.8.)
//   backward  source side (tzk_peer_bucketize, on a side stream during the forward pass): a stable multi-split of the
//             rank's ids by destination into its OWN wire buffers — per destination, in (feature, bag, position)
//             order: wire_key = the owner-local linearised (table,row) key, wire_idx = bag (pooled) / id position
//             (sequence) — plus the per-destination counts.  No [W*F*B] lengths array, no scan over it: per-tile
//             destination histograms (1024 bags a tile), one scan per destination over the tiles, one scatter pass.
//             owner side (tzk_bwd.cu: tzk_fused_bwd_sort_peer / tzk_fused_bwd_apply_peer): after a barrier the owner
//             reads, per source, its chunk of keys / indices straight into the radix sort's input (coalesced NVLink
//             reads), sorts, and the run kernels fetch every 64-B gradient slice from the SOURCE's published gradient
//             buffer in place.  No gradient expansion, no gradient all-to-all, no staging copy.
//   barrier   peer_barrier_kernel: one flag per (src, dst) pair in symmetric memory, st.release.sys / ld.acquire.sys,
//             epoch kept on the device so the whole step replays as one CUDA graph.  Barrier sites that may run
//             concurrently (different streams) use different flag arrays / epochs.
//   dense     peer_allreduce_mean_kernel: the replicated dense gradients, summed in rank order straight out of every
//             rank's published flat buffer (bit-identical on every rank; replaces the DDP all-reduce, SURVEY C5).
//   weighted  (per-sample weights of weighted id features; pooled, push transport) the weights never leave the sample's
//             rank: the gather pools w * row, the scatter records each wire slot's weight in a local buffer, the push
//             sends w * g (/ L).  Each weighted kernel is the unweighted one's body with a compile-time switch.
//   FP16      (data_type = FP16 tables) the arenas and the mirror hold halfs; the gathers widen every row to fp32 and pool
//             exactly as the unsharded f16 lookups do, the mirror refresh copies the halfs' bits.  Gradients on the wire,
//             the partial sums and the optimizer state stay fp32 (the owner's update rounds the row back, tzk_bwd.cu).
//             Each _f16 kernel is the fp32 one's body instantiated for the table type TT = __half.
//
// This file compiles for the host too (TZK_CPU_SHIM, tests/test_peer_exchange_model.py runs the kernels' source on
// std::threads), so it uses plain CUDA + warp shuffles only; the barrier (PTX) is excluded from that build.
#ifdef TZK_CPU_SHIM
#include "cuda_cpu_shim.h"
#include "half_cpu_shim.h"
#else
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include "tzk_launch.cuh"
#endif
#include <stdint.h>
#include <stdlib.h>

#include <type_traits>

namespace {

constexpr int kMaxPeers = 16;
constexpr int kThreads = 256;
struct Peers { unsigned long long p[kMaxPeers]; };

struct FeatDesc {
  int64_t rows;    // global rows of the table (ids are clamped like the unsharded gather: out of range -> row 0)
  int64_t block;   // row-wise block (>= rows for table-wise)
  int32_t owner;   // first owner rank
  int32_t dim;
  int32_t col;
  int32_t pool;    // 0 sum, 1 mean
};

__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }

// Rows that another GPU rewrote in the previous step: a coherent load (not ld.global.nc) that does not allocate in L1.
__device__ __forceinline__ float4 ld_peer_f4(const float* p) {
#ifdef TZK_CPU_SHIM
  return *reinterpret_cast<const float4*>(p);
#else
  float4 r;
  asm("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
#endif
}

// FP16 tables: ld_peer_f4's half-width twin — 4 halfs (8 B) with the same coherent no-L1-allocate load, widened to fp32
__device__ __forceinline__ float4 ld_peer_h4(const __half* p) {
#ifdef TZK_CPU_SHIM
  return make_float4(__half2float(p[0]), __half2float(p[1]), __half2float(p[2]), __half2float(p[3]));
#else
  unsigned int a, b;
  asm("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(a), "=r"(b) : "l"(p));
  const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&a));
  const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&b));
  return make_float4(lo.x, lo.y, hi.x, hi.y);
#endif
}
template <typename TT> __device__ __forceinline__ float4 ld_peer_row4(const TT* p);
template <> __device__ __forceinline__ float4 ld_peer_row4<float>(const float* p) { return ld_peer_f4(p); }
template <> __device__ __forceinline__ float4 ld_peer_row4<__half>(const __half* p) { return ld_peer_h4(p); }

// 4 table elements moved as one vector, bits unchanged (mirror refresh): 16 B of floats, 8 B of halfs
struct __align__(8) H4 { uint32_t a, b; };
template <typename TT> struct Unit4;
template <> struct Unit4<float> {
  using V = float4;
  __device__ __forceinline__ static V ld(const float* p) { return ld_peer_f4(p); }
};
template <> struct Unit4<__half> {
  using V = H4;
  __device__ __forceinline__ static V ld(const __half* p) {
#ifdef TZK_CPU_SHIM
    return *reinterpret_cast<const H4*>(p);
#else
    H4 r;
    asm("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.a), "=r"(r.b) : "l"(p));
    return r;
#endif
  }
};

// owner rank and owner-local row of a (clamped, non-negative) id — tzk_dist.cu's dest_of.  The quotient is below W <= 16:
// a float estimate plus one exact fix-up replaces the 64-bit integer division (~100 instructions on the SM, per row,
// which made the requester-side gather instruction-bound).
__device__ __forceinline__ int owner_of(int64_t id, int64_t block, int owner, int W, int64_t* local) {
#ifdef TZK_CPU_SHIM
  int64_t q = id / block;
#else
  int64_t q = (int64_t)__fdividef((float)id, (float)block);
  if (q * block > id) --q;
  else if ((q + 1) * block <= id) ++q;
#endif
  int64_t r = owner + q;
  if (r >= W) { q -= r - (W - 1); r = W - 1; }
  *local = id - q * block;
  return (int)r;
}

// ---- forward: requester-side gather over peer memory ------------------------------------------------------------
// A CTA owns 32 consecutive samples x all features (its output block is contiguous); a bag is served by G lanes,
// one 16-B load per lane per row; U bags per lane group are in flight because a remote row costs an NVLink round trip.
// WTD: weighted bags (per-sample weights psw[l], the sample's own rank holds them): out = sum_l psw[l] * row(ids[l]) in
// list order as acc = fmaf(psw[l], row, acc), the first term psw[l0] * row, MEAN then * 1/L — the arithmetic of
// tzk_gather.cu's pooled_gather_fwd_weighted_kernel, so the bits equal the unsharded weighted lookup's.
// TT: the table element (float, or __half for FP16 tables: arena and mirror rows are halfs, widened exactly on load, so
// the sums are the unsharded f16 lookup's).
template <int G, bool WTD, typename TT = float>
__device__ __forceinline__ void
peer_pooled_gather_body(const Peers& tables, const int64_t* __restrict__ rf_w_off, const int64_t* __restrict__ feat_rows,
                        const int64_t* __restrict__ feat_block, const int32_t* __restrict__ feat_owner,
                        const int32_t* __restrict__ feat_dim, const int32_t* __restrict__ feat_col,
                        const int32_t* __restrict__ feat_pool, const int64_t* __restrict__ ids,
                        const int64_t* __restrict__ offsets, int F, int B, int W, float* __restrict__ out,
                        int64_t ld_out, const TT* __restrict__ mirror, const int64_t* __restrict__ feat_mirror_off,
                        const int32_t* __restrict__ feat_sel, int n_sel, const float* __restrict__ psw) {
  // feat_sel (nullable): this launch serves only the listed features (e.g. the mirrored ones, or the ones whose rows
  // cross NVLink — two launches on two streams overlap the local and the remote half of the lookup)
  constexpr int NG = kThreads / G, TB = 32, U = 8;
  TZK_DYN_SMEM(unsigned char, smem_raw);
  FeatDesc* fd = reinterpret_cast<FeatDesc*>(smem_raw);
  int64_t* w_off = reinterpret_cast<int64_t*>(fd + F);                      // [W * F] arena offsets per (rank, feature)
  unsigned long long* base = reinterpret_cast<unsigned long long*>(w_off + (size_t)W * F);   // [W]
  int64_t* m_off = reinterpret_cast<int64_t*>(base + W);                    // [F] offset in the local mirror, or -1
  int32_t* sel = reinterpret_cast<int32_t*>(m_off + F);                     // [F] features of this launch
  const int nF = feat_sel ? n_sel : F;
  for (int f = threadIdx.x; f < nF; f += kThreads) sel[f] = feat_sel ? feat_sel[f] : f;
  for (int f = threadIdx.x; f < F; f += kThreads) m_off[f] = (mirror && feat_mirror_off) ? feat_mirror_off[f] : -1;
  for (int f = threadIdx.x; f < F; f += kThreads) {
    fd[f].rows = feat_rows[f];
    fd[f].block = feat_block[f];
    fd[f].owner = feat_owner ? feat_owner[f] : 0;
    fd[f].dim = feat_dim[f];
    fd[f].col = feat_col[f];
    fd[f].pool = feat_pool[f];
  }
  for (int i = threadIdx.x; i < W * F; i += kThreads) w_off[i] = rf_w_off[i];
  if (threadIdx.x < W) base[threadIdx.x] = tables.p[threadIdx.x];
  __syncthreads();

  auto row_ptr = [&](int f, const FeatDesc& d, int64_t id) -> const TT* {
    if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
    if (m_off[f] >= 0) return mirror + m_off[f] + id * d.dim;     // small table: this step's local copy of all its rows
    int64_t loc;
    const int r = owner_of(id, d.block, d.owner, W, &loc);
    return reinterpret_cast<const TT*>(base[r]) + w_off[r * F + f] + loc * d.dim;
  };

  const int g = threadIdx.x / G, lane = threadIdx.x % G;
  const int n_tiles = (B + TB - 1) / TB;
  const int items = nF * TB;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int b0 = tile * TB;
    for (int i0 = g; i0 < items; i0 += NG * U) {
      int32_t s[U];                       // nnz < 2^31
      int32_t len[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = i0 + u * NG, b = b0 + (i % TB);
        s[u] = 0;
        len[u] = -1;
        if (i < items && b < B) {
          const int64_t bag = (int64_t)sel[i / TB] * B + b;
          s[u] = (int32_t)__ldg(offsets + bag);
          len[u] = (int32_t)__ldg(offsets + bag + 1) - s[u];
        }
      }
      int64_t id0[U];
#pragma unroll
      for (int u = 0; u < U; ++u) id0[u] = len[u] > 0 ? __ldg(ids + s[u]) : 0;
      float w0[U];                        // WTD: the first weight of each bag, loaded next to its first id
      if constexpr (WTD) {
#pragma unroll
        for (int u = 0; u < U; ++u) w0[u] = len[u] > 0 ? __ldg(psw + s[u]) : 0.f;
      }
      float4 acc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (len[u] > 0) {
          const int f = sel[(i0 + u * NG) / TB];
          const FeatDesc& d = fd[f];
          if (lane * 4 < d.dim) acc[u] = ld_peer_row4<TT>(row_ptr(f, d, id0[u]) + lane * 4);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (len[u] < 0) continue;
        const int i = i0 + u * NG, f = sel[i / TB];
        const FeatDesc d = fd[f];
        float* orow = out + (int64_t)(b0 + (i % TB)) * ld_out + d.col;
        for (int c = lane * 4; c < d.dim; c += G * 4) {
          float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
          if (len[u] > 0) {
            a = (c == lane * 4) ? acc[u] : ld_peer_row4<TT>(row_ptr(f, d, id0[u]) + c);
            if constexpr (WTD) {
              a = make_float4(a.x * w0[u], a.y * w0[u], a.z * w0[u], a.w * w0[u]);
              for (int l = 1; l < len[u]; ++l) {
                const float wl = __ldg(psw + s[u] + l);
                const float4 r = ld_peer_row4<TT>(row_ptr(f, d, __ldg(ids + s[u] + l)) + c);
                a = make_float4(fmaf(wl, r.x, a.x), fmaf(wl, r.y, a.y), fmaf(wl, r.z, a.z), fmaf(wl, r.w, a.w));
              }
            } else {
              for (int l = 1; l < len[u]; ++l)
                a = f4_add(a, ld_peer_row4<TT>(row_ptr(f, d, __ldg(ids + s[u] + l)) + c));
            }
            if (d.pool == 1) {
              const float inv = 1.0f / (float)len[u];
              a = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
            }
          }
          *reinterpret_cast<float4*>(orow + c) = a;
        }
      }
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads)
peer_pooled_gather_fwd_kernel(const __grid_constant__ Peers tables, const int64_t* __restrict__ rf_w_off, const int64_t* __restrict__ feat_rows,
                              const int64_t* __restrict__ feat_block, const int32_t* __restrict__ feat_owner,
                              const int32_t* __restrict__ feat_dim, const int32_t* __restrict__ feat_col,
                              const int32_t* __restrict__ feat_pool, const int64_t* __restrict__ ids,
                              const int64_t* __restrict__ offsets, int F, int B, int W, float* __restrict__ out,
                              int64_t ld_out, const float* __restrict__ mirror,
                              const int64_t* __restrict__ feat_mirror_off, const int32_t* __restrict__ feat_sel,
                              int n_sel) {
  peer_pooled_gather_body<G, false>(tables, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                    ids, offsets, F, B, W, out, ld_out, mirror, feat_mirror_off, feat_sel, n_sel,
                                    nullptr);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
peer_pooled_gather_fwd_weighted_kernel(const __grid_constant__ Peers tables, const int64_t* __restrict__ rf_w_off,
                                       const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                                       const int32_t* __restrict__ feat_owner, const int32_t* __restrict__ feat_dim,
                                       const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                                       const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets, int F,
                                       int B, int W, float* __restrict__ out, int64_t ld_out,
                                       const float* __restrict__ mirror, const int64_t* __restrict__ feat_mirror_off,
                                       const int32_t* __restrict__ feat_sel, int n_sel, const float* __restrict__ psw) {
  peer_pooled_gather_body<G, true>(tables, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                   ids, offsets, F, B, W, out, ld_out, mirror, feat_mirror_off, feat_sel, n_sel, psw);
}

// FP16 tables (arenas and mirror of halfs), plain (WTD = false, psw unused) and weighted bags
template <int G, bool WTD>
__global__ void __launch_bounds__(kThreads)
peer_pooled_gather_fwd_f16_kernel(const __grid_constant__ Peers tables, const int64_t* __restrict__ rf_w_off,
                                  const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                                  const int32_t* __restrict__ feat_owner, const int32_t* __restrict__ feat_dim,
                                  const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                                  const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets, int F, int B,
                                  int W, float* __restrict__ out, int64_t ld_out, const __half* __restrict__ mirror,
                                  const int64_t* __restrict__ feat_mirror_off, const int32_t* __restrict__ feat_sel,
                                  int n_sel, const float* __restrict__ psw) {
  peer_pooled_gather_body<G, WTD, __half>(tables, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col,
                                          feat_pool, ids, offsets, F, B, W, out, ld_out, mirror, feat_mirror_off,
                                          feat_sel, n_sel, psw);
}

// un-pooled (sequence) lookup: one lane group per id position, feature by binary search over the segment starts
template <int G, typename TT>
__device__ __forceinline__ void
peer_seq_gather_body(const Peers& tables, const int64_t* __restrict__ rf_w_off, const int64_t* __restrict__ feat_rows,
                     const int64_t* __restrict__ feat_block, const int32_t* __restrict__ feat_owner,
                     const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets, int F, int B, int W, int D,
                     int64_t nnz, float* __restrict__ out, const TT* __restrict__ mirror,
                     const int64_t* __restrict__ feat_mirror_off) {
  constexpr int NG = kThreads / G, U = 4;
  TZK_DYN_SMEM(unsigned char, smem_raw);
  int64_t* seg = reinterpret_cast<int64_t*>(smem_raw);   // [F + 1] first id position of every feature
  int64_t* rows = seg + (F + 1);                          // [F]
  int64_t* block = rows + F;                              // [F]
  int64_t* w_off = block + F;                             // [W * F]
  unsigned long long* base = reinterpret_cast<unsigned long long*>(w_off + (size_t)W * F);   // [W]
  int32_t* owner = reinterpret_cast<int32_t*>(base + W);  // [F]
  for (int f = threadIdx.x; f <= F; f += kThreads) seg[f] = offsets[(int64_t)f * B];
  for (int f = threadIdx.x; f < F; f += kThreads) {
    rows[f] = feat_rows[f];
    block[f] = feat_block[f];
    owner[f] = feat_owner ? feat_owner[f] : 0;
  }
  for (int i = threadIdx.x; i < W * F; i += kThreads) w_off[i] = rf_w_off[i];
  if (threadIdx.x < W) base[threadIdx.x] = tables.p[threadIdx.x];
  __syncthreads();
  const int lane = threadIdx.x % G;
  const int64_t stride = (int64_t)gridDim.x * NG * U;
  for (int64_t l0 = ((int64_t)blockIdx.x * NG + threadIdx.x / G) * U; l0 < nnz; l0 += stride) {
    const TT* src[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int64_t l = l0 + u;
      src[u] = nullptr;
      if (l < nnz) {
        int lo = 0, hi = F;
        while (hi - lo > 1) {
          const int mid = (lo + hi) >> 1;
          if (seg[mid] <= l) lo = mid; else hi = mid;
        }
        int64_t id = __ldg(ids + l);
        if ((uint64_t)id >= (uint64_t)rows[lo]) id = 0;
        const int64_t mo = (mirror && feat_mirror_off) ? __ldg(feat_mirror_off + lo) : -1;
        if (mo >= 0) {
          src[u] = mirror + mo + id * D;
        } else {
          int64_t loc;
          const int r = owner_of(id, block[lo], owner[lo], W, &loc);
          src[u] = reinterpret_cast<const TT*>(base[r]) + w_off[r * F + lo] + loc * D;
        }
      }
    }
    for (int c = lane * 4; c < D; c += G * 4) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = src[u] ? ld_peer_row4<TT>(src[u] + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (src[u]) *reinterpret_cast<float4*>(out + (l0 + u) * D + c) = v[u];
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads)
peer_seq_gather_fwd_kernel(const __grid_constant__ Peers tables, const int64_t* __restrict__ rf_w_off,
                           const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                           const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ ids,
                           const int64_t* __restrict__ offsets, int F, int B, int W, int D, int64_t nnz,
                           float* __restrict__ out, const float* __restrict__ mirror,
                           const int64_t* __restrict__ feat_mirror_off) {
  peer_seq_gather_body<G, float>(tables, rf_w_off, feat_rows, feat_block, feat_owner, ids, offsets, F, B, W, D, nnz, out,
                                 mirror, feat_mirror_off);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
peer_seq_gather_fwd_f16_kernel(const __grid_constant__ Peers tables, const int64_t* __restrict__ rf_w_off,
                               const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                               const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ ids,
                               const int64_t* __restrict__ offsets, int F, int B, int W, int D, int64_t nnz,
                               float* __restrict__ out, const __half* __restrict__ mirror,
                               const int64_t* __restrict__ feat_mirror_off) {
  peer_seq_gather_body<G, __half>(tables, rf_w_off, feat_rows, feat_block, feat_owner, ids, offsets, F, B, W, D, nnz,
                                  out, mirror, feat_mirror_off);
}

// ---- per-step local copy of the small tables ------------------------------------------------------------------------------
// Most lookups of a Criteo-like workload hit tables of a few thousand rows (18 of 26 features, 69 % of the ids): their
// shards are a few MB in total, so every rank copies them from the owners once per step — long sequential NVLink reads
// — and its gather reads those features from local memory; only the big tables' rows cross NVLink as
// random 64-B reads.  Segment s: n[s] elements from rank r[s]'s arena at src[s] to mirror + dst[s].
// TT: the table element; the copy moves 4 elements per vector (16 B of floats, 8 B of halfs — table starts and row
// sizes are multiples of 4 elements, which for halfs is 8-B but not always 16-B alignment) and keeps their bits.
template <typename TT>
__device__ __forceinline__ void
peer_mirror_refresh_simple_body(const Peers& tables, const int32_t* __restrict__ seg_rank,
                                const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                                const int64_t* __restrict__ seg_n, int n_seg, TT* __restrict__ mirror) {
  using V = typename Unit4<TT>::V;
  for (int s = blockIdx.y; s < n_seg; s += gridDim.y) {
    const TT* src = reinterpret_cast<const TT*>(tables.p[__ldg(seg_rank + s)]) + __ldg(seg_src + s);
    TT* dst = mirror + __ldg(seg_dst + s);
    const int64_t n4 = __ldg(seg_n + s) >> 2;       // table starts and row sizes are multiples of 4 elements
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
      reinterpret_cast<V*>(dst)[i] = Unit4<TT>::ld(src + i * 4);
  }
}

__global__ void __launch_bounds__(kThreads)
peer_mirror_refresh_simple_kernel(const __grid_constant__ Peers tables, const int32_t* __restrict__ seg_rank,
                                  const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                                  const int64_t* __restrict__ seg_n, int n_seg, float* __restrict__ mirror) {
  peer_mirror_refresh_simple_body<float>(tables, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
}

__global__ void __launch_bounds__(kThreads)
peer_mirror_refresh_simple_f16_kernel(const __grid_constant__ Peers tables, const int32_t* __restrict__ seg_rank,
                                      const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                                      const int64_t* __restrict__ seg_n, int n_seg, __half* __restrict__ mirror) {
  peer_mirror_refresh_simple_body<__half>(tables, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
}

// The segments cut into chunks of kMirrorChunk floats, chunks dealt round-robin to the CTAs: every thread has
// kMirrorChunk / (4 * kThreads) independent 16-B NVLink reads in flight (one load in flight per thread — the simple kernel —
// pays the NVLink round trip once per 16 B and thread).  n_seg <= kMirrorMaxSeg.
constexpr int kMirrorChunk = 4096;
constexpr int kMirrorMaxSeg = 4 * kThreads;
template <typename TT>
__device__ __forceinline__ void
peer_mirror_refresh_body(const Peers& tables, const int32_t* __restrict__ seg_rank, const int64_t* __restrict__ seg_src,
                         const int64_t* __restrict__ seg_dst, const int64_t* __restrict__ seg_n, int n_seg,
                         TT* __restrict__ mirror) {
  using V = typename Unit4<TT>::V;
  TZK_DYN_SMEM(int32_t, pre);                     // [kMirrorMaxSeg + 1] chunks before segment s
  int32_t* part = pre + kMirrorMaxSeg + 1;        // [kThreads]
  {   // exclusive scan of the segments' chunk counts: 4 segments per thread + a Hillis-Steele scan of the 256 partial sums
    int32_t c[4], tot = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int sidx = threadIdx.x * 4 + q;
      c[q] = sidx < n_seg ? (int32_t)((__ldg(seg_n + sidx) + kMirrorChunk - 1) / kMirrorChunk) : 0;
      tot += c[q];
    }
    part[threadIdx.x] = tot;
    __syncthreads();
    for (int d = 1; d < kThreads; d <<= 1) {
      const int32_t add = (int)threadIdx.x >= d ? part[threadIdx.x - d] : 0;
      __syncthreads();
      part[threadIdx.x] += add;
      __syncthreads();
    }
    int32_t run = part[threadIdx.x] - tot;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int sidx = threadIdx.x * 4 + q;
      if (sidx < n_seg) pre[sidx] = run;
      run += c[q];
    }
    if (threadIdx.x == kThreads - 1) pre[n_seg] = part[kThreads - 1];
    __syncthreads();
  }
  const int total = pre[n_seg];
  constexpr int Q = kMirrorChunk / (4 * kThreads);
  for (int chunk = blockIdx.x; chunk < total; chunk += gridDim.x) {
    int lo = 0, hi = n_seg;                       // largest s with pre[s] <= chunk (empty segments share a prefix: skip them)
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (pre[mid] <= chunk) lo = mid; else hi = mid;
    }
    const int sg = lo;
    const TT* src = reinterpret_cast<const TT*>(tables.p[__ldg(seg_rank + sg)]) + __ldg(seg_src + sg);
    TT* dst = mirror + __ldg(seg_dst + sg);
    const int64_t n4 = __ldg(seg_n + sg) >> 2;
    const int64_t base4 = (int64_t)(chunk - pre[sg]) * (kMirrorChunk / 4);
    V v[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int64_t i = base4 + threadIdx.x + q * kThreads;
      if (i < n4) v[q] = Unit4<TT>::ld(src + i * 4);
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int64_t i = base4 + threadIdx.x + q * kThreads;
      if (i < n4) reinterpret_cast<V*>(dst)[i] = v[q];
    }
  }
}

__global__ void __launch_bounds__(kThreads)
peer_mirror_refresh_kernel(const __grid_constant__ Peers tables, const int32_t* __restrict__ seg_rank,
                           const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                           const int64_t* __restrict__ seg_n, int n_seg, float* __restrict__ mirror) {
  peer_mirror_refresh_body<float>(tables, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
}

// FP16 tables: the same chunks (kMirrorChunk elements = 8 KB of halfs), 8-B vectors
__global__ void __launch_bounds__(kThreads)
peer_mirror_refresh_f16_kernel(const __grid_constant__ Peers tables, const int32_t* __restrict__ seg_rank,
                               const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                               const int64_t* __restrict__ seg_n, int n_seg, __half* __restrict__ mirror) {
  peer_mirror_refresh_body<__half>(tables, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
}

// ---- source side of the backward: stable multi-split of the ids by destination ---------------------------------------
// A tile = kBktTile consecutive bags (key-major order), 4 per thread; order inside a destination = bag order, then the
// order of the ids inside the bag — the order the unsharded backward's stable sort sees.
constexpr int kBktPerThread = 4;
constexpr int kBktTile = kThreads * kBktPerThread;

struct BktFeat {
  int64_t rows, block;
  int32_t owner, pad;
};

__device__ __forceinline__ void bkt_stage(BktFeat* fd, const int64_t* feat_rows, const int64_t* feat_block,
                                          const int32_t* feat_owner, int F) {
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    fd[f].rows = feat_rows[f];
    fd[f].block = feat_block[f];
    fd[f].owner = feat_owner ? feat_owner[f] : 0;
    fd[f].pad = 0;
  }
}

__global__ void __launch_bounds__(kThreads)
peer_bkt_count_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                      const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                      const int32_t* __restrict__ feat_owner, int F, int B, int W, int32_t* __restrict__ tile_counts,
                      int32_t* __restrict__ counts) {
  TZK_DYN_SMEM(unsigned char, smem_raw);
  BktFeat* fd = reinterpret_cast<BktFeat*>(smem_raw);
  int32_t* hist = reinterpret_cast<int32_t*>(fd + F);   // [W]
  bkt_stage(fd, feat_rows, feat_block, feat_owner, F);
  if ((int)threadIdx.x < W) hist[threadIdx.x] = 0;
  if (blockIdx.x == 0 && threadIdx.x == 0) counts[W] = 0;   // this step's overflow flag (set by the scan kernel)
  __syncthreads();
  const int64_t n_bags = (int64_t)F * B;
  const int64_t bag0 = (int64_t)blockIdx.x * kBktTile + (int64_t)threadIdx.x * kBktPerThread;
  for (int k = 0; k < kBktPerThread; ++k) {
    const int64_t bag = bag0 + k;
    if (bag >= n_bags) break;
    const BktFeat d = fd[(uint32_t)bag / (uint32_t)B];
    if (d.block <= 0) continue;        // feature kept off the wire (small table: its gradient is reduced at the source)
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    for (int64_t l = s; l < e; ++l) {
      int64_t id = __ldg(ids + l), loc;
      if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
      atomicAdd(hist + owner_of(id, d.block, d.owner, W, &loc), (int32_t)1);
    }
  }
  __syncthreads();
  if ((int)threadIdx.x < W) tile_counts[(int64_t)blockIdx.x * W + threadIdx.x] = hist[threadIdx.x];
}

// CTA w: exclusive scan over the tiles of destination w's counts (in place), total -> counts[w] (clamped to cap)
__global__ void __launch_bounds__(1024)
peer_bkt_scan_kernel(int32_t* __restrict__ tile_counts, int64_t n_tiles, int W, int64_t cap, int32_t* __restrict__ counts) {
  TZK_DYN_SMEM(int32_t, warp_tot);   // [32]
  const int w = blockIdx.x;
  const int T = blockDim.x;
  const int64_t per = (n_tiles + T - 1) / T;
  const int64_t t0 = (int64_t)threadIdx.x * per, t1 = t0 + per < n_tiles ? t0 + per : n_tiles;
  int32_t local = 0;
  for (int64_t t = t0; t < t1; ++t) local += tile_counts[t * W + w];
  // block-wide exclusive scan of `local`
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int32_t inc = local;
  for (int d = 1; d < 32; d <<= 1) {
    const int32_t o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) warp_tot[wid] = inc;
  __syncthreads();
  int32_t before = 0, total = 0;
  for (int i = 0; i < (T + 31) / 32; ++i) {
    const int32_t v = warp_tot[i];
    if (i < wid) before += v;
    total += v;
  }
  int32_t run = before + inc - local;
  for (int64_t t = t0; t < t1; ++t) {
    const int32_t c = tile_counts[t * W + w];
    tile_counts[t * W + w] = run;
    run += c;
  }
  if (threadIdx.x == 0) {
    counts[w] = (int64_t)total < cap ? total : (int32_t)cap;
    if ((int64_t)total > cap) atomicOr(counts + W, (int32_t)1);
  }
}

// WTD (pooled): also wire_w[slot] = psw[l], the weight of the id in that slot — read only by this rank's own push
template <bool WTD>
__device__ __forceinline__ void
peer_bkt_scatter_body(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                      const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                      const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ rf_key_base, int F, int B,
                      int W, int pooled, int64_t cap, const int32_t* __restrict__ tile_base,
                      int64_t* __restrict__ wire_key, int32_t* __restrict__ wire_idx, const float* __restrict__ psw,
                      float* __restrict__ wire_w) {
  TZK_DYN_SMEM(unsigned char, smem_raw);
  BktFeat* fd = reinterpret_cast<BktFeat*>(smem_raw);
  int32_t* sbase = reinterpret_cast<int32_t*>(fd + F);            // [W][kThreads]: next slot of (destination, thread)
  int32_t* wtot = sbase + (size_t)W * kThreads;                   // [W][8] warp totals
  bkt_stage(fd, feat_rows, feat_block, feat_owner, F);
  for (int i = threadIdx.x; i < W * kThreads; i += kThreads) sbase[i] = 0;
  __syncthreads();
  const int64_t n_bags = (int64_t)F * B;
  const int64_t bag0 = (int64_t)blockIdx.x * kBktTile + (int64_t)threadIdx.x * kBktPerThread;
  // pass 1: this thread's count per destination
  for (int k = 0; k < kBktPerThread; ++k) {
    const int64_t bag = bag0 + k;
    if (bag >= n_bags) break;
    const BktFeat d = fd[(uint32_t)bag / (uint32_t)B];
    if (d.block <= 0) continue;
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    for (int64_t l = s; l < e; ++l) {
      int64_t id = __ldg(ids + l), loc;
      if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
      sbase[owner_of(id, d.block, d.owner, W, &loc) * kThreads + threadIdx.x] += 1;
    }
  }
  // exclusive scan over the threads of the tile, per destination (thread order = bag order)
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int32_t mine[kMaxPeers];
#pragma unroll
  for (int w = 0; w < kMaxPeers; ++w) {
    mine[w] = 0;
    if (w < W) {                      // (W is block-uniform: every lane takes the same branch)
      const int32_t c = sbase[w * kThreads + threadIdx.x];
      int32_t inc = c;
      for (int d = 1; d < 32; d <<= 1) {
        const int32_t o = __shfl_up_sync(0xffffffffu, inc, d);
        if (lane >= d) inc += o;
      }
      if (lane == 31) wtot[w * 8 + wid] = inc;
      mine[w] = inc - c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int w = 0; w < kMaxPeers; ++w) {
    if (w < W) {
      int32_t before = 0;
      for (int i = 0; i < wid; ++i) before += wtot[w * 8 + i];
      sbase[w * kThreads + threadIdx.x] = tile_base[(int64_t)blockIdx.x * W + w] + before + mine[w];
    }
  }
  // (each thread only touches its own column of sbase from here on: no barrier needed)
  // pass 2: write
  for (int k = 0; k < kBktPerThread; ++k) {
    const int64_t bag = bag0 + k;
    if (bag >= n_bags) break;
    const int f = (int)((uint32_t)bag / (uint32_t)B);
    const BktFeat d = fd[f];
    if (d.block <= 0) continue;
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    for (int64_t l = s; l < e; ++l) {
      int64_t id = __ldg(ids + l), loc;
      if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
      const int r = owner_of(id, d.block, d.owner, W, &loc);
      const int32_t slot = sbase[r * kThreads + threadIdx.x]++;
      if (slot < cap) {               // ids beyond the wire capacity are dropped; the overflow flag reports it
        wire_key[(int64_t)r * cap + slot] = __ldg(rf_key_base + (int64_t)r * F + f) + loc;
        wire_idx[(int64_t)r * cap + slot] = pooled ? (int32_t)bag : (int32_t)l;
        if constexpr (WTD) wire_w[(int64_t)r * cap + slot] = __ldg(psw + l);
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
peer_bkt_scatter_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                        const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                        const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ rf_key_base, int F, int B,
                        int W, int pooled, int64_t cap, const int32_t* __restrict__ tile_base,
                        int64_t* __restrict__ wire_key, int32_t* __restrict__ wire_idx) {
  peer_bkt_scatter_body<false>(ids, offsets, feat_rows, feat_block, feat_owner, rf_key_base, F, B, W, pooled, cap,
                               tile_base, wire_key, wire_idx, nullptr, nullptr);
}

__global__ void __launch_bounds__(kThreads, 1)     // (the default register heuristic spilled the per-destination bases)
peer_bkt_scatter_weighted_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                                 const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                                 const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ rf_key_base, int F,
                                 int B, int W, int64_t cap, const int32_t* __restrict__ tile_base,
                                 int64_t* __restrict__ wire_key, int32_t* __restrict__ wire_idx,
                                 const float* __restrict__ psw, float* __restrict__ wire_w) {
  peer_bkt_scatter_body<true>(ids, offsets, feat_rows, feat_block, feat_owner, rf_key_base, F, B, W, 1, cap, tile_base,
                              wire_key, wire_idx, psw, wire_w);
}

// ---- publish the pooled-output gradient: dst = grad (MEAN bags pre-divided by their length, so that the owner needs
// nothing but the 64-B slice) ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
peer_publish_grad_kernel(const float* __restrict__ grad, int64_t ld_grad, const int32_t* __restrict__ feat_col,
                         const int32_t* __restrict__ feat_dim, const int32_t* __restrict__ feat_pool,
                         const int64_t* __restrict__ offsets, int F, int B, float* __restrict__ dst, int64_t ld_dst) {
  const int64_t n = (int64_t)F * B;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / F), f = (int)(i - (int64_t)b * F);       // consecutive threads: consecutive columns of a row
    const int col = __ldg(feat_col + f), dim = __ldg(feat_dim + f);
    float sc = 1.f;
    if (__ldg(feat_pool + f) == 1) {
      const int64_t bag = (int64_t)f * B + b;
      const int64_t L = __ldg(offsets + bag + 1) - __ldg(offsets + bag);
      sc = L > 0 ? 1.0f / (float)L : 0.f;
    }
    const float* s = grad + (int64_t)b * ld_grad + col;
    float* d = dst + (int64_t)b * ld_dst + col;
    for (int c = 0; c < dim; ++c) d[c] = s[c] * sc;
  }
}

// ---- push the gradient to the owners, in wire order -----------------------------------------------------------------
// Wire slot (dest r, j) of this rank -> row (me * cap + j) of rank r's receive buffer: consecutive slots are consecutive
// 64-B rows at the destination, so the NVLink writes are long coalesced bursts (posted, no round trip) while the
// scattered 64-B reads stay in local HBM.  The slice comes straight from the pooled-output gradient (no staging copy);
// MEAN bags are divided by their length here, so the owner's update needs nothing but the row.
// WTD (pooled): the slot's per-sample weight wire_w[s] (tzk_peer_bucketize_weighted) joins the scale.  The order is
// sc = (1/L) * w (SUM: 1 * w), then slice * sc — the unsharded weighted update's entry scale (grad_scale/L) * w with
// grad_scale = 1; the owner's update multiplies by its 1/W after that.  All-ones weights leave every bit unchanged.
template <int G, bool WTD>
__device__ __forceinline__ void
peer_push_grad_body(const Peers& recv, const float* __restrict__ grad, int64_t ld_grad,
                    const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                    const int64_t* __restrict__ offsets, const int32_t* __restrict__ wire_idx,
                    const int32_t* __restrict__ counts, int me, int W, int64_t cap, int B, int D, int pooled,
                    const float* __restrict__ wire_w) {
  constexpr int NG = kThreads / G;
  const int lane = threadIdx.x % G;
  const int64_t n = (int64_t)W * cap;
  for (int64_t s = (int64_t)blockIdx.x * NG + threadIdx.x / G; s < n; s += (int64_t)gridDim.x * NG) {
    const int r = (int)((uint32_t)s / (uint32_t)cap);          // W * cap < 2^31
    const int64_t j = s - (int64_t)r * cap;
    if (j >= __ldg(counts + r)) continue;
    const int32_t idx = __ldg(wire_idx + s);
    float w = 1.f;
    if constexpr (WTD) w = __ldg(wire_w + s);                  // (independent of idx: in flight next to it)
    const float* src;
    float sc = 1.f;
    if (pooled) {
      const int f = idx / B, b = idx - f * B;
      src = grad + (int64_t)b * ld_grad + __ldg(feat_col + f);
      if (__ldg(feat_pool + f) == 1) {
        const int64_t L = __ldg(offsets + idx + 1) - __ldg(offsets + idx);
        sc = 1.0f / (float)L;                       // L >= 1: the slot exists
      }
      if constexpr (WTD) sc *= w;
    } else {
      src = grad + (int64_t)idx * ld_grad;
    }
    float* dst = reinterpret_cast<float*>(recv.p[r]) + ((int64_t)me * cap + j) * D;
    for (int c = lane * 4; c < D; c += G * 4) {
      float4 v = *reinterpret_cast<const float4*>(src + c);
      v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
      *reinterpret_cast<float4*>(dst + c) = v;
    }
  }
}

template <int G>
__global__ void __launch_bounds__(kThreads)
peer_push_grad_kernel(const __grid_constant__ Peers recv, const float* __restrict__ grad, int64_t ld_grad,
                      const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                      const int64_t* __restrict__ offsets, const int32_t* __restrict__ wire_idx,
                      const int32_t* __restrict__ counts, int me, int W, int64_t cap, int B, int D, int pooled) {
  peer_push_grad_body<G, false>(recv, grad, ld_grad, feat_col, feat_pool, offsets, wire_idx, counts, me, W, cap, B, D,
                                pooled, nullptr);
}

template <int G>
__global__ void __launch_bounds__(kThreads)
peer_push_grad_weighted_kernel(const __grid_constant__ Peers recv, const float* __restrict__ grad, int64_t ld_grad,
                               const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                               const int64_t* __restrict__ offsets, const int32_t* __restrict__ wire_idx,
                               const int32_t* __restrict__ counts, int me, int W, int64_t cap, int B, int D,
                               const float* __restrict__ wire_w) {
  peer_push_grad_body<G, true>(recv, grad, ld_grad, feat_col, feat_pool, offsets, wire_idx, counts, me, W, cap, B, D, 1,
                               wire_w);
}

// ---- dense gradients: out = mean over ranks of src_r, summed in rank order (the same bits on every rank) --------------
__global__ void __launch_bounds__(kThreads)
peer_allreduce_mean_kernel(const __grid_constant__ Peers src, int W, int64_t n, float* __restrict__ out) {
  const float inv = 1.0f / (float)W;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v[kMaxPeers];           // every rank's value requested before the first one is consumed: ONE NVLink round trip
#pragma unroll
    for (int r = 0; r < kMaxPeers; ++r) v[r] = r < W ? reinterpret_cast<const float*>(src.p[r])[i] : 0.f;
    float acc = v[0];
#pragma unroll
    for (int r = 1; r < kMaxPeers; ++r)
      if (r < W) acc += v[r];     // rank order: the same bits on every rank
    out[i] = acc * inv;
  }
}

#ifndef TZK_CPU_SHIM
// ---- barrier over the NVSwitch domain ------------------------------------------------------------------------------
// pads.p[r] -> rank r's flag array (uint32 [W]) in symmetric memory; flag[src] on rank dst = last epoch src reached.
__global__ void peer_barrier_kernel(const __grid_constant__ Peers pads, int me, int W, uint32_t* __restrict__ epoch) {
  __shared__ uint32_t e;
  if (threadIdx.x == 0) {
    e = *epoch + 1;
    *epoch = e;
  }
  __syncthreads();
  __threadfence_system();               // everything this GPU wrote before the barrier is visible system-wide
  if ((int)threadIdx.x < W) {
    uint32_t* theirs = reinterpret_cast<uint32_t*>(pads.p[threadIdx.x]) + me;
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(theirs), "r"(e) : "memory");
    const uint32_t* mine = reinterpret_cast<const uint32_t*>(pads.p[me]) + threadIdx.x;
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory");
    } while ((int32_t)(v - e) < 0);
  }
}
#endif  // TZK_CPU_SHIM

int fill(Peers* dst, const uint64_t* host_ptrs, int W) {
  if (W < 1 || W > kMaxPeers || !host_ptrs) return 1;
  for (int r = 0; r < kMaxPeers; ++r) dst->p[r] = r < W ? host_ptrs[r] : 0ull;
  return 0;
}
int grid_for(int64_t work_ctas) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t cap = (int64_t)sms * 8;
  return (int)(work_ctas < cap ? (work_ctas > 0 ? work_ctas : 1) : cap);
}
inline int64_t bkt_tiles(int64_t n_bags) { return (n_bags + kBktTile - 1) / kBktTile; }
}  // namespace

// table_ptrs: HOST array [W] of device addresses (rank r's arena as mapped in THIS process); rf_w_off: device
// [W * F] int64 arena element offset of feature f's table on rank r; the other feature arrays as in tzk.h.
template <typename TT>
static int peer_pooled_gather_fwd_impl(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                       const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                       const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                       const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim,
                                       float* out, int64_t ld_out, const TT* mirror,
                                       const int64_t* feat_mirror_off, const int32_t* feat_sel, int32_t n_sel,
                                       void* stream, const float* psw = nullptr) {
  Peers t;
  if (fill(&t, table_ptrs, W) || F <= 0 || B <= 0 || max_dim <= 0 || (max_dim % 4) || (ld_out % 4)) return 1;
  if (feat_sel && (n_sel < 0 || n_sel > F)) return 1;
  if (feat_sel && n_sel == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)F * sizeof(FeatDesc) + (size_t)W * F * 8 + (size_t)W * 8 + (size_t)F * 8 + (size_t)F * 4;
  const int grid = grid_for((B + 31) / 32);
  if constexpr (!std::is_same<TT, float>::value) {     // FP16 tables
#define TZK_PEER_LAUNCH_H(G, WTD_)                                                                                     \
  TZK_LAUNCH((peer_pooled_gather_fwd_f16_kernel<G, WTD_>), grid, kThreads, smem, st, t, rf_w_off, feat_rows,          \
             feat_block, feat_owner, feat_dim, feat_col, feat_pool, ids, offsets, F, B, W, out, ld_out, mirror,        \
             feat_mirror_off, feat_sel, n_sel, psw)
    if (psw) {
      if (max_dim <= 16) TZK_PEER_LAUNCH_H(4, true);
      else if (max_dim <= 32) TZK_PEER_LAUNCH_H(8, true);
      else if (max_dim <= 64) TZK_PEER_LAUNCH_H(16, true);
      else TZK_PEER_LAUNCH_H(32, true);
    } else if (max_dim <= 16) TZK_PEER_LAUNCH_H(4, false);
    else if (max_dim <= 32) TZK_PEER_LAUNCH_H(8, false);
    else if (max_dim <= 64) TZK_PEER_LAUNCH_H(16, false);
    else TZK_PEER_LAUNCH_H(32, false);
#undef TZK_PEER_LAUNCH_H
    return cudaGetLastError() == cudaSuccess ? 0 : 3;
  } else {
#define TZK_PEER_LAUNCH(G)                                                                                             \
  TZK_LAUNCH((peer_pooled_gather_fwd_kernel<G>), grid, kThreads, smem, st, t, rf_w_off, feat_rows, feat_block,         \
             feat_owner, feat_dim, feat_col, feat_pool, ids, offsets, F, B, W, out, ld_out, mirror, feat_mirror_off,   \
             feat_sel, n_sel)
#define TZK_PEER_LAUNCH_W(G)                                                                                           \
  TZK_LAUNCH((peer_pooled_gather_fwd_weighted_kernel<G>), grid, kThreads, smem, st, t, rf_w_off, feat_rows,            \
             feat_block, feat_owner, feat_dim, feat_col, feat_pool, ids, offsets, F, B, W, out, ld_out, mirror,        \
             feat_mirror_off, feat_sel, n_sel, psw)
  if (psw) {
    if (max_dim <= 16) TZK_PEER_LAUNCH_W(4);
    else if (max_dim <= 32) TZK_PEER_LAUNCH_W(8);
    else if (max_dim <= 64) TZK_PEER_LAUNCH_W(16);
    else TZK_PEER_LAUNCH_W(32);
  } else if (max_dim <= 16) TZK_PEER_LAUNCH(4);
  else if (max_dim <= 32) TZK_PEER_LAUNCH(8);
  else if (max_dim <= 64) TZK_PEER_LAUNCH(16);
  else TZK_PEER_LAUNCH(32);
#undef TZK_PEER_LAUNCH_W
#undef TZK_PEER_LAUNCH
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
  }
}

extern "C" int tzk_peer_pooled_gather_fwd(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                          const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                          const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                          const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim,
                                          float* out, int64_t ld_out, const float* mirror,
                                          const int64_t* feat_mirror_off, void* stream) {
  return peer_pooled_gather_fwd_impl(table_ptrs, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                     ids, offsets, F, B, W, max_dim, out, ld_out, mirror, feat_mirror_off, nullptr, 0,
                                     stream);
}

// The same lookup restricted to the features listed in feat_sel [n_sel] (device int32, indices into the F descriptors):
// only their output columns are written.  Two launches over complementary lists on two streams overlap the local half
// of the lookup (mirrored tables) with the half whose rows cross NVLink.
extern "C" int tzk_peer_pooled_gather_fwd_sel(const uint64_t* table_ptrs, const int64_t* rf_w_off,
                                              const int64_t* feat_rows, const int64_t* feat_block,
                                              const int32_t* feat_owner, const int32_t* feat_dim, const int32_t* feat_col,
                                              const int32_t* feat_pool, const int64_t* ids, const int64_t* offsets,
                                              int32_t F, int32_t B, int32_t W, int32_t max_dim, float* out, int64_t ld_out,
                                              const float* mirror, const int64_t* feat_mirror_off,
                                              const int32_t* feat_sel, int32_t n_sel, void* stream) {
  if (!feat_sel) return 1;
  return peer_pooled_gather_fwd_impl(table_ptrs, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                     ids, offsets, F, B, W, max_dim, out, ld_out, mirror, feat_mirror_off, feat_sel, n_sel,
                                     stream);
}

// Weighted bags (per_sample_weights [nnz] of this rank's own batch): the same lookup, pooled as
// tzk_pooled_gather_fwd_weighted does.  feat_sel nullable (NULL: every feature, as tzk_peer_pooled_gather_fwd).
extern "C" int tzk_peer_pooled_gather_fwd_weighted(const uint64_t* table_ptrs, const int64_t* rf_w_off,
                                                   const int64_t* feat_rows, const int64_t* feat_block,
                                                   const int32_t* feat_owner, const int32_t* feat_dim,
                                                   const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                                   const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                                   int32_t max_dim, float* out, int64_t ld_out, const float* mirror,
                                                   const int64_t* feat_mirror_off, const float* per_sample_weights,
                                                   const int32_t* feat_sel, int32_t n_sel, void* stream) {
  if (!per_sample_weights) return 1;
  return peer_pooled_gather_fwd_impl(table_ptrs, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                     ids, offsets, F, B, W, max_dim, out, ld_out, mirror, feat_mirror_off, feat_sel, n_sel,
                                     stream, per_sample_weights);
}

// FP16 tables: the same lookups over arenas and a mirror of halfs (pooling and outputs fp32, the bits of
// tzk_pooled_gather_fwd_f16 / tzk_pooled_gather_fwd_weighted with weights_f16).  Rows are 8-B aligned (dims multiples of 4).
extern "C" int tzk_peer_pooled_gather_fwd_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off,
                                              const int64_t* feat_rows, const int64_t* feat_block,
                                              const int32_t* feat_owner, const int32_t* feat_dim, const int32_t* feat_col,
                                              const int32_t* feat_pool, const int64_t* ids, const int64_t* offsets,
                                              int32_t F, int32_t B, int32_t W, int32_t max_dim, float* out,
                                              int64_t ld_out, const void* mirror, const int64_t* feat_mirror_off,
                                              void* stream) {
  return peer_pooled_gather_fwd_impl(table_ptrs, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                     ids, offsets, F, B, W, max_dim, out, ld_out, static_cast<const __half*>(mirror),
                                     feat_mirror_off, nullptr, 0, stream);
}

extern "C" int tzk_peer_pooled_gather_fwd_sel_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off,
                                                  const int64_t* feat_rows, const int64_t* feat_block,
                                                  const int32_t* feat_owner, const int32_t* feat_dim,
                                                  const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                                  const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                                  int32_t max_dim, float* out, int64_t ld_out, const void* mirror,
                                                  const int64_t* feat_mirror_off, const int32_t* feat_sel, int32_t n_sel,
                                                  void* stream) {
  if (!feat_sel) return 1;
  return peer_pooled_gather_fwd_impl(table_ptrs, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                     ids, offsets, F, B, W, max_dim, out, ld_out, static_cast<const __half*>(mirror),
                                     feat_mirror_off, feat_sel, n_sel, stream);
}

extern "C" int tzk_peer_pooled_gather_fwd_weighted_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off,
                                                       const int64_t* feat_rows, const int64_t* feat_block,
                                                       const int32_t* feat_owner, const int32_t* feat_dim,
                                                       const int32_t* feat_col, const int32_t* feat_pool,
                                                       const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B,
                                                       int32_t W, int32_t max_dim, float* out, int64_t ld_out,
                                                       const void* mirror, const int64_t* feat_mirror_off,
                                                       const float* per_sample_weights, const int32_t* feat_sel,
                                                       int32_t n_sel, void* stream) {
  if (!per_sample_weights) return 1;
  return peer_pooled_gather_fwd_impl(table_ptrs, rf_w_off, feat_rows, feat_block, feat_owner, feat_dim, feat_col, feat_pool,
                                     ids, offsets, F, B, W, max_dim, out, ld_out, static_cast<const __half*>(mirror),
                                     feat_mirror_off, feat_sel, n_sel, stream, per_sample_weights);
}

extern "C" int tzk_peer_seq_gather_fwd(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                       const int64_t* feat_block, const int32_t* feat_owner, const int64_t* ids,
                                       const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t D, int64_t nnz,
                                       float* out, const float* mirror, const int64_t* feat_mirror_off, void* stream) {
  Peers t;
  if (fill(&t, table_ptrs, W) || F <= 0 || B <= 0 || D <= 0 || (D % 4) || nnz < 0) return 1;
  if (nnz == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)(F + 1) * 8 + (size_t)F * 16 + (size_t)W * F * 8 + (size_t)W * 8 + (size_t)F * 4 + 16;
#define TZK_PEER_LAUNCH(G)                                                                                            \
  TZK_LAUNCH((peer_seq_gather_fwd_kernel<G>), grid_for((nnz + (kThreads / G) * 4 - 1) / ((kThreads / G) * 4)),        \
             kThreads, smem, st, t, rf_w_off, feat_rows, feat_block, feat_owner, ids, offsets, F, B, W, D, nnz, out,   \
             mirror, feat_mirror_off)
  if (D <= 16) TZK_PEER_LAUNCH(4);
  else if (D <= 32) TZK_PEER_LAUNCH(8);
  else if (D <= 64) TZK_PEER_LAUNCH(16);
  else TZK_PEER_LAUNCH(32);
#undef TZK_PEER_LAUNCH
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

extern "C" int tzk_peer_seq_gather_fwd_f16(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                           const int64_t* feat_block, const int32_t* feat_owner, const int64_t* ids,
                                           const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t D,
                                           int64_t nnz, float* out, const void* mirror, const int64_t* feat_mirror_off,
                                           void* stream) {
  Peers t;
  if (fill(&t, table_ptrs, W) || F <= 0 || B <= 0 || D <= 0 || (D % 4) || nnz < 0) return 1;
  if (nnz == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const __half* mh = static_cast<const __half*>(mirror);
  const size_t smem = (size_t)(F + 1) * 8 + (size_t)F * 16 + (size_t)W * F * 8 + (size_t)W * 8 + (size_t)F * 4 + 16;
#define TZK_PEER_LAUNCH(G)                                                                                            \
  TZK_LAUNCH((peer_seq_gather_fwd_f16_kernel<G>), grid_for((nnz + (kThreads / G) * 4 - 1) / ((kThreads / G) * 4)),    \
             kThreads, smem, st, t, rf_w_off, feat_rows, feat_block, feat_owner, ids, offsets, F, B, W, D, nnz, out,   \
             mh, feat_mirror_off)
  if (D <= 16) TZK_PEER_LAUNCH(4);
  else if (D <= 32) TZK_PEER_LAUNCH(8);
  else if (D <= 64) TZK_PEER_LAUNCH(16);
  else TZK_PEER_LAUNCH(32);
#undef TZK_PEER_LAUNCH
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

// Copies n_seg contiguous pieces of the ranks' arenas into the local mirror (see peer_mirror_refresh_kernel); the
// segment arrays are device arrays built once from the sharding plan.
template <typename TT>
static int peer_mirror_refresh_impl(const uint64_t* table_ptrs, int32_t W, const int32_t* seg_rank,
                                    const int64_t* seg_src, const int64_t* seg_dst, const int64_t* seg_n,
                                    int32_t n_seg, TT* mirror, void* stream) {
  constexpr bool f16 = !std::is_same<TT, float>::value;
  Peers t;
  if (fill(&t, table_ptrs, W) || n_seg < 0) return 1;
  if (n_seg == 0) return 0;
  if (!seg_rank || !seg_src || !seg_dst || !seg_n || !mirror) return 1;
  // the chunked kernel is the default; TZK_PEER_MIRROR_CHUNKED=0:
  // one load in flight per thread
  const char* mc = getenv("TZK_PEER_MIRROR_CHUNKED");
  const char* xp = "1";
#ifdef TZK_CPU_SHIM
  const bool chunked = !(mc && mc[0] == '0');      // (host emulation: the chunked kernel unless told otherwise)
  (void)xp;
#else
  const bool chunked = (mc && (mc[0] == '0' || mc[0] == '1')) ? mc[0] == '1' : (xp && xp[0] == '1');
#endif
  if (n_seg > kMirrorMaxSeg || !chunked) {
#ifdef TZK_CPU_SHIM
    dim3 grid(1, n_seg);          // (one std::thread per CUDA thread — keep the launch small)
#else
    dim3 grid(8, n_seg < 4096 ? n_seg : 4096);
#endif
    if constexpr (f16)
      TZK_LAUNCH((peer_mirror_refresh_simple_f16_kernel), grid, kThreads, 0, reinterpret_cast<cudaStream_t>(stream), t,
                 seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
    else
      TZK_LAUNCH((peer_mirror_refresh_simple_kernel), grid, kThreads, 0, reinterpret_cast<cudaStream_t>(stream), t,
                 seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
    return cudaGetLastError() == cudaSuccess ? 0 : 3;
  }
#ifdef TZK_CPU_SHIM
  const int grid = 3;             // (host emulation: one std::thread per CUDA thread — keep the launch small)
#else
  const int grid = 132 * 4;
#endif
  if constexpr (f16)
    TZK_LAUNCH((peer_mirror_refresh_f16_kernel), grid, kThreads, (kMirrorMaxSeg + 1 + kThreads) * sizeof(int32_t),
               reinterpret_cast<cudaStream_t>(stream), t, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
  else
    TZK_LAUNCH((peer_mirror_refresh_kernel), grid, kThreads, (kMirrorMaxSeg + 1 + kThreads) * sizeof(int32_t),
               reinterpret_cast<cudaStream_t>(stream), t, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

extern "C" int tzk_peer_mirror_refresh(const uint64_t* table_ptrs, int32_t W, const int32_t* seg_rank,
                                       const int64_t* seg_src, const int64_t* seg_dst, const int64_t* seg_n,
                                       int32_t n_seg, float* mirror, void* stream) {
  return peer_mirror_refresh_impl(table_ptrs, W, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror, stream);
}

// FP16 tables: segments counted in halfs (multiples of 4: 8-B vectors), mirror of halfs, bits copied unchanged
extern "C" int tzk_peer_mirror_refresh_f16(const uint64_t* table_ptrs, int32_t W, const int32_t* seg_rank,
                                           const int64_t* seg_src, const int64_t* seg_dst, const int64_t* seg_n,
                                           int32_t n_seg, void* mirror, void* stream) {
  return peer_mirror_refresh_impl(table_ptrs, W, seg_rank, seg_src, seg_dst, seg_n, n_seg, static_cast<__half*>(mirror),
                                  stream);
}

#ifndef TZK_CPU_SHIM
extern "C" int tzk_peer_barrier(const uint64_t* pad_ptrs, int32_t me, int32_t W, uint32_t* epoch, void* stream) {
  Peers p;
  if (fill(&p, pad_ptrs, W) || me < 0 || me >= W || !epoch) return 1;
  peer_barrier_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, me, W, epoch);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
#endif

// workspace: per-tile destination counts / bases, int32 [tiles * W]
extern "C" size_t tzk_peer_bucketize_workspace_bytes(int32_t F, int32_t B, int32_t W) {
  return (size_t)(bkt_tiles((int64_t)F * B) * (W < 1 ? 1 : W) + 64) * sizeof(int32_t);
}

// ids of the local batch -> this rank's wire buffers.  Destination r's entries start at r * cap, in (feature, bag,
// position) order; wire_key = rf_key_base[r * F + f] + owner-local row, wire_idx = bag index (pooled) or id position
// (sequence).  counts [W + 1]: ids per destination (clamped to cap) and, in counts[W], 1 if any destination overflowed.
static int peer_bucketize_impl(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                               const int64_t* feat_block, const int32_t* feat_owner, const int64_t* feat_rows,
                               const int64_t* rf_key_base, int32_t pooled, int64_t cap, int64_t* wire_key,
                               int32_t* wire_idx, int32_t* counts, void* workspace, size_t workspace_bytes, void* stream,
                               const float* psw = nullptr, float* wire_w = nullptr) {
  if (F <= 0 || B <= 0 || W < 1 || W > kMaxPeers || cap <= 0 || cap * W >= ((int64_t)1 << 31)) return 1;
  if (!offsets || !feat_block || !feat_rows || !rf_key_base || !wire_key || !wire_idx || !counts || !workspace)
    return 1;
  if (workspace_bytes < tzk_peer_bucketize_workspace_bytes(F, B, W)) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t tiles = bkt_tiles((int64_t)F * B);
  int32_t* tile_counts = static_cast<int32_t*>(workspace);
  const size_t smem_c = (size_t)F * sizeof(BktFeat) + (size_t)W * 4;
  TZK_LAUNCH((peer_bkt_count_kernel), (unsigned)tiles, kThreads, smem_c, st, ids, offsets, feat_rows, feat_block,
             feat_owner, F, B, W, tile_counts, counts);
  TZK_LAUNCH((peer_bkt_scan_kernel), (unsigned)W, 1024, (size_t)32 * 4, st, tile_counts, tiles, W, cap, counts);
  const size_t smem_s = (size_t)F * sizeof(BktFeat) + (size_t)W * kThreads * 4 + (size_t)W * 8 * 4;
  if (wire_w) {
    TZK_LAUNCH((peer_bkt_scatter_weighted_kernel), (unsigned)tiles, kThreads, smem_s, st, ids, offsets, feat_rows,
               feat_block, feat_owner, rf_key_base, F, B, W, cap, tile_counts, wire_key, wire_idx, psw, wire_w);
  } else {
    TZK_LAUNCH((peer_bkt_scatter_kernel), (unsigned)tiles, kThreads, smem_s, st, ids, offsets, feat_rows, feat_block,
               feat_owner, rf_key_base, F, B, W, pooled, cap, tile_counts, wire_key, wire_idx);
  }
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

extern "C" int tzk_peer_bucketize(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                  const int64_t* feat_block, const int32_t* feat_owner, const int64_t* feat_rows,
                                  const int64_t* rf_key_base, int32_t pooled, int64_t cap, int64_t* wire_key,
                                  int32_t* wire_idx, int32_t* counts, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  return peer_bucketize_impl(ids, offsets, F, B, W, feat_block, feat_owner, feat_rows, rf_key_base, pooled, cap, wire_key,
                             wire_idx, counts, workspace, workspace_bytes, stream);
}

// Weighted bags (pooled only): tzk_peer_bucketize plus wire_w [W * cap] (this rank's local memory, not symmetric), the
// per-sample weight of the id in every wire slot, written next to its key and bag.  Only this rank's push reads it.
extern "C" int tzk_peer_bucketize_weighted(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                           const int64_t* feat_block, const int32_t* feat_owner,
                                           const int64_t* feat_rows, const int64_t* rf_key_base, int32_t pooled,
                                           int64_t cap, int64_t* wire_key, int32_t* wire_idx, int32_t* counts,
                                           void* workspace, size_t workspace_bytes, const float* per_sample_weights,
                                           float* wire_w, void* stream) {
  if (!pooled || !per_sample_weights || !wire_w) return 1;
  return peer_bucketize_impl(ids, offsets, F, B, W, feat_block, feat_owner, feat_rows, rf_key_base, pooled, cap, wire_key,
                             wire_idx, counts, workspace, workspace_bytes, stream, per_sample_weights, wire_w);
}

extern "C" int tzk_peer_publish_grad(const float* grad, int64_t ld_grad, const int32_t* feat_col, const int32_t* feat_dim,
                                     const int32_t* feat_pool, const int64_t* offsets, int32_t F, int32_t B, float* dst,
                                     int64_t ld_dst, void* stream) {
  if (F <= 0 || B <= 0 || !grad || !dst || !feat_col || !feat_dim || !feat_pool || !offsets) return 1;
  const int64_t n = (int64_t)F * B;
  TZK_LAUNCH((peer_publish_grad_kernel), grid_for((n + kThreads - 1) / kThreads), kThreads, 0,
             reinterpret_cast<cudaStream_t>(stream), grad, ld_grad, feat_col, feat_dim, feat_pool, offsets, F, B, dst,
             ld_dst);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

// grad: this rank's pooled-output gradient [B, ld_grad] (pooled) or row gradient [nnz, ld_grad] (sequence);
// recv_ptrs[r]: rank r's receive buffer [W * cap, D]; wire_idx / counts: this rank's own wire buffers (tzk_peer_bucketize).
extern "C" int tzk_peer_push_grad(const uint64_t* recv_ptrs, const float* grad, int64_t ld_grad, const int32_t* feat_col,
                                  const int32_t* feat_pool, const int64_t* offsets, const int32_t* wire_idx,
                                  const int32_t* counts, int32_t me, int32_t W, int64_t cap, int32_t B, int32_t D,
                                  int32_t pooled, void* stream) {
  Peers p;
  if (fill(&p, recv_ptrs, W) || me < 0 || me >= W || cap <= 0 || B <= 0 || D <= 0 || (D % 4) || (ld_grad % 4)) return 1;
  if (!grad || !wire_idx || !counts || (pooled && (!feat_col || !feat_pool || !offsets))) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t slots = (int64_t)W * cap;
#define TZK_PEER_LAUNCH(G)                                                                                           \
  TZK_LAUNCH((peer_push_grad_kernel<G>), grid_for((slots + kThreads / G - 1) / (kThreads / G)), kThreads, 0, st, p,  \
             grad, ld_grad, feat_col, feat_pool, offsets, wire_idx, counts, me, W, cap, B, D, pooled)
  if (D <= 16) TZK_PEER_LAUNCH(4);
  else if (D <= 32) TZK_PEER_LAUNCH(8);
  else if (D <= 64) TZK_PEER_LAUNCH(16);
  else TZK_PEER_LAUNCH(32);
#undef TZK_PEER_LAUNCH
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

// Weighted bags (pooled only): tzk_peer_push_grad with every slice scaled by its slot's weight wire_w[s]
// (tzk_peer_bucketize_weighted), folded into the MEAN 1/L — the pushed row is w * g (/ L).
extern "C" int tzk_peer_push_grad_weighted(const uint64_t* recv_ptrs, const float* grad, int64_t ld_grad,
                                           const int32_t* feat_col, const int32_t* feat_pool, const int64_t* offsets,
                                           const int32_t* wire_idx, const int32_t* counts, int32_t me, int32_t W,
                                           int64_t cap, int32_t B, int32_t D, int32_t pooled, const float* wire_w,
                                           void* stream) {
  Peers p;
  if (fill(&p, recv_ptrs, W) || me < 0 || me >= W || cap <= 0 || B <= 0 || D <= 0 || (D % 4) || (ld_grad % 4)) return 1;
  if (!pooled || !wire_w || !grad || !wire_idx || !counts || !feat_col || !feat_pool || !offsets) return 1;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t slots = (int64_t)W * cap;
#define TZK_PEER_LAUNCH(G)                                                                                           \
  TZK_LAUNCH((peer_push_grad_weighted_kernel<G>), grid_for((slots + kThreads / G - 1) / (kThreads / G)), kThreads, 0, \
             st, p, grad, ld_grad, feat_col, feat_pool, offsets, wire_idx, counts, me, W, cap, B, D, wire_w)
  if (D <= 16) TZK_PEER_LAUNCH(4);
  else if (D <= 32) TZK_PEER_LAUNCH(8);
  else if (D <= 64) TZK_PEER_LAUNCH(16);
  else TZK_PEER_LAUNCH(32);
#undef TZK_PEER_LAUNCH
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

extern "C" int tzk_peer_allreduce_mean(const uint64_t* src_ptrs, int32_t W, int64_t n, float* out, void* stream) {
  Peers p;
  if (fill(&p, src_ptrs, W) || n < 0 || !out) return 1;
  if (n == 0) return 0;
  TZK_LAUNCH((peer_allreduce_mean_kernel), grid_for((n + kThreads - 1) / kThreads), kThreads, 0,
             reinterpret_cast<cudaStream_t>(stream), p, W, n, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
