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
//
// This file compiles for the host too (TZK_CPU_SHIM, tests/test_peer_exchange_model.py runs the kernels' source on
// std::threads), so it uses plain CUDA + warp shuffles only; the barrier (PTX) is excluded from that build.
#ifdef TZK_CPU_SHIM
#include "cuda_cpu_shim.h"
#else
#include <cuda_runtime.h>
#define TZK_DYN_SMEM(type, name) extern __shared__ __align__(16) type name[]
#define TZK_UNPAREN(...) __VA_ARGS__
#define TZK_LAUNCH(kernel, grid, block, smem, stream, ...) TZK_UNPAREN kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#endif
#include <stdint.h>
#include <stdlib.h>

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

  auto row_ptr = [&](int f, const FeatDesc& d, int64_t id) -> const float* {
    if ((uint64_t)id >= (uint64_t)d.rows) id = 0;
    if (m_off[f] >= 0) return mirror + m_off[f] + id * d.dim;     // small table: this step's local copy of all its rows
    int64_t loc;
    const int r = owner_of(id, d.block, d.owner, W, &loc);
    return reinterpret_cast<const float*>(base[r]) + w_off[r * F + f] + loc * d.dim;
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
      float4 acc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        acc[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (len[u] > 0) {
          const int f = sel[(i0 + u * NG) / TB];
          const FeatDesc& d = fd[f];
          if (lane * 4 < d.dim) acc[u] = ld_peer_f4(row_ptr(f, d, id0[u]) + lane * 4);
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
            a = (c == lane * 4) ? acc[u] : ld_peer_f4(row_ptr(f, d, id0[u]) + c);
            for (int l = 1; l < len[u]; ++l)
              a = f4_add(a, ld_peer_f4(row_ptr(f, d, __ldg(ids + s[u] + l)) + c));
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

// un-pooled (sequence) lookup: one lane group per id position, feature by binary search over the segment starts
template <int G>
__global__ void __launch_bounds__(kThreads)
peer_seq_gather_fwd_kernel(const __grid_constant__ Peers tables, const int64_t* __restrict__ rf_w_off,
                           const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                           const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ ids,
                           const int64_t* __restrict__ offsets, int F, int B, int W, int D, int64_t nnz,
                           float* __restrict__ out, const float* __restrict__ mirror,
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
    const float* src[U];
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
          src[u] = reinterpret_cast<const float*>(base[r]) + w_off[r * F + lo] + loc * D;
        }
      }
    }
    for (int c = lane * 4; c < D; c += G * 4) {
      float4 v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = src[u] ? ld_peer_f4(src[u] + c) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (src[u]) *reinterpret_cast<float4*>(out + (l0 + u) * D + c) = v[u];
    }
  }
}

// ---- per-step local copy of the small tables ------------------------------------------------------------------------------
// Most lookups of a Criteo-like workload hit tables of a few thousand rows (18 of 26 features, 69 % of the ids): their
// shards are a few MB in total, so every rank copies them from the owners once per step — long sequential NVLink reads
// — and its gather reads those features from local memory; only the big tables' rows cross NVLink as
// random 64-B reads.  Segment s: n[s] floats from rank r[s]'s arena at src[s] to mirror + dst[s].
__global__ void __launch_bounds__(kThreads)
peer_mirror_refresh_simple_kernel(const __grid_constant__ Peers tables, const int32_t* __restrict__ seg_rank,
                                  const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                                  const int64_t* __restrict__ seg_n, int n_seg, float* __restrict__ mirror) {
  for (int s = blockIdx.y; s < n_seg; s += gridDim.y) {
    const float* src = reinterpret_cast<const float*>(tables.p[__ldg(seg_rank + s)]) + __ldg(seg_src + s);
    float* dst = mirror + __ldg(seg_dst + s);
    const int64_t n4 = __ldg(seg_n + s) >> 2;       // table starts and row sizes are multiples of 4 floats
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x)
      reinterpret_cast<float4*>(dst)[i] = ld_peer_f4(src + i * 4);
  }
}

// The segments cut into chunks of kMirrorChunk floats, chunks dealt round-robin to the CTAs: every thread has
// kMirrorChunk / (4 * kThreads) independent 16-B NVLink reads in flight (one load in flight per thread — the simple kernel —
// pays the NVLink round trip once per 16 B and thread).  n_seg <= kMirrorMaxSeg.
constexpr int kMirrorChunk = 4096;
constexpr int kMirrorMaxSeg = 4 * kThreads;
__global__ void __launch_bounds__(kThreads)
peer_mirror_refresh_kernel(const __grid_constant__ Peers tables, const int32_t* __restrict__ seg_rank,
                           const int64_t* __restrict__ seg_src, const int64_t* __restrict__ seg_dst,
                           const int64_t* __restrict__ seg_n, int n_seg, float* __restrict__ mirror) {
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
    const float* src = reinterpret_cast<const float*>(tables.p[__ldg(seg_rank + sg)]) + __ldg(seg_src + sg);
    float* dst = mirror + __ldg(seg_dst + sg);
    const int64_t n4 = __ldg(seg_n + sg) >> 2;
    const int64_t base4 = (int64_t)(chunk - pre[sg]) * (kMirrorChunk / 4);
    float4 v[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int64_t i = base4 + threadIdx.x + q * kThreads;
      if (i < n4) v[q] = ld_peer_f4(src + i * 4);
    }
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int64_t i = base4 + threadIdx.x + q * kThreads;
      if (i < n4) reinterpret_cast<float4*>(dst)[i] = v[q];
    }
  }
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

__global__ void __launch_bounds__(kThreads)
peer_bkt_scatter_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                        const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_block,
                        const int32_t* __restrict__ feat_owner, const int64_t* __restrict__ rf_key_base, int F, int B,
                        int W, int pooled, int64_t cap, const int32_t* __restrict__ tile_base,
                        int64_t* __restrict__ wire_key, int32_t* __restrict__ wire_idx) {
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
      }
    }
  }
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
template <int G>
__global__ void __launch_bounds__(kThreads)
peer_push_grad_kernel(const __grid_constant__ Peers recv, const float* __restrict__ grad, int64_t ld_grad,
                      const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                      const int64_t* __restrict__ offsets, const int32_t* __restrict__ wire_idx,
                      const int32_t* __restrict__ counts, int me, int W, int64_t cap, int B, int D, int pooled) {
  constexpr int NG = kThreads / G;
  const int lane = threadIdx.x % G;
  const int64_t n = (int64_t)W * cap;
  for (int64_t s = (int64_t)blockIdx.x * NG + threadIdx.x / G; s < n; s += (int64_t)gridDim.x * NG) {
    const int r = (int)((uint32_t)s / (uint32_t)cap);          // W * cap < 2^31
    const int64_t j = s - (int64_t)r * cap;
    if (j >= __ldg(counts + r)) continue;
    const int32_t idx = __ldg(wire_idx + s);
    const float* src;
    float sc = 1.f;
    if (pooled) {
      const int f = idx / B, b = idx - f * B;
      src = grad + (int64_t)b * ld_grad + __ldg(feat_col + f);
      if (__ldg(feat_pool + f) == 1) {
        const int64_t L = __ldg(offsets + idx + 1) - __ldg(offsets + idx);
        sc = 1.0f / (float)L;                       // L >= 1: the slot exists
      }
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
static int peer_pooled_gather_fwd_impl(const uint64_t* table_ptrs, const int64_t* rf_w_off, const int64_t* feat_rows,
                                       const int64_t* feat_block, const int32_t* feat_owner, const int32_t* feat_dim,
                                       const int32_t* feat_col, const int32_t* feat_pool, const int64_t* ids,
                                       const int64_t* offsets, int32_t F, int32_t B, int32_t W, int32_t max_dim,
                                       float* out, int64_t ld_out, const float* mirror,
                                       const int64_t* feat_mirror_off, const int32_t* feat_sel, int32_t n_sel,
                                       void* stream) {
  Peers t;
  if (fill(&t, table_ptrs, W) || F <= 0 || B <= 0 || max_dim <= 0 || (max_dim % 4) || (ld_out % 4)) return 1;
  if (feat_sel && (n_sel < 0 || n_sel > F)) return 1;
  if (feat_sel && n_sel == 0) return 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const size_t smem = (size_t)F * sizeof(FeatDesc) + (size_t)W * F * 8 + (size_t)W * 8 + (size_t)F * 8 + (size_t)F * 4;
  const int grid = grid_for((B + 31) / 32);
#define TZK_PEER_LAUNCH(G)                                                                                             \
  TZK_LAUNCH((peer_pooled_gather_fwd_kernel<G>), grid, kThreads, smem, st, t, rf_w_off, feat_rows, feat_block,         \
             feat_owner, feat_dim, feat_col, feat_pool, ids, offsets, F, B, W, out, ld_out, mirror, feat_mirror_off,   \
             feat_sel, n_sel)
  if (max_dim <= 16) TZK_PEER_LAUNCH(4);
  else if (max_dim <= 32) TZK_PEER_LAUNCH(8);
  else if (max_dim <= 64) TZK_PEER_LAUNCH(16);
  else TZK_PEER_LAUNCH(32);
#undef TZK_PEER_LAUNCH
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
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

// Copies n_seg contiguous pieces of the ranks' arenas into the local mirror (see peer_mirror_refresh_kernel); the
// segment arrays are device arrays built once from the sharding plan.
extern "C" int tzk_peer_mirror_refresh(const uint64_t* table_ptrs, int32_t W, const int32_t* seg_rank,
                                       const int64_t* seg_src, const int64_t* seg_dst, const int64_t* seg_n,
                                       int32_t n_seg, float* mirror, void* stream) {
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
    TZK_LAUNCH((peer_mirror_refresh_simple_kernel), grid, kThreads, 0, reinterpret_cast<cudaStream_t>(stream), t, seg_rank,
               seg_src, seg_dst, seg_n, n_seg, mirror);
    return cudaGetLastError() == cudaSuccess ? 0 : 3;
  }
#ifdef TZK_CPU_SHIM
  const int grid = 3;             // (host emulation: one std::thread per CUDA thread — keep the launch small)
#else
  const int grid = 132 * 4;
#endif
  TZK_LAUNCH((peer_mirror_refresh_kernel), grid, kThreads, (kMirrorMaxSeg + 1 + kThreads) * sizeof(int32_t),
             reinterpret_cast<cudaStream_t>(stream), t, seg_rank, seg_src, seg_dst, seg_n, n_seg, mirror);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
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
extern "C" int tzk_peer_bucketize(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                  const int64_t* feat_block, const int32_t* feat_owner, const int64_t* feat_rows,
                                  const int64_t* rf_key_base, int32_t pooled, int64_t cap, int64_t* wire_key,
                                  int32_t* wire_idx, int32_t* counts, void* workspace, size_t workspace_bytes,
                                  void* stream) {
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
  TZK_LAUNCH((peer_bkt_scatter_kernel), (unsigned)tiles, kThreads, smem_s, st, ids, offsets, feat_rows, feat_block,
             feat_owner, rf_key_base, F, B, W, pooled, cap, tile_counts, wire_key, wire_idx);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
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

extern "C" int tzk_peer_allreduce_mean(const uint64_t* src_ptrs, int32_t W, int64_t n, float* out, void* stream) {
  Peers p;
  if (fill(&p, src_ptrs, W) || n < 0 || !out) return 1;
  if (n == 0) return 0;
  TZK_LAUNCH((peer_allreduce_mean_kernel), grid_for((n + kThreads - 1) / kThreads), kThreads, 0,
             reinterpret_cast<cudaStream_t>(stream), p, W, n, out);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
