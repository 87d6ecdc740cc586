// tzk_bwd.cu — K5 fused segmented backward + sparse optimizer (sm_90a).
//
// Pipeline (all on the caller's stream, no host sync):
//   1. linearize : key[l] = feat_key_base[f] + id[l], val[l] = bag (pooled) or l (sequence)
//   2. stable LSD radix sort of (key,val) over ceil(log2(total_keys)) bits (CUB DeviceRadixSort — the one
//      library primitive on this path; everything else is hand-written)
//   3. fused run kernel: one lane group per sorted position; the group that sits on the head of a run of
//      equal keys sums the run's gradient rows in sorted (= stable, ascending bag) order and applies ONE
//      optimizer update to the table row in place — no dense gradient, no atomics, run-to-run
//      deterministic.  Runs longer than kShortRun are deferred to
//   4. long-run kernel: one CTA per long run (tiny tables / hot ids), strided partial sums per lane group
//      + fixed-order tree in shared memory, then the update.
#include <algorithm>
#include <cstdlib>
#include <cub/device/device_radix_sort.cuh>

#include "tzk_common.cuh"

using namespace tzk;

namespace {

constexpr int kThreads = 256;
constexpr int kShortRun = 32;

// TZK_OPT_ACCUM_OUT (include/tzk.h): do not update — store the summed row gradient in `weights` (a dense per-row buffer)
// and raise `state[key]` (int32 flags): the source-side half of "reduce small tables locally, exchange per-row partial
// sums" (tzk_peer_small_update is the owner-side half)
struct BwdFeat {
  int64_t w_off;
  int64_t rows;
  int64_t key_base;
  int32_t dim;
  int32_t col;
  int32_t pool;
  int32_t stride;   // elements between consecutive rows of the table: dim, or 2 * dim when a.interleaved
};

// q = v / d for 0 <= v < 2^31, d >= 1: m = ceil(2^(31 + l) / d), l = ceil(log2 d) fits 32 bits and
// floor(v * m / 2^(31 + l)) is exact for 31-bit v (Granlund & Montgomery); d == 1 -> mul = 0.
struct FastDiv {
  uint32_t mul;
  int32_t shift;   // l - 1 (applied after the high word of the product)
};
inline FastDiv make_fast_div(int64_t d) {
  FastDiv f;
  f.mul = 0;
  f.shift = 0;
  if (d <= 1) return f;
  int l = 0;
  while (((int64_t)1 << l) < d) ++l;
  const unsigned __int128 num = (unsigned __int128)1 << (31 + l);
  f.mul = (uint32_t)((num + (unsigned __int128)d - 1) / (unsigned __int128)d);
  f.shift = l - 1;
  return f;
}
__device__ __forceinline__ int fast_div(int v, const FastDiv& f) {
  return f.mul ? (int)(__umulhi((unsigned)v, f.mul) >> f.shift) : v;
}

struct BwdArgs {
  const float* grad_out;
  int64_t ld_grad;
  const int64_t* offsets;
  float* weights;
  float* state;
  float lr, eps, grad_scale;
  int32_t F, B;
  int32_t optimizer;
  int32_t pooled;
  int64_t n;
  uint64_t sentinel;  // key of ids that belong to a zero-row (padding) feature: sorted last, never updated
  // extended optimizers (tzk_opt_args): second state, Adam constants, clipping
  float* state2;
  const float* step;  // device scalar: iteration count t >= 1 of this update (bias correction)
  float beta1, beta2, weight_decay, max_gradient;   // LARS_SGD: beta1 = momentum, beta2 = eta (no moment decays there)
  float bc1, bc2;     // 1 - beta^t, filled in by init_bias_correction() at kernel start
  // peer mode (sharded step over peer memory, tzk_peer.cu): the sorted value is src_rank * idx_span + idx and the
  // gradient row lives in the SOURCE rank's published buffer grad_peer[src_rank] (already divided by the bag length
  // for MEAN pooling); idx = bag (pooled) or id position (sequence).  peer_w == 0: everything is local.
  int32_t peer_w;
  int32_t idx_span;
  int32_t w_f16;      // 1: `weights` is an arena of halfs (FP16 tables): rows are widened, updated in fp32, rounded back
  int32_t interleaved;  // 1: [weight row | state row] back to back (row stride 2 * dim): the first state of table row r is
                        // at weights + w_off + r * 2 dim + dim — one 128-B line per D = 16 row, written whole
  // v / B and v / idx_span for 0 <= v < 2^31 as a multiply-high + shift (the division by a run-time divisor was 20 % of
  // the kernel's instructions): mul == 0 means "divisor is 1"
  FastDiv div_b, div_span;
  int32_t ld32;         // = ld_grad (< 2^31, checked on the host): row offsets are ONE 32 x 32 -> 64-bit multiply
  int32_t wd_mode;      // row-wise Adagrad weight decay mode (tzk_opt_args.weight_decay_mode; read by finish_run_norm)
};

// Optimizer family of the run kernels, a template parameter chosen on the host.  kFamNorm: the updates whose step
// depends on norms over the whole row (LAMB, partial row-wise LAMB, LARS-SGD) and row-wise Adagrad with L2 / decoupled
// weight decay — two passes over the row with a group reduction in between (finish_run_norm).  Keeping them out of the
// kFamClassic instantiations leaves the register allocation of the classic optimizers' kernels as it was.
constexpr int kFamClassic = 0;
constexpr int kFamNorm = 1;
// peer mode: the sources' published gradient buffers.  A kernel parameter of its own (__grid_constant__): indexing it
// with a run-time rank must not drag the whole argument block into local memory.
struct PeerGrads { unsigned long long p[16]; };

template <int FAM = kFamClassic>
__device__ __forceinline__ void init_bias_correction(BwdArgs& a) {
  a.bc1 = a.bc2 = 1.f;
  const bool adam_like = FAM == kFamClassic
                             ? (a.optimizer == TZK_OPT_ADAM || a.optimizer == TZK_OPT_PARTIAL_ROWWISE_ADAM)
                             : (a.optimizer == TZK_OPT_LAMB || a.optimizer == TZK_OPT_PARTIAL_ROWWISE_LAMB);
  if (adam_like) {
    const float t = a.step ? __ldg(a.step) : 1.f;
    a.bc1 = 1.f - powf(a.beta1, t);
    a.bc2 = 1.f - powf(a.beta2, t);
  }
}

__device__ __forceinline__ void stage_feats(BwdFeat* fd, const int64_t* feat_w_off, const int64_t* feat_rows,
                                            const int64_t* feat_key_base, const int32_t* feat_dim,
                                            const int32_t* feat_col, const int32_t* feat_pool, int F,
                                            int interleaved = 0) {
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    fd[f].w_off = feat_w_off[f];
    fd[f].rows = feat_rows[f];
    fd[f].key_base = feat_key_base[f];
    fd[f].dim = feat_dim[f];
    fd[f].col = feat_col ? feat_col[f] : 0;
    fd[f].pool = feat_pool ? feat_pool[f] : 0;
    fd[f].stride = interleaved ? 2 * feat_dim[f] : feat_dim[f];
  }
  __syncthreads();
}

// ---- 1. linearize ------------------------------------------------------------------------------
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
linearize_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                 const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_key_base, int F,
                 int B, int pooled, KeyT sentinel, KeyT* __restrict__ keys, int32_t* __restrict__ vals) {
  const int64_t n_bags = (int64_t)F * B;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t bag = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; bag < n_bags; bag += stride) {
    const int f = (int)(bag / B);
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    const int64_t base = __ldg(feat_key_base + f), rows = __ldg(feat_rows + f);
    for (int64_t l = s; l < e; ++l) {
      int64_t id = __ldg(ids + l);
      if ((uint64_t)id >= (uint64_t)rows) id = 0;
      keys[l] = rows > 0 ? (KeyT)(base + id) : sentinel;
      vals[l] = pooled ? (int32_t)bag : (int32_t)l;
    }
  }
}

// sequence layout (pooled == 0): bags may be arbitrarily long (a whole (src,feature) segment when B == 1), so
// the work item is the id position and the feature comes from a binary search over the key boundaries.
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
linearize_seq_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                     const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_key_base, int F,
                     int B, int64_t n, KeyT sentinel, KeyT* __restrict__ keys, int32_t* __restrict__ vals) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int64_t* key_start = reinterpret_cast<int64_t*>(smem_raw);  // [F+1]
  int64_t* base = key_start + (F + 1);
  int64_t* rows = base + F;
  for (int f = threadIdx.x; f <= F; f += blockDim.x) key_start[f] = offsets[(int64_t)f * B];
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    base[f] = feat_key_base[f];
    rows[f] = feat_rows[f];
  }
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t l = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; l < n; l += stride) {
    int lo = 0, hi = F;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (key_start[mid] <= l) lo = mid; else hi = mid;
    }
    int64_t id = __ldg(ids + l);
    if ((uint64_t)id >= (uint64_t)rows[lo]) id = 0;
    keys[l] = rows[lo] > 0 ? (KeyT)(base[lo] + id) : sentinel;   // zero-row feature = wire padding
    vals[l] = (int32_t)l;
  }
}

// ---- 1w. weighted bags (per-sample weights): the sort value is the id position l, so that the weight of every sorted
// entry can be found; bag_of[l] keeps the bag.  After the sort, sorted_bag_weight_kernel turns each sorted value back into
// its bag and writes w[l] next to it (sw[i]) — both still in the id half, so the gradient half reads the weight of
// sorted position i as one more coalesced 4-B load instead of a dependent random one.  The sort is stable and l grows
// with the bag, so a run's entries keep the ascending-bag order of the unweighted sort.
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
linearize_weighted_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                          const int64_t* __restrict__ feat_rows, const int64_t* __restrict__ feat_key_base, int F,
                          int B, KeyT sentinel, KeyT* __restrict__ keys, int32_t* __restrict__ vals,
                          int32_t* __restrict__ bag_of) {
  const int64_t n_bags = (int64_t)F * B;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t bag = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; bag < n_bags; bag += stride) {
    const int f = (int)(bag / B);
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    const int64_t base = __ldg(feat_key_base + f), rows = __ldg(feat_rows + f);
    for (int64_t l = s; l < e; ++l) {
      int64_t id = __ldg(ids + l);
      if ((uint64_t)id >= (uint64_t)rows) id = 0;
      keys[l] = rows > 0 ? (KeyT)(base + id) : sentinel;
      vals[l] = (int32_t)l;
      bag_of[l] = (int32_t)bag;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
sorted_bag_weight_kernel(int32_t* __restrict__ vals, const int32_t* __restrict__ bag_of, const float* __restrict__ psw,
                         int64_t n, float* __restrict__ sw) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int32_t l = vals[i];
    vals[i] = __ldg(bag_of + l);
    sw[i] = __ldg(psw + l);
  }
}

// ---- 1'. peer mode: the owner reads its chunk of every source rank's wire buffers (tzk_peer.cu: destination-major,
// fixed capacity, counts per destination) straight into the sort's input.  Slot s = (src r, j): valid while j is below
// the count r published for this rank; the rest are padding (sentinel key: sorted last, never updated).
struct PeerWire {
  unsigned long long key[16], idx[16], cnt[16];   // per source rank: wire_key / wire_idx / counts as mapped here
  int32_t me, W;
  int64_t cap;
  int32_t idx_span, pad;
};

template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
peer_pull_linearize_kernel(const __grid_constant__ PeerWire pw, KeyT sentinel, KeyT* __restrict__ keys,
                           int32_t* __restrict__ vals, int32_t* __restrict__ overflow) {
  __shared__ int32_t cnt[16];
  if ((int)threadIdx.x < pw.W) {
    const int32_t* c = reinterpret_cast<const int32_t*>(pw.cnt[threadIdx.x]);
    cnt[threadIdx.x] = c[pw.me];
    if (blockIdx.x == 0 && overflow && c[pw.W]) atomicOr(overflow, 1);   // any source dropped ids -> every owner knows
  }
  __syncthreads();
  const int64_t n = (int64_t)pw.W * pw.cap;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; s < n; s += stride) {
    const int r = (int)((uint32_t)s / (uint32_t)pw.cap);          // W * cap < 2^31
    const int64_t j = s - (int64_t)r * pw.cap;
    KeyT k = sentinel;
    int32_t v = 0;
    if (j < cnt[r]) {
      k = (KeyT) reinterpret_cast<const int64_t*>(pw.key[r])[(int64_t)pw.me * pw.cap + j];
      // idx_span == 0 ("slot mode"): the gradient row of this entry was pushed to row s of the local receive buffer
      v = pw.idx_span > 0 ? r * pw.idx_span + reinterpret_cast<const int32_t*>(pw.idx[r])[(int64_t)pw.me * pw.cap + j]
                          : (int32_t)s;
    }
    keys[s] = k;
    vals[s] = v;
  }
}

// sample-owner half of the sharded backward: one gradient row per id position, written to its wire slot
__global__ void __launch_bounds__(kThreads)
bag_grad_expand_kernel(const float* __restrict__ grad_out, int64_t ld_grad, const int32_t* __restrict__ feat_col,
                       const int32_t* __restrict__ feat_pool, const int64_t* __restrict__ offsets,
                       const int32_t* __restrict__ slot, int F, int B, int D, float* __restrict__ g_rows) {
  const int D4 = D >> 2;  // D % 4 == 0 on this path (checked by the host wrapper), else scalar kernel below
  const int64_t n_items = (int64_t)F * B * D4;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += stride) {
    const int64_t bag = i / D4;
    const int c = (int)(i - bag * D4) * 4;
    const int f = (int)(bag / B);
    const int b = (int)(bag - (int64_t)f * B);
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    if (e == s) continue;
    float4 g = ld_row_f4(grad_out + (int64_t)b * ld_grad + __ldg(feat_col + f) + c);
    if (__ldg(feat_pool + f) == TZK_POOL_MEAN) g = f4_scale(g, 1.0f / (float)(e - s));
    for (int64_t l = s; l < e; ++l) st_stream_f4(g_rows + (int64_t)__ldg(slot + l) * D + c, g);
  }
}

__global__ void __launch_bounds__(kThreads)
bag_grad_expand_scalar_kernel(const float* __restrict__ grad_out, int64_t ld_grad,
                              const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                              const int64_t* __restrict__ offsets, const int32_t* __restrict__ slot, int F, int B,
                              int D, float* __restrict__ g_rows) {
  const int64_t n_items = (int64_t)F * B * D;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_items; i += stride) {
    const int64_t bag = i / D;
    const int c = (int)(i - bag * D);
    const int f = (int)(bag / B);
    const int b = (int)(bag - (int64_t)f * B);
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    if (e == s) continue;
    float g = __ldg(grad_out + (int64_t)b * ld_grad + __ldg(feat_col + f) + c);
    if (__ldg(feat_pool + f) == TZK_POOL_MEAN) g *= 1.0f / (float)(e - s);
    for (int64_t l = s; l < e; ++l) g_rows[(int64_t)__ldg(slot + l) * D + c] = g;
  }
}

// gradient-row address + scale of one sorted entry
struct Entry {
  const float* g;
  float scale;
  int f;
};

__device__ __forceinline__ Entry entry_of(const BwdArgs& a, const PeerGrads& gp, const BwdFeat* fd, int32_t v,
                                          int f_hint) {
  Entry en;
  const float* base = a.grad_out;
  if (a.peer_w) {
    const int r = fast_div(v, a.div_span);
    v -= r * a.idx_span;
    base = reinterpret_cast<const float*>(gp.p[r]);
  }
  if (a.pooled) {
    const int f = fast_div(v, a.div_b);
    const int b = v - f * a.B;
    en.f = f;
    en.g = base + (int64_t)b * a.ld32 + fd[f].col;
    en.scale = a.grad_scale;
    if (fd[f].pool == TZK_POOL_MEAN && !a.peer_w) {
      const int64_t L = __ldg(a.offsets + v + 1) - __ldg(a.offsets + v);
      en.scale = a.grad_scale / (float)L;  // L >= 1 because the entry exists
    }
  } else {
    en.f = f_hint;
    en.g = base + (int64_t)v * a.ld32;
    en.scale = a.grad_scale;
  }
  return en;
}

// feature of a sorted entry: from the bag index for pooled layouts, from the key ranges otherwise
__device__ __forceinline__ int bag_feat(const BwdArgs& a, int32_t v) {
  if (a.peer_w) v -= fast_div(v, a.div_span) * a.idx_span;
  return fast_div(v, a.div_b);
}

template <typename KeyT>
__device__ __forceinline__ int feat_of_key(const BwdFeat* fd, int F, KeyT key) {
  // features sharing a table share key_base; any of them gives the right table geometry
  int best = 0;
  int64_t best_base = -1;
  for (int f = 0; f < F; ++f) {
    const int64_t kb = fd[f].key_base;
    if (kb <= (int64_t)key && kb > best_base) { best = f; best_base = kb; }
  }
  return best;
}

// apply the optimizer to one chunk of a row.  `s` = first state (Adagrad accumulator / Adam first moment), `s2` =
// Adam second moment; `rw_denom` = the already computed per-row denominator of the row-wise variants.
// fbgemm formulas (App. A.10 and [EXT] split_embedding_optimizer_codegen):
//   ADAM                 m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; w -= lr (m^/(sqrt(v^)+eps) + wd w)
//   PARTIAL_ROWWISE_ADAM m element-wise as above, v one value per row from mean_d(g^2) (-> rw_denom)
template <int VEC>
__device__ __forceinline__ void apply_update(const BwdArgs& a, float* w, float* s, float* s2, const float* g,
                                             float rw_denom) {
#pragma unroll
  for (int k = 0; k < VEC; ++k) {
    const float gk = g[k];
    if (a.optimizer == TZK_OPT_SGD) {
      w[k] = w[k] - a.lr * gk;
    } else if (a.optimizer == TZK_OPT_ADAGRAD) {
      const float sk = s[k] + gk * gk;
      s[k] = sk;
      w[k] = w[k] - __fdividef(a.lr * gk, sqrtf(sk) + a.eps);   // (2-ulp quotient: the IEEE division was 10 % of the kernel)
    } else if (a.optimizer == TZK_OPT_ROWWISE_ADAGRAD) {
      w[k] = w[k] - a.lr * gk / rw_denom;
    } else if (a.optimizer == TZK_OPT_ADAM) {
      const float m = a.beta1 * s[k] + (1.f - a.beta1) * gk;
      const float v = a.beta2 * s2[k] + (1.f - a.beta2) * gk * gk;
      s[k] = m;
      s2[k] = v;
      w[k] = w[k] - a.lr * ((m / a.bc1) / (sqrtf(v / a.bc2) + a.eps) + a.weight_decay * w[k]);
    } else {  // TZK_OPT_PARTIAL_ROWWISE_ADAM
      const float m = a.beta1 * s[k] + (1.f - a.beta1) * gk;
      s[k] = m;
      w[k] = w[k] - a.lr * ((m / a.bc1) / rw_denom + a.weight_decay * w[k]);
    }
  }
}

template <int G>
__device__ __forceinline__ unsigned group_mask_of();
__device__ __forceinline__ float clip_grad(const BwdArgs& a, float g) {
  return a.max_gradient > 0.f ? fminf(fmaxf(g, -a.max_gradient), a.max_gradient) : g;
}
__device__ __forceinline__ bool has_elem_state(const BwdArgs& a) {   // first state laid out like the weights
  return a.optimizer == TZK_OPT_ADAGRAD || a.optimizer == TZK_OPT_ADAM || a.optimizer == TZK_OPT_PARTIAL_ROWWISE_ADAM;
}
// per-row denominator of the row-wise variants; `ss` = sum over the row of g^2 (already reduced over the lane group),
// lane 0 of the group owns the state element
template <int G>
__device__ __forceinline__ float rowwise_denom(const BwdArgs& a, int64_t key, float ss, int dim, int lane) {
  float d = 1.f;
  if (a.optimizer == TZK_OPT_ROWWISE_ADAGRAD) {
    float sr = 0.f;
    if (lane == 0) {
      sr = a.state[key] + ss / (float)dim;
      a.state[key] = sr;
    }
    sr = __shfl_sync(group_mask_of<G>(), sr, 0, G);
    d = sqrtf(sr) + a.eps;
  } else if (a.optimizer == TZK_OPT_PARTIAL_ROWWISE_ADAM) {
    float v = 0.f;
    if (lane == 0) {
      v = a.beta2 * a.state2[key] + (1.f - a.beta2) * (ss / (float)dim);
      a.state2[key] = v;
    }
    v = __shfl_sync(group_mask_of<G>(), v, 0, G);
    d = sqrtf(v / a.bc2) + a.eps;
  }
  return d;
}

// mask of the G lanes of this thread's lane group inside its warp (groups diverge independently)
template <int G>
__device__ __forceinline__ unsigned group_mask() {
  if (G >= 32) return 0xffffffffu;
  const unsigned lane_in_warp = threadIdx.x & 31u;
  return ((1u << G) - 1u) << (lane_in_warp / G * G);
}
template <int G>
__device__ __forceinline__ unsigned group_mask_of() { return group_mask<G>(); }
template <int G>
__device__ __forceinline__ float group_sum(float v) {
  const unsigned m = group_mask<G>();
#pragma unroll
  for (int d = G / 2; d >= 1; d >>= 1) v += __shfl_xor_sync(m, v, d, G);
  return v;
}

// first state laid out like the weights, per optimizer family
template <int FAM>
__device__ __forceinline__ bool elem_state(const BwdArgs& a) {
  if (FAM == kFamClassic) return has_elem_state(a);
  return a.optimizer == TZK_OPT_LAMB || a.optimizer == TZK_OPT_PARTIAL_ROWWISE_LAMB || a.optimizer == TZK_OPT_LARS_SGD;
}

template <int VEC>
__device__ __forceinline__ void unpack4(const float4& x, float (&v)[VEC]) {
  if constexpr (VEC == 4) {
    v[0] = x.x; v[1] = x.y; v[2] = x.z; v[3] = x.w;
  } else {
    v[0] = x.x;
  }
}
template <int VEC>
__device__ __forceinline__ void load_vec(const float* p, float (&v)[VEC]) {
  if constexpr (VEC == 4) unpack4<4>(*reinterpret_cast<const float4*>(p), v);
  else v[0] = p[0];
}
template <int VEC>
__device__ __forceinline__ void store_vec(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else p[0] = v[0];
}

// finish a run of the kFamNorm optimizers (fbgemm [EXT] split_embedding_optimizer_codegen, DESIGN.md §5); |.| is the L2
// norm over the row's D elements, mult = lr / (sqrt(s_row) + eps):
//   LAMB                 m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; u = m^/(sqrt(v^)+eps) + wd w ; w -= lr |w|/|u| u
//   PARTIAL_ROWWISE_LAMB m element-wise as LAMB, v one value per row from mean_d(g^2) ; u and the step as LAMB
//   LARS_SGD             lr' = lr eta |w| / (|g| + wd |w|) ; m = momentum m + lr' (g + wd w) ; w -= m
//   ROWWISE_ADAGRAD  L2  s_row += mean_d((g + wd w)^2) ; w = (1 - mult wd) w - mult g
//                    DEC s_row += mean_d(g^2)          ; w = (1 - lr wd) w - mult g
// Phase 1 widens this lane's chunks of the row into registers, updates the moments and forms u (LARS keeps g), adding
// up |w|^2 and |u|^2 (|g|^2); one group reduction; phase 2 applies the scaled step and stores the row.  The literal
// formulas hold for degenerate rows too (|u| = 0, or |g| + wd |w| = 0: the row becomes NaN / inf as the arithmetic says).
template <int G, int VEC, int CH>
__device__ __forceinline__ void finish_run_norm(const BwdArgs& a, const BwdFeat& d, int64_t row, int64_t key,
                                                float (&acc)[CH][VEC], int lane, const float4* pre_w,
                                                const float4* pre_s) {
  const int op = a.optimizer;
  const bool lamb = op == TZK_OPT_LAMB, pr_lamb = op == TZK_OPT_PARTIAL_ROWWISE_LAMB, lars = op == TZK_OPT_LARS_SGD;
  const bool rw_adagrad = op == TZK_OPT_ROWWISE_ADAGRAD;
  if (a.max_gradient > 0.f) {
#pragma unroll
    for (int ch = 0; ch < CH; ++ch)
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[ch][k] = clip_grad(a, acc[ch][k]);
  }
  const int64_t base = d.w_off + row * d.stride;
  float w[CH][VEC];
#pragma unroll
  for (int ch = 0; ch < CH; ++ch) {
    const int c = (ch * G + lane) * VEC;
#pragma unroll
    for (int k = 0; k < VEC; ++k) w[ch][k] = 0.f;
    if (c >= d.dim) continue;
    if (a.w_f16) {
      const __half* wph = reinterpret_cast<const __half*>(a.weights) + base + c;
      if constexpr (VEC == 4) {
        const uint2 raw = *reinterpret_cast<const uint2*>(wph);
        const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
        const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
        w[ch][0] = lo.x; w[ch][1] = lo.y; w[ch][2] = hi.x; w[ch][3] = hi.y;
      } else {
        w[ch][0] = __half2float(wph[0]);
      }
    } else if (pre_w) {
      unpack4<VEC>(*pre_w, w[ch]);
    } else {
      load_vec<VEC>(a.weights + base + c, w[ch]);
    }
  }
  // the row-wise second moment / accumulator: needs the row's sum of squares before u
  float rw_denom = 1.f;
  if (pr_lamb || rw_adagrad) {
    const float wd_l2 = (rw_adagrad && a.wd_mode == 1) ? a.weight_decay : 0.f;
    float ss = 0.f;
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      const int c = (ch * G + lane) * VEC;
#pragma unroll
      for (int k = 0; k < VEC; ++k)
        if (c + k < d.dim) {
          const float gk = acc[ch][k] + wd_l2 * w[ch][k];
          ss += gk * gk;
        }
    }
    ss = group_sum<G>(ss);
    float v = 0.f;
    if (lane == 0) {
      if (rw_adagrad) {
        v = a.state[key] + ss / (float)d.dim;
        a.state[key] = v;
      } else {
        v = a.beta2 * a.state2[key] + (1.f - a.beta2) * (ss / (float)d.dim);
        a.state2[key] = v;
      }
    }
    v = __shfl_sync(group_mask_of<G>(), v, 0, G);
    rw_denom = rw_adagrad ? sqrtf(v) + a.eps : sqrtf(v / a.bc2) + a.eps;
  }
  // phase 1: moments, u (in acc), |w|^2 and |u|^2 (LARS: |g|^2)
  float ww = 0.f, uu = 0.f;
  if (!rw_adagrad) {
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      const int c = (ch * G + lane) * VEC;
      if (c >= d.dim) continue;
      if (lamb || pr_lamb) {
        float* sp = a.state + base + c;
        float m[VEC];
        if (pre_s) unpack4<VEC>(*pre_s, m);
        else load_vec<VEC>(sp, m);
        float v[VEC];
        if (lamb) load_vec<VEC>(a.state2 + base + c, v);
#pragma unroll
        for (int k = 0; k < VEC; ++k) {
          const float gk = acc[ch][k];
          m[k] = a.beta1 * m[k] + (1.f - a.beta1) * gk;
          float den = rw_denom;
          if (lamb) {
            v[k] = a.beta2 * v[k] + (1.f - a.beta2) * gk * gk;
            den = sqrtf(v[k] / a.bc2) + a.eps;
          }
          acc[ch][k] = (m[k] / a.bc1) / den + a.weight_decay * w[ch][k];
        }
        store_vec<VEC>(sp, m);
        if (lamb) store_vec<VEC>(a.state2 + base + c, v);
      }
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        ww += w[ch][k] * w[ch][k];
        uu += acc[ch][k] * acc[ch][k];
      }
    }
    ww = group_sum<G>(ww);
    uu = group_sum<G>(uu);
  }
  // phase 2: the step
  float scale = 0.f, keep = 1.f, mult = 0.f;
  if (lamb || pr_lamb) {
    scale = a.lr * (sqrtf(ww) / sqrtf(uu));
  } else if (lars) {
    const float wn = sqrtf(ww);
    scale = a.lr * a.beta2 * wn / (sqrtf(uu) + a.weight_decay * wn);   // beta2 = eta
  } else {
    mult = a.lr / rw_denom;
    keep = a.wd_mode == 1 ? 1.f - mult * a.weight_decay : 1.f - a.lr * a.weight_decay;
  }
#pragma unroll
  for (int ch = 0; ch < CH; ++ch) {
    const int c = (ch * G + lane) * VEC;
    if (c >= d.dim) continue;
    if (lars) {
      float* sp = a.state + base + c;
      float m[VEC];
      if (pre_s) unpack4<VEC>(*pre_s, m);
      else load_vec<VEC>(sp, m);
#pragma unroll
      for (int k = 0; k < VEC; ++k) {
        m[k] = a.beta1 * m[k] + scale * (acc[ch][k] + a.weight_decay * w[ch][k]);   // beta1 = momentum
        w[ch][k] = w[ch][k] - m[k];
      }
      store_vec<VEC>(sp, m);
    } else if (rw_adagrad) {
#pragma unroll
      for (int k = 0; k < VEC; ++k) w[ch][k] = keep * w[ch][k] - mult * acc[ch][k];
    } else {
#pragma unroll
      for (int k = 0; k < VEC; ++k) w[ch][k] = w[ch][k] - scale * acc[ch][k];
    }
    if (a.w_f16) {      // round to nearest even, as the classic update
      __half* wph = reinterpret_cast<__half*>(a.weights) + base + c;
      if constexpr (VEC == 4) {
        uint2 raw;
        *reinterpret_cast<__half2*>(&raw.x) = __floats2half2_rn(w[ch][0], w[ch][1]);
        *reinterpret_cast<__half2*>(&raw.y) = __floats2half2_rn(w[ch][2], w[ch][3]);
        *reinterpret_cast<uint2*>(wph) = raw;
      } else {
        wph[0] = __float2half_rn(w[ch][0]);
      }
    } else {
      store_vec<VEC>(a.weights + base + c, w[ch]);
    }
  }
}

// finish a run: `acc` holds this lane's chunk(s) of the summed gradient.  Only called with all G lanes
// of the group active (needed for the row-wise shuffle).
// `pre_w` / `pre_s` (CH == 1, VEC == 4, fp32 tables): the row's weight / first-state chunk of this lane, already
// requested by the caller (next to the gradient rows instead of after them).
template <int G, int VEC, int CH, int FAM = kFamClassic>
__device__ __forceinline__ void finish_run(const BwdArgs& a, const BwdFeat& d, int64_t row, int64_t key,
                                           float (&acc)[CH][VEC], int lane, const float4* pre_w = nullptr,
                                           const float4* pre_s = nullptr) {
  if constexpr (FAM == kFamNorm) {
    finish_run_norm<G, VEC, CH>(a, d, row, key, acc, lane, pre_w, pre_s);
    return;
  }
  if (a.optimizer == TZK_OPT_ACCUM_OUT) {
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      const int c = (ch * G + lane) * VEC;
      if (c >= d.dim) continue;
      float* wp = a.weights + d.w_off + row * d.stride + c;
      if (VEC == 4) *reinterpret_cast<float4*>(wp) = make_float4(acc[ch][0], acc[ch][1], acc[ch][2], acc[ch][3]);
      else wp[0] = acc[ch][0];
    }
    if (lane == 0) reinterpret_cast<int32_t*>(a.state)[key] = 1;
    return;
  }
  if (a.max_gradient > 0.f) {
#pragma unroll
    for (int ch = 0; ch < CH; ++ch)
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[ch][k] = clip_grad(a, acc[ch][k]);
  }
  float rw_denom = 1.f;
  if (a.optimizer == TZK_OPT_ROWWISE_ADAGRAD || a.optimizer == TZK_OPT_PARTIAL_ROWWISE_ADAM) {
    float ss = 0.f;
#pragma unroll
    for (int ch = 0; ch < CH; ++ch) {
      const int c = (ch * G + lane) * VEC;
#pragma unroll
      for (int k = 0; k < VEC; ++k)
        if (c + k < d.dim) ss += acc[ch][k] * acc[ch][k];
    }
    ss = group_sum<G>(ss);
    rw_denom = rowwise_denom<G>(a, key, ss, d.dim, lane);
  }
  const bool es = has_elem_state(a);
  const bool es2 = a.optimizer == TZK_OPT_ADAM;
#pragma unroll
  for (int ch = 0; ch < CH; ++ch) {
    const int c = (ch * G + lane) * VEC;
    if (c >= d.dim) continue;
    const int64_t off = d.w_off + row * d.stride + c;
    float* wp = a.weights + off;
    __half* wph = reinterpret_cast<__half*>(a.weights) + off;       // (FP16 tables: same element offset, half the bytes)
    float* sp = es ? (a.interleaved ? wp + d.dim : a.state + off) : nullptr;
    float* sp2 = es2 ? a.state2 + off : nullptr;
    if (VEC == 4) {
      float4 w4;
      if (a.w_f16) {
        const uint2 raw = *reinterpret_cast<const uint2*>(wph);
        const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&raw.x));
        const float2 hi = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
        w4 = make_float4(lo.x, lo.y, hi.x, hi.y);
      } else {
        w4 = pre_w ? *pre_w : *reinterpret_cast<float4*>(wp);
      }
      float w[4] = {w4.x, w4.y, w4.z, w4.w};
      float s[4] = {0.f, 0.f, 0.f, 0.f};
      float s2[4] = {0.f, 0.f, 0.f, 0.f};
      if (sp) {
        float4 s4 = pre_s ? *pre_s : *reinterpret_cast<float4*>(sp);
        s[0] = s4.x; s[1] = s4.y; s[2] = s4.z; s[3] = s4.w;
      }
      if (sp2) {
        float4 s4 = *reinterpret_cast<float4*>(sp2);
        s2[0] = s4.x; s2[1] = s4.y; s2[2] = s4.z; s2[3] = s4.w;
      }
      apply_update<4>(a, w, s, s2, acc[ch], rw_denom);
      if (a.w_f16) {      // round to nearest even (fbgemm's optional stochastic rounding is not reproduced)
        uint2 raw;
        *reinterpret_cast<__half2*>(&raw.x) = __floats2half2_rn(w[0], w[1]);
        *reinterpret_cast<__half2*>(&raw.y) = __floats2half2_rn(w[2], w[3]);
        *reinterpret_cast<uint2*>(wph) = raw;
      } else {
        *reinterpret_cast<float4*>(wp) = make_float4(w[0], w[1], w[2], w[3]);
      }
      if (sp) *reinterpret_cast<float4*>(sp) = make_float4(s[0], s[1], s[2], s[3]);
      if (sp2) *reinterpret_cast<float4*>(sp2) = make_float4(s2[0], s2[1], s2[2], s2[3]);
    } else {
      float w[1] = {a.w_f16 ? __half2float(wph[0]) : wp[0]};
      float s[1] = {sp ? sp[0] : 0.f};
      float s2[1] = {sp2 ? sp2[0] : 0.f};
      apply_update<1>(a, w, s, s2, acc[ch], rw_denom);
      if (a.w_f16) wph[0] = __float2half_rn(w[0]); else wp[0] = w[0];
      if (sp) sp[0] = s[0];
      if (sp2) sp2[0] = s2[0];
    }
  }
}

template <int VEC>
__device__ __forceinline__ void load_grad(const float* p, float (&g)[VEC], int peer) {
  if (VEC == 4) {
    float4 v = peer ? ld_coh_f4(p) : ld_row_f4(p);   // peer memory: not through the non-coherent path
    g[0] = v.x; g[1] = v.y; g[2] = v.z; g[3] = v.w;
  } else {
    g[0] = peer ? *p : __ldg(p);
  }
}

// ---- 3. short runs ---------------------------------------------------------------------------------
// Work lists for runs longer than kShortRun (tiny tables, hot ids).  A long run is cut into chunks of kChunk
// sorted positions; one CTA reduces one chunk (4a).  Single-chunk runs are finished by that CTA; multi-chunk
// runs park per-chunk partial sums that 4b adds up in chunk order — so the result does not depend on which
// CTA ran what.
constexpr int kChunk = 256;
struct ChunkItem {
  int32_t start, end;   // sorted positions [start, end)
  int32_t n_chunks;     // chunks of the run
  int32_t pbase;        // multi-chunk runs: first partial slot of the run (-1 for single-chunk runs)
  int32_t cc;           // index of this chunk inside its run
  int32_t pad;
};
struct WorkLists {
  ChunkItem* items;
  int32_t* run_done;  // [partial slots] per multi-chunk run (indexed by pbase): chunks finished so far
  int32_t* counters;  // [0] items, [2] partial slots, [3] short-run heads
  float* partials;    // [slots][ROWF]
  // compact list of the SHORT runs (<= kShortRun positions): first sorted position and length of each, written by the id
  // half (find_long_runs_kernel) into the sort's dead input buffers; NULL: the gradient half walks every sorted position
  int32_t* head_pos;
  int32_t* head_len;
};

// ---- 2'. work list of the long runs (id half: runs right after the sort, on the side stream) ---------------------------
// A run head whose key repeats kShortRun positions further on is a long run: its end is found by gallop + binary search
// and its chunks are appended to the list.  (The list's order depends on scheduling; the results do not: a chunk's
// partial sum and the chunk order of the combine are fixed by the sorted positions.)
template <typename KeyT>
__global__ void __launch_bounds__(kThreads)
find_long_runs_kernel(const KeyT* __restrict__ keys, int64_t n, KeyT sentinel, WorkLists wl) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31u;
  // (every lane of a warp makes the same number of trips: the short-run list is appended with one atomic per warp)
  for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < n; base += stride) {
    const int64_t p = base + threadIdx.x;
    bool is_head = false, is_long = false, starts = false;
    KeyT k0 = 0;
    if (p < n) {
      k0 = keys[p];
      starts = !(p > 0 && keys[p - 1] == k0);               // first position of a run of equal keys (sentinel runs too)
      is_head = starts && k0 != sentinel;
      is_long = is_head && p + kShortRun < n && keys[p + kShortRun] == k0;
    }
    if (wl.head_pos) {
      const bool is_short = is_head && !is_long;
      // a short run ends where the next run starts: inside the warp's 32 consecutive positions that is a bit scan over
      // the ballot of run starts; only runs that reach past the warp's last position scan forward
      const unsigned starts_m = __ballot_sync(0xffffffffu, starts || p >= n);
      int len = 1;
      if (is_short) {
        const unsigned later = lane == 31 ? 0u : (starts_m >> (lane + 1)) << (lane + 1);
        if (later) {
          len = (__ffs(later) - 1) - (int)lane;
        } else {
          len = 32 - (int)lane;
          while (p + len < n && keys[p + len] == k0) ++len;   // <= kShortRun in all
        }
      }
      const unsigned m = __ballot_sync(0xffffffffu, is_short);
      int wbase = 0;
      if (lane == 0 && m) wbase = atomicAdd(wl.counters + 3, __popc(m));
      wbase = __shfl_sync(0xffffffffu, wbase, 0);
      if (is_short) {
        const int idx = wbase + __popc(m & ((1u << lane) - 1u));
        wl.head_pos[idx] = (int32_t)p;
        wl.head_len[idx] = len;
      }
    }
    if (!is_long) continue;
    int64_t lo = p + kShortRun, step = kShortRun;  // keys[lo] == k0
    int64_t hi = lo + step;
    while (hi < n && keys[hi] == k0) { lo = hi; step <<= 1; hi = lo + step; }
    if (hi > n) hi = n;
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] == k0) lo = mid; else hi = mid;
    }
    const int64_t end = hi;
    const int n_chunks = (int)((end - p + kChunk - 1) / kChunk);
    const int base_i = atomicAdd(wl.counters + 0, n_chunks);
    int pbase = -1;
    if (n_chunks > 1) {
      pbase = atomicAdd(wl.counters + 2, n_chunks);
      wl.run_done[pbase] = 0;
    }
    for (int cc = 0; cc < n_chunks; ++cc) {
      ChunkItem it;
      it.start = (int32_t)(p + (int64_t)cc * kChunk);
      it.end = (int32_t)((p + (int64_t)(cc + 1) * kChunk) < end ? (p + (int64_t)(cc + 1) * kChunk) : end);
      it.n_chunks = n_chunks;
      it.pbase = pbase;
      it.cc = cc;
      it.pad = 0;
      wl.items[base_i + cc] = it;
    }
  }
}

// CH = float4 (or scalar) chunks per lane: dims up to G*VEC*CH are supported.
// Each lane group owns kPos consecutive sorted positions per iteration.  Runs of length 1 (the common case on
// big tables) take a batched path: the gradient / weight / state rows of all of them are requested before any
// is consumed, so a group keeps 3*kPos independent 64-B requests in flight instead of one dependent chain.
// One short run (<= kShortRun sorted positions starting at p, key k0, first value v0): sum its gradient rows in sorted
// order, ONE optimizer update.  All G lanes of the group call it together.
// WTD: weighted bags — sw[i] is the per-sample weight of sorted position i (sorted_bag_weight_kernel); it multiplies
// the entry's scale.
template <typename KeyT, int G, int VEC, int CH, int FAM, bool WTD = false>
__device__ __forceinline__ void short_run(const BwdArgs& a, const PeerGrads& gp, const BwdFeat* fd,
                                          const int32_t* __restrict__ vals, int64_t p, KeyT k0, int32_t v0, int len,
                                          int lane, const float* __restrict__ sw = nullptr) {
        int f00;
    if (a.pooled) f00 = bag_feat(a, v0); else f00 = feat_of_key<KeyT>(fd, a.F, k0);
    const BwdFeat d = fd[f00];
    const int64_t row = (int64_t)k0 - d.key_base;
    // the row's weight / state chunks depend on the key only: requested here, next to the gradient rows, so that a
    // single-position run costs ONE exposed DRAM latency instead of two dependent ones
    constexpr bool kPre = (VEC == 4 && CH == 1);
    float4 pre_w = make_float4(0.f, 0.f, 0.f, 0.f), pre_s = pre_w;
    const bool pre = kPre && !a.w_f16 && a.optimizer != TZK_OPT_ACCUM_OUT;      // (group-uniform)
    if (pre && lane * 4 < d.dim) {
      const float* wp = a.weights + d.w_off + row * d.stride + lane * 4;
      pre_w = ld_rw_f4(wp);
      if (elem_state<FAM>(a)) pre_s = ld_rw_f4(a.interleaved ? wp + d.dim : a.state + (d.w_off + row * d.stride + lane * 4));
    }
    float acc[CH][VEC];
#pragma unroll
    for (int ch = 0; ch < CH; ++ch)
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[ch][k] = 0.f;
    // kGU gradient rows of the run in flight; added in sorted order
    constexpr int kGU = 4;
    for (int j0 = 0; j0 < len; j0 += kGU) {
      Entry en[kGU];
      bool ok[kGU];
#pragma unroll
      for (int q = 0; q < kGU; ++q) {
        const int j = j0 + q;
        ok[q] = j < len;
        en[q] = entry_of(a, gp, fd, (j == 0 || !ok[q]) ? v0 : vals[p + j], f00);
        if (WTD && ok[q]) en[q].scale *= __ldg(sw + p + j);
      }
#pragma unroll
      for (int ch = 0; ch < CH; ++ch) {
        const int c = (ch * G + lane) * VEC;
        if (c < d.dim) {
          float gg[kGU][VEC];
#pragma unroll
          for (int q = 0; q < kGU; ++q) {
            if (ok[q]) {
              load_grad<VEC>(en[q].g + c, gg[q], a.peer_w);
            } else {
#pragma unroll
              for (int k = 0; k < VEC; ++k) gg[q][k] = 0.f;
            }
          }
#pragma unroll
          for (int q = 0; q < kGU; ++q)
            if (ok[q]) {
#pragma unroll
              for (int k = 0; k < VEC; ++k) acc[ch][k] += gg[q][k] * en[q].scale;
            }
        }
      }
    }
    // (one call site: the row-wise variants shuffle inside, every lane of the group must arrive at the same instruction)
    finish_run<G, VEC, CH, FAM>(a, d, row, (int64_t)k0, acc, lane, pre ? &pre_w : nullptr,
                                (pre && elem_state<FAM>(a)) ? &pre_s : nullptr);
}

template <typename KeyT, int G, int VEC, int CH, int FAM, bool WTD = false>
__device__ __forceinline__ void run_update_body(const BwdArgs& a, const PeerGrads& gp, const BwdFeat* fd,
                                                const KeyT* __restrict__ keys,
                                                const int32_t* __restrict__ vals, const WorkLists& wl, int cta,
                                                int n_ctas, const float* __restrict__ sw = nullptr) {
  constexpr int NG = kThreads / G;
  const int lane = threadIdx.x % G;
  const int64_t stride = (int64_t)n_ctas * NG;
  // all G lanes of a group follow the same control flow (positions, keys, run lengths are group-uniform)
  if (wl.head_pos) {
    // the id half left a compact list of the short runs: no neighbour compares, no length scan, no iterations spent on
    // the ~60 % of the sorted positions that do not start a run
    const int64_t n_heads = wl.counters[3];
    int64_t h = (int64_t)cta * NG + threadIdx.x / G;
    int32_t hp = 0, hl = 0;
    if (h < n_heads) { hp = wl.head_pos[h]; hl = wl.head_len[h]; }
    for (; h < n_heads; h += stride) {
      const int64_t p = hp;
      const int len = hl;
      if (h + stride < n_heads) { hp = wl.head_pos[h + stride]; hl = wl.head_len[h + stride]; }   // next head, early
      short_run<KeyT, G, VEC, CH, FAM, WTD>(a, gp, fd, vals, p, keys[p], vals[p], len, lane, sw);
    }
    return;
  }
  // One sorted position per lane group and iteration (2 and 4 positions with a batched single-run path were slower on
  // DLRM-Criteo).  The keys / value of the NEXT position are
  // requested before the current one is worked on.
  int64_t p0 = (int64_t)cta * NG + threadIdx.x / G;
  KeyT kl = 0, kc = 0, kr = 0;     // left neighbour, this position, right neighbour
  int32_t vc = 0;
  auto fetch = [&](int64_t p, KeyT& l, KeyT& c, KeyT& r, int32_t& vv) {
    if (p < a.n) {
      c = keys[p];
      l = p > 0 ? keys[p - 1] : (KeyT)~c;
      r = p + 1 < a.n ? keys[p + 1] : (KeyT)~c;
      vv = vals[p];
    }
  };
  fetch(p0, kl, kc, kr, vc);
  for (; p0 < a.n; p0 += stride) {
    KeyT nl = 0, nc = 0, nr = 0;
    int32_t nv = 0;
    fetch(p0 + stride, nl, nc, nr, nv);
    const KeyT key_l = kl, key_c = kc, key_r = kr;
    const int32_t v_c = vc;
    kl = nl; kc = nc; kr = nr; vc = nv;
    // every run head: sum the run (<= kShortRun) in sorted order and update; long runs are on the work list
    // (find_long_runs_kernel, id half) for the chunk CTAs
    if (key_c == key_l || key_c == (KeyT)a.sentinel) continue;
    int len = 1;
    if (key_r == key_c) {
      len = 2;
      while (len <= kShortRun && p0 + len < a.n && keys[p0 + len] == key_c) ++len;
    }
    if (len > kShortRun) continue;
    short_run<KeyT, G, VEC, CH, FAM, WTD>(a, gp, fd, vals, p0, key_c, v_c, len, lane, sw);
  }
}

// ---- 4. one WARP per chunk of a long run ----------------------------------------------------------------------
// 32/G lane groups stride over the chunk with kLU gradient rows in flight each, then a fixed-order shuffle tree folds
// the groups' partial sums into group 0, which either finishes the run or parks the chunk's partial.  The warp that
// parks the LAST partial of a multi-chunk run (a counter per run) adds the run's partials in chunk order and applies
// the update — the order of the additions is fixed by the sorted positions, whoever happens to execute them.
// These CTAs ride in the same launch as the short-run CTAs (fused_apply_kernel): tiny tables / hot ids and the big
// tables' rows are updated side by side instead of in three dependent launches.
template <typename KeyT, int G, int VEC, int CH, int FAM, bool WTD = false>
__device__ __forceinline__ void long_chunk_body(const BwdArgs& a, const PeerGrads& gp, const BwdFeat* fd,
                                                const KeyT* __restrict__ keys,
                                                const int32_t* __restrict__ vals, const WorkLists& wl, int cta,
                                                int n_ctas, const float* __restrict__ sw = nullptr) {
  constexpr int GW = 32 / G;          // lane groups per warp
  constexpr int ROWF = CH * G * VEC;  // floats per partial row
  constexpr int kLU = 4;              // independent gradient rows in flight per lane group
  const int lane = threadIdx.x % G;
  const int gw = (threadIdx.x & 31) / G;
  const int warp = threadIdx.x >> 5;
  constexpr int WPC = kThreads / 32;
  const int n_items = wl.counters[0];

  for (int r = cta * WPC + warp; r < n_items; r += n_ctas * WPC) {
    const ChunkItem it = wl.items[r];
    const KeyT key = keys[it.start];
    const int32_t v0 = vals[it.start];
    int f0;
    if (a.pooled) f0 = bag_feat(a, v0); else f0 = feat_of_key<KeyT>(fd, a.F, key);
    const BwdFeat d = fd[f0];
    const int64_t row = (int64_t)key - d.key_base;

    float acc[CH][VEC];
#pragma unroll
    for (int ch = 0; ch < CH; ++ch)
#pragma unroll
      for (int k = 0; k < VEC; ++k) acc[ch][k] = 0.f;
    for (int q0 = it.start + gw; q0 < it.end; q0 += GW * kLU) {
      Entry en[kLU];
      bool ok[kLU];
#pragma unroll
      for (int u = 0; u < kLU; ++u) {
        const int q = q0 + u * GW;
        ok[u] = q < it.end;
        en[u] = entry_of(a, gp, fd, ok[u] ? vals[q] : v0, f0);
        if (WTD && ok[u]) en[u].scale *= __ldg(sw + q);
      }
#pragma unroll
      for (int ch = 0; ch < CH; ++ch) {
        const int c = (ch * G + lane) * VEC;
        if (c < d.dim) {
          float gr[kLU][VEC];
#pragma unroll
          for (int u = 0; u < kLU; ++u) load_grad<VEC>(en[u].g + c, gr[u], a.peer_w);
#pragma unroll
          for (int u = 0; u < kLU; ++u)
            if (ok[u]) {
#pragma unroll
              for (int k = 0; k < VEC; ++k) acc[ch][k] += gr[u][k] * en[u].scale;
            }
        }
      }
    }
    // fixed-order tree over the GW lane groups of the warp (whole warp participates)
#pragma unroll
    for (int off = GW / 2; off >= 1; off >>= 1) {
#pragma unroll
      for (int ch = 0; ch < CH; ++ch)
#pragma unroll
        for (int k = 0; k < VEC; ++k) acc[ch][k] += __shfl_down_sync(0xffffffffu, acc[ch][k], off * G);
    }
    if (gw == 0) {
      if (it.n_chunks == 1) {
        finish_run<G, VEC, CH, FAM>(a, d, row, (int64_t)key, acc, lane);
      } else {
        float* dst = wl.partials + (int64_t)(it.pbase + it.cc) * ROWF;
#pragma unroll
        for (int ch = 0; ch < CH; ++ch)
#pragma unroll
          for (int k = 0; k < VEC; ++k) dst[(ch * G + lane) * VEC + k] = acc[ch][k];
        __threadfence();                                    // this chunk's partial is visible before the count moves
        int done = 0;
        if (lane == 0) done = atomicAdd(wl.run_done + it.pbase, 1);
        done = __shfl_sync(group_mask<G>(), done, 0, G);
        if (done == it.n_chunks - 1) {                      // last chunk of the run: combine in chunk order, update
          __threadfence();
#pragma unroll
          for (int ch = 0; ch < CH; ++ch)
#pragma unroll
            for (int k = 0; k < VEC; ++k) acc[ch][k] = 0.f;
          for (int c = 0; c < it.n_chunks; ++c) {
            const float* src = wl.partials + (int64_t)(it.pbase + c) * ROWF;
#pragma unroll
            for (int ch = 0; ch < CH; ++ch)
#pragma unroll
              for (int k = 0; k < VEC; ++k) acc[ch][k] += __ldcg(src + (ch * G + lane) * VEC + k);
          }
          finish_run<G, VEC, CH, FAM>(a, d, row, (int64_t)key, acc, lane);
          if (lane == 0) wl.run_done[it.pbase] = 0;         // the list can be replayed (same sort, another gradient)
        }
      }
    }
    __syncwarp();
  }
}

// ---- 3 + 4 in one launch: CTAs [0, n_short) walk the sorted positions (short runs), the rest serve the long-run list
template <typename KeyT, int G, int VEC, int CH, int FAM>
__global__ void __launch_bounds__(kThreads, CH == 1 ? 4 : 1)     // 4 CTAs / SM: 64 registers (weight / state prefetch + 2 gradient rows in flight)
fused_apply_kernel(BwdArgs a, const int64_t* __restrict__ feat_w_off, const int64_t* __restrict__ feat_rows,
                   const int64_t* __restrict__ feat_key_base, const int32_t* __restrict__ feat_dim,
                   const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                   const KeyT* __restrict__ keys, const int32_t* __restrict__ vals, WorkLists wl, int n_long,
                   const __grid_constant__ PeerGrads gp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdFeat* fd = reinterpret_cast<BwdFeat*>(smem_raw);
  stage_feats(fd, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, a.F, a.interleaved);
  init_bias_correction<FAM>(a);
  // the long-run CTAs come FIRST in the grid: they are few, each has a lot to do, and the hardware starts CTAs in
  // index order — their work overlaps the whole short-run sweep instead of trailing it
  if ((int)blockIdx.x < n_long) long_chunk_body<KeyT, G, VEC, CH, FAM>(a, gp, fd, keys, vals, wl, blockIdx.x, n_long);
  else run_update_body<KeyT, G, VEC, CH, FAM>(a, gp, fd, keys, vals, wl, blockIdx.x - n_long, gridDim.x - n_long);
}

// the same launch for weighted bags: sw = the sorted per-sample weights the id half left in the workspace
template <typename KeyT, int G, int VEC, int CH, int FAM>
__global__ void __launch_bounds__(kThreads, CH == 1 ? 2 : 1)    // (2 CTAs / SM: at 64 and 80 registers the weighted runs spilled)
fused_apply_weighted_kernel(BwdArgs a, const int64_t* __restrict__ feat_w_off, const int64_t* __restrict__ feat_rows,
                            const int64_t* __restrict__ feat_key_base, const int32_t* __restrict__ feat_dim,
                            const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                            const KeyT* __restrict__ keys, const int32_t* __restrict__ vals, WorkLists wl, int n_long,
                            const __grid_constant__ PeerGrads gp, const float* __restrict__ sw) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdFeat* fd = reinterpret_cast<BwdFeat*>(smem_raw);
  stage_feats(fd, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, a.F, a.interleaved);
  init_bias_correction<FAM>(a);
  if ((int)blockIdx.x < n_long)
    long_chunk_body<KeyT, G, VEC, CH, FAM, true>(a, gp, fd, keys, vals, wl, blockIdx.x, n_long, sw);
  else
    run_update_body<KeyT, G, VEC, CH, FAM, true>(a, gp, fd, keys, vals, wl, blockIdx.x - n_long, gridDim.x - n_long, sw);
}

// ---- 3'. tile path: rows of <= 128 floats, 16-B aligned (vec4, one chunk per lane) -------------------------
// The sorted positions are cut into tiles of TP = 4096 / ROWF positions (ROWF = 4*G floats per padded row), one CTA
// per tile:
//   A. keys (+ both neighbours) and vals of the tile -> shared memory (coalesced);
//   B. every lane group loads the gradient rows of its U = 4 positions (independent 16-B loads, scaled) into a
//      shared-memory tile AND, for positions that head a run which lives entirely inside the tile, the weight and
//      state rows — so all global requests of a tile are in flight together instead of one dependent chain per run;
//   C. run heads add their run up from shared memory in sorted (= ascending bag) order and apply ONE update.
// A run that crosses a tile border leaves its partial sum in carry_first[t] (run entered from the left and ends
// here) or carry_last[t] (run leaves to the right; a tile that is one single key from border to border counts as
// "leaves to the right"); carry_combine_kernel adds the partials of such a run in tile order and updates the row.
// No atomics, summation order fixed by the sort -> run-to-run deterministic.
template <int G>
struct TileCfg {
  static constexpr int ROWF = G * 4;
  static constexpr int TP = 4096 / ROWF;
  static constexpr int NG = kThreads / G;
  static constexpr int U = TP / NG;  // = 4 for every G
};

inline int64_t tile_carry_floats(int64_t n, int rowf) {  // per carry array
  const int tp = 4096 / rowf;
  return ((n + tp - 1) / tp + 1) * rowf;
}

template <typename KeyT, int G>
__global__ void __launch_bounds__(kThreads, 3)
tile_update_kernel(BwdArgs a, const int64_t* __restrict__ feat_w_off, const int64_t* __restrict__ feat_rows,
                   const int64_t* __restrict__ feat_key_base, const int32_t* __restrict__ feat_dim,
                   const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                   const KeyT* __restrict__ keys, const int32_t* __restrict__ vals,
                   float* __restrict__ carry_first, float* __restrict__ carry_last,
                   const __grid_constant__ PeerGrads gp) {
  using C = TileCfg<G>;
  constexpr int ROWF = C::ROWF, TP = C::TP, NG = C::NG, U = C::U;
  constexpr int KPT = (TP + 2 + kThreads - 1) / kThreads;  // keys per thread (tile + both neighbours)
  constexpr int VPT = (TP + kThreads - 1) / kThreads;      // vals per thread
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* rows = reinterpret_cast<float*>(smem_raw);                      // [TP][ROWF]
  KeyT* sk = reinterpret_cast<KeyT*>(rows + TP * ROWF);                   // [TP + 2]: left nb, tile, right nb
  int32_t* sv = reinterpret_cast<int32_t*>(sk + (TP + 2));                // [TP]
  BwdFeat* fd = reinterpret_cast<BwdFeat*>(smem_raw + align16((size_t)TP * ROWF * 4 + (TP + 2) * sizeof(KeyT) + TP * 4));
  stage_feats(fd, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, a.F);
  init_bias_correction(a);

  const int lane = threadIdx.x % G, grp = threadIdx.x / G;
  const int c = lane * 4;
  const KeyT sentinel = (KeyT)a.sentinel;
  const int64_t n_tiles = (a.n + TP - 1) / TP;

  // keys / vals of a tile travel global -> registers -> shared memory; the loads of tile t+grid are issued before
  // tile t is processed, so their latency hides behind phases B and C
  KeyT pk[KPT];
  int32_t pv[VPT];
  auto prefetch = [&](int64_t t) {
    const int64_t base = t * TP;
#pragma unroll
    for (int q = 0; q < KPT; ++q) {
      const int64_t p = base + threadIdx.x + q * kThreads - 1;
      pk[q] = (t < n_tiles && threadIdx.x + q * kThreads < TP + 2 && p >= 0 && p < a.n) ? keys[p] : sentinel;
    }
#pragma unroll
    for (int q = 0; q < VPT; ++q) {
      const int64_t p = base + threadIdx.x + q * kThreads;
      pv[q] = (t < n_tiles && threadIdx.x + q * kThreads < TP && p < a.n) ? vals[p] : 0;
    }
  };
  prefetch(blockIdx.x);

  for (int64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const int64_t base = t * TP;
    const int cnt = (int)((a.n - base) < TP ? (a.n - base) : TP);
    // ---- A: registers -> shared memory ----------------------------------------------------------------
#pragma unroll
    for (int q = 0; q < KPT; ++q)
      if (threadIdx.x + q * kThreads < TP + 2) sk[threadIdx.x + q * kThreads] = pk[q];
#pragma unroll
    for (int q = 0; q < VPT; ++q)
      if (threadIdx.x + q * kThreads < TP) sv[threadIdx.x + q * kThreads] = pv[q];
    __syncthreads();
    prefetch(t + gridDim.x);
    const KeyT k_first = sk[1], k_last = sk[cnt];
    const bool first_cont = (t > 0) && sk[0] == k_first;
    const bool last_cont = (base + cnt < a.n) && sk[cnt + 1] == k_last;
    // ---- B: all global requests of the tile ------------------------------------------------------------
    float4 w4[U], s4[U], g4[U];
    int kind[U], fx[U];    // kind: 0 none, 1 -> carry_first, 2 -> carry_last, 3 -> update here
    bool multi[U];         // run head whose run has more than one position inside the tile
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = grp + NG * u;
      kind[u] = 0;
      fx[u] = 0;
      multi[u] = false;
      w4[u] = make_float4(0.f, 0.f, 0.f, 0.f);
      s4[u] = w4[u];
      g4[u] = w4[u];
      if (i >= cnt) continue;
      const KeyT key = sk[i + 1];
      if (key == sentinel) continue;
      const int32_t v = sv[i];
      const int f = a.pooled ? bag_feat(a, v) : feat_of_key<KeyT>(fd, a.F, key);
      fx[u] = f;
      const int dim = fd[f].dim;
      const Entry en = entry_of(a, gp, fd, v, f);
      if (c < dim) g4[u] = f4_scale(a.peer_w ? ld_coh_f4(en.g + c) : ld_row_f4(en.g + c), en.scale);
      if (i == 0 || sk[i] != key) {
        const bool cl = (i == 0) && first_cont;
        const bool cr = (key == k_last) && last_cont;
        kind[u] = cr ? 2 : (cl ? 1 : 3);
        multi[u] = (i + 1 < cnt) && sk[i + 2] == key;
        if (kind[u] == 3 && c < dim) {
          const int64_t off = fd[f].w_off + ((int64_t)key - fd[f].key_base) * dim + c;
          w4[u] = ld_rw_f4(a.weights + off);
          if (has_elem_state(a)) s4[u] = ld_rw_f4(a.state + off);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = grp + NG * u;
      if (i < cnt) *reinterpret_cast<float4*>(rows + i * ROWF + c) = g4[u];
    }
    __syncthreads();
    // ---- C: in-tile segmented reduction, three levels (8 / 64 / tile), fixed order -------------------------
    // level 1: positions that start a run or an aligned block of 8 add up their block-of-8 part of the run
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = grp + NG * u;
      if (i >= cnt) continue;
      const KeyT key = sk[i + 1];
      if (key == sentinel) continue;
      const bool head = (i == 0) || sk[i] != key;
      if (!(head || (i & 7) == 0)) continue;
      if (!(i + 1 < cnt && ((i + 1) & 7) != 0 && sk[i + 2] == key)) continue;
      float4 acc = *reinterpret_cast<const float4*>(rows + i * ROWF + c);
      for (int j = i + 1; j < cnt && (j & 7) != 0 && sk[j + 1] == key; ++j)
        acc = f4_add(acc, *reinterpret_cast<const float4*>(rows + j * ROWF + c));
      *reinterpret_cast<float4*>(rows + i * ROWF + c) = acc;
    }
    __syncthreads();
    // level 2: run starts / aligned blocks of 64 add the block-of-8 partials of their part of the run
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = grp + NG * u;
      if (i >= cnt) continue;
      const KeyT key = sk[i + 1];
      if (key == sentinel) continue;
      const bool head = (i == 0) || sk[i] != key;
      if (!(head || (i & 63) == 0)) continue;
      int j = (i | 7) + 1;
      if (!(j < cnt && (j & 63) != 0 && sk[j + 1] == key)) continue;
      float4 acc = *reinterpret_cast<const float4*>(rows + i * ROWF + c);
      for (; j < cnt && (j & 63) != 0 && sk[j + 1] == key; j += 8)
        acc = f4_add(acc, *reinterpret_cast<const float4*>(rows + j * ROWF + c));
      *reinterpret_cast<float4*>(rows + i * ROWF + c) = acc;
    }
    __syncthreads();
    // level 3: run heads add the block-of-64 partials, then update / park the sum
#pragma unroll
    for (int u = 0; u < U; ++u) {
      if (kind[u] == 0) continue;
      const int i = grp + NG * u;
      const KeyT key = sk[i + 1];
      float4 acc = *reinterpret_cast<const float4*>(rows + i * ROWF + c);
      if (multi[u]) {
        for (int j = (i | 63) + 1; j < cnt && sk[j + 1] == key; j += 64)
          acc = f4_add(acc, *reinterpret_cast<const float4*>(rows + j * ROWF + c));
      }
      if (kind[u] == 1) {
        *reinterpret_cast<float4*>(carry_first + t * ROWF + c) = acc;
      } else if (kind[u] == 2) {
        *reinterpret_cast<float4*>(carry_last + t * ROWF + c) = acc;
      } else {
        const BwdFeat& d = fd[fx[u]];
        float g[4] = {clip_grad(a, acc.x), clip_grad(a, acc.y), clip_grad(a, acc.z), clip_grad(a, acc.w)};
        float rw_denom = 1.f;
        if (a.optimizer == TZK_OPT_ROWWISE_ADAGRAD || a.optimizer == TZK_OPT_PARTIAL_ROWWISE_ADAM) {
          float ss = g[0] * g[0] + g[1] * g[1] + g[2] * g[2] + g[3] * g[3];  // lanes beyond the row hold zeros
          ss = group_sum<G>(ss);
          rw_denom = rowwise_denom<G>(a, (int64_t)key, ss, d.dim, lane);
        }
        if (c < d.dim) {
          const int64_t off = d.w_off + ((int64_t)key - d.key_base) * d.dim + c;
          float w[4] = {w4[u].x, w4[u].y, w4[u].z, w4[u].w};
          float s[4] = {s4[u].x, s4[u].y, s4[u].z, s4[u].w};
          float s2[4] = {0.f, 0.f, 0.f, 0.f};
          if (a.optimizer == TZK_OPT_ADAM) {
            const float4 v4 = ld_rw_f4(a.state2 + off);
            s2[0] = v4.x; s2[1] = v4.y; s2[2] = v4.z; s2[3] = v4.w;
          }
          apply_update<4>(a, w, s, s2, g, rw_denom);
          *reinterpret_cast<float4*>(a.weights + off) = make_float4(w[0], w[1], w[2], w[3]);
          if (has_elem_state(a))
            *reinterpret_cast<float4*>(a.state + off) = make_float4(s[0], s[1], s[2], s[3]);
          if (a.optimizer == TZK_OPT_ADAM)
            *reinterpret_cast<float4*>(a.state2 + off) = make_float4(s2[0], s2[1], s2[2], s2[3]);
        }
      }
    }
    __syncthreads();  // the next tile overwrites sk / sv / rows
  }
}

// one lane group per tile border: if a run crosses it and STARTS in the tile left of it, add the run's per-tile
// partials in tile order (carry_last[t], carry_last of every tile the key fills completely, carry_first of the
// tile it ends in) and update the row.
template <typename KeyT, int G>
__global__ void __launch_bounds__(kThreads)
carry_combine_kernel(BwdArgs a, const int64_t* __restrict__ feat_w_off, const int64_t* __restrict__ feat_rows,
                     const int64_t* __restrict__ feat_key_base, const int32_t* __restrict__ feat_dim,
                     const int32_t* __restrict__ feat_col, const int32_t* __restrict__ feat_pool,
                     const KeyT* __restrict__ keys, const int32_t* __restrict__ vals,
                     const float* __restrict__ carry_first, const float* __restrict__ carry_last) {
  using C = TileCfg<G>;
  constexpr int ROWF = C::ROWF, TP = C::TP, NG = C::NG;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdFeat* fd = reinterpret_cast<BwdFeat*>(smem_raw);
  stage_feats(fd, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, a.F);
  init_bias_correction(a);
  const int lane = threadIdx.x % G;
  const int c = lane * 4;
  const KeyT sentinel = (KeyT)a.sentinel;
  const int64_t n_tiles = (a.n + TP - 1) / TP;
  for (int64_t t = (int64_t)blockIdx.x * NG + threadIdx.x / G; t + 1 < n_tiles; t += (int64_t)gridDim.x * NG) {
    const int64_t pe = (t + 1) * TP;  // first position of tile t+1 (< n)
    const KeyT k0 = keys[pe - 1];
    if (keys[pe] != k0 || k0 == sentinel) continue;
    const int64_t ps = t * TP;
    if (t > 0 && keys[ps] == k0 && keys[ps - 1] == k0) continue;  // the run started further left
    // end of the run: gallop over tiles, then binary search
    int64_t lo = pe, step = TP, hi = lo + step;
    while (hi < a.n && keys[hi] == k0) { lo = hi; step <<= 1; hi = lo + step; }
    if (hi > a.n) hi = a.n;
    while (hi - lo > 1) {
      const int64_t mid = (lo + hi) >> 1;
      if (keys[mid] == k0) lo = mid; else hi = mid;
    }
    const int64_t te = (hi - 1) / TP;  // tile holding the run's last position (> t)
    float4 acc = *reinterpret_cast<const float4*>(carry_last + t * ROWF + c);
    int64_t tt = t + 1;
    for (; tt + 4 <= te; tt += 4) {
      float4 r[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) r[q] = *reinterpret_cast<const float4*>(carry_last + (tt + q) * ROWF + c);
#pragma unroll
      for (int q = 0; q < 4; ++q) acc = f4_add(acc, r[q]);
    }
    for (; tt < te; ++tt) acc = f4_add(acc, *reinterpret_cast<const float4*>(carry_last + tt * ROWF + c));
    acc = f4_add(acc, *reinterpret_cast<const float4*>(carry_first + te * ROWF + c));
    const int32_t v0 = vals[pe - 1];
    const int f0 = a.pooled ? bag_feat(a, v0) : feat_of_key<KeyT>(fd, a.F, k0);
    const BwdFeat d = fd[f0];
    float accv[1][4] = {{acc.x, acc.y, acc.z, acc.w}};
    finish_run<G, 4, 1>(a, d, (int64_t)k0 - d.key_base, (int64_t)k0, accv, lane);
  }
}

__global__ void zero_counters(int32_t* c) { c[0] = 0; c[1] = 0; c[2] = 0; c[3] = 0; }

inline int bits_for(int64_t total_keys) {
  int b = 1;
  while (b < 63 && ((int64_t)1 << b) < total_keys) ++b;
  return b;
}

struct WsLayout {
  size_t keys_in, keys_out, vals_in, vals_out, items, runs, counters, partials, carry, cub_tmp, total;
  size_t cub_bytes, carry_floats;
};

template <typename KeyT>
cudaError_t cub_sort(void* tmp, size_t& tmp_bytes, const KeyT* kin, KeyT* kout, const int32_t* vin,
                     int32_t* vout, int64_t n, int bits, cudaStream_t st) {
  return cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, kin, kout, vin, vout, (int)n, 0, bits, st);
}

inline int64_t max_items(int64_t n) { return n / kShortRun + n / kChunk + 2; }   // every long run has > 32 ids
inline int64_t max_pslots(int64_t n) { return 2 * (n / kChunk) + 2; }            // multi-chunk runs have > kChunk

WsLayout ws_layout(int64_t nnz, int64_t total_keys, int max_dim) {
  WsLayout L;
  const bool k64 = total_keys >= ((int64_t)1 << 32);
  const size_t ksz = k64 ? 8 : 4;
  const int64_t n = nnz < 1 ? 1 : nnz;
  size_t o = 0;
  L.keys_in = o; o = align_up(o + n * ksz, 256);
  L.keys_out = o; o = align_up(o + n * ksz, 256);
  L.vals_in = o; o = align_up(o + n * 4, 256);
  L.vals_out = o; o = align_up(o + n * 4, 256);
  L.items = o; o = align_up(o + max_items(n) * sizeof(ChunkItem), 256);
  L.runs = o; o = align_up(o + (size_t)max_pslots(n) * sizeof(int32_t), 256);        // run_done counters
  L.counters = o; o = align_up(o + 256, 256);
  const size_t rowf = (size_t)((max_dim + 127) / 128 * 128 < 128 ? 128 : (max_dim + 127) / 128 * 128) * 4;
  L.partials = o; o = align_up(o + max_pslots(n) * rowf * sizeof(float), 256);
  {  // tile path (dims <= 128): carry_first | carry_last
    int g = 1;
    while (g * 4 < max_dim && g < 32) g <<= 1;
    L.carry_floats = (size_t)tile_carry_floats(n, g * 4);
    L.carry = o; o = align_up(o + 2 * L.carry_floats * sizeof(float), 256);
  }
  size_t tb = 0;
  const int bits = bits_for(total_keys + 1);
  if (k64) cub_sort<uint64_t>(nullptr, tb, nullptr, nullptr, nullptr, nullptr, n, bits, 0);
  else cub_sort<uint32_t>(nullptr, tb, nullptr, nullptr, nullptr, nullptr, n, bits, 0);
  L.cub_bytes = tb;
  L.cub_tmp = o; o = align_up(o + tb, 256);
  L.total = o;
  return L;
}

}  // namespace

#define TZK_BWD_LAUNCH(KeyT, G_, VEC_, CH_, FAM_)                                                    \
  do {                                                                                                \
    size_t smem_s = (size_t)F * sizeof(BwdFeat);                                                      \
    if (sw) {                                                                                         \
      if (smem_s > 48 * 1024)                                                                         \
        cudaFuncSetAttribute(fused_apply_weighted_kernel<KeyT, G_, VEC_, CH_, FAM_>,                  \
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_s);               \
      fused_apply_weighted_kernel<KeyT, G_, VEC_, CH_, FAM_><<<grid_s + n_long, kThreads, smem_s, st>>>( \
          a, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, (const KeyT*)keys_out, \
          vals_out, wl, n_long, gp, sw);                                                              \
      TZK_CHECK_LAUNCH("fused_apply_weighted_kernel");                                                \
      break;                                                                                          \
    }                                                                                                 \
    if (smem_s > 48 * 1024)                                                                           \
      cudaFuncSetAttribute(fused_apply_kernel<KeyT, G_, VEC_, CH_, FAM_>,                             \
                           cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_s);                 \
    fused_apply_kernel<KeyT, G_, VEC_, CH_, FAM_><<<grid_s + n_long, kThreads, smem_s, st>>>(         \
        a, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, (const KeyT*)keys_out, \
        vals_out, wl, n_long, gp);                                                                    \
    TZK_CHECK_LAUNCH("fused_apply_kernel");                                                           \
  } while (0)

#define TZK_BWD_DISPATCH_G(KeyT, VEC_, CH_, FAM_)                 \
  switch (G) {                                                    \
    case 1: TZK_BWD_LAUNCH(KeyT, 1, VEC_, CH_, FAM_); break;      \
    case 2: TZK_BWD_LAUNCH(KeyT, 2, VEC_, CH_, FAM_); break;      \
    case 4: TZK_BWD_LAUNCH(KeyT, 4, VEC_, CH_, FAM_); break;      \
    case 8: TZK_BWD_LAUNCH(KeyT, 8, VEC_, CH_, FAM_); break;      \
    case 16: TZK_BWD_LAUNCH(KeyT, 16, VEC_, CH_, FAM_); break;    \
    default: TZK_BWD_LAUNCH(KeyT, 32, VEC_, CH_, FAM_); break;    \
  }

// general path, every (key width, VEC, G, CH) of one optimizer family
#define TZK_BWD_DISPATCH(FAM_)                                                                                         \
  do {                                                                                                                 \
    if (k64) {                                                                                                         \
      if (vec == 4) { if (ch == 1) { TZK_BWD_DISPATCH_G(uint64_t, 4, 1, FAM_) } else if (ch <= 2) { TZK_BWD_LAUNCH(uint64_t, 32, 4, 2, FAM_); } else { TZK_BWD_LAUNCH(uint64_t, 32, 4, 8, FAM_); } } \
      else { if (ch == 1) { TZK_BWD_DISPATCH_G(uint64_t, 1, 1, FAM_) } else if (ch <= 2) { TZK_BWD_LAUNCH(uint64_t, 32, 1, 2, FAM_); } else { TZK_BWD_LAUNCH(uint64_t, 32, 1, 8, FAM_); } } \
    } else {                                                                                                           \
      if (vec == 4) { if (ch == 1) { TZK_BWD_DISPATCH_G(uint32_t, 4, 1, FAM_) } else if (ch <= 2) { TZK_BWD_LAUNCH(uint32_t, 32, 4, 2, FAM_); } else { TZK_BWD_LAUNCH(uint32_t, 32, 4, 8, FAM_); } } \
      else { if (ch == 1) { TZK_BWD_DISPATCH_G(uint32_t, 1, 1, FAM_) } else if (ch <= 2) { TZK_BWD_LAUNCH(uint32_t, 32, 1, 2, FAM_); } else { TZK_BWD_LAUNCH(uint32_t, 32, 1, 8, FAM_); } } \
    }                                                                                                                  \
  } while (0)

// kFamNorm: the optimizers of finish_run_norm (row-wise Adagrad only with a weight decay mode and a nonzero decay;
// without them it is the classic update)
static bool norm_family(const tzk_opt_args& o) {
  return o.optimizer == TZK_OPT_LAMB || o.optimizer == TZK_OPT_PARTIAL_ROWWISE_LAMB || o.optimizer == TZK_OPT_LARS_SGD ||
         (o.optimizer == TZK_OPT_ROWWISE_ADAGRAD && o.weight_decay_mode != 0 && o.weight_decay != 0.f);
}
static bool elem_state_opt(int32_t optimizer) {   // first state laid out like the weights
  return optimizer == TZK_OPT_ADAGRAD || optimizer == TZK_OPT_ADAM || optimizer == TZK_OPT_PARTIAL_ROWWISE_ADAM ||
         optimizer == TZK_OPT_LAMB || optimizer == TZK_OPT_PARTIAL_ROWWISE_LAMB || optimizer == TZK_OPT_LARS_SGD;
}

extern "C" size_t tzk_fused_bwd_workspace_bytes(int64_t nnz, int64_t total_keys, int32_t max_dim) {
  return ws_layout(nnz, total_keys, max_dim < 1 ? 1 : max_dim).total;
}

// weighted bags: the unweighted layout, then bag_of [n] int32 (id position -> bag) and sw [n] fp32 (sorted weights)
struct WsWeighted { size_t bag_of, sw, total; };
static WsWeighted ws_weighted(const WsLayout& L, int64_t nnz) {
  const int64_t n = nnz < 1 ? 1 : nnz;
  WsWeighted W;
  W.bag_of = L.total;
  W.sw = align_up(W.bag_of + (size_t)n * 4, 256);
  W.total = align_up(W.sw + (size_t)n * 4, 256);
  return W;
}

extern "C" size_t tzk_fused_bwd_weighted_workspace_bytes(int64_t nnz, int64_t total_keys, int32_t max_dim) {
  return ws_weighted(ws_layout(nnz, total_keys, max_dim < 1 ? 1 : max_dim), nnz).total;
}

// phases: 1 = linearize + sort (needs ids / offsets only), 2 = reduce runs + update (needs the gradient)
static int fused_bwd_impl(int phases, const tzk_opt_args& opt, int32_t pooled, const float* grad_out,
                          int64_t ld_grad, const int64_t* feat_w_off, const int64_t* feat_rows,
                          const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_pool,
                          const int64_t* feat_key_base, const int64_t* ids, const int64_t* offsets,
                          int32_t F, int32_t B, int64_t nnz, int64_t total_keys, int32_t max_dim,
                          int32_t vec_ok, float* weights, float grad_scale, void* workspace,
                          size_t workspace_bytes, tzk_stream_t stream, const PeerWire* pw = nullptr,
                          const uint64_t* grad_ptrs = nullptr, int32_t* overflow = nullptr) {
  // weighted bags (opt.per_sample_weights != NULL, pooled local layouts only): phase 1 reads the weights and leaves them
  // sorted in the workspace, phase 2 reads them from there
  const float* psw = opt.per_sample_weights;
  // peer mode (pw != nullptr): nnz = W * cap wire slots; phase 1 pulls the keys from the sources' wire buffers instead
  // of linearising local ids; phase 2 reads every gradient slice from grad_ptrs[src] (tzk_peer.cu, DESIGN.md §6)
  const int32_t optimizer = opt.optimizer;
  float* state = opt.state;
  const float lr = opt.lr, eps = opt.eps;
  TZK_REQUIRE((optimizer >= 0 && optimizer <= TZK_OPT_LARS_SGD) || optimizer == TZK_OPT_ACCUM_OUT,
              "fused_bwd: unknown optimizer %d", optimizer);
  TZK_REQUIRE(F >= 0 && B >= 0 && nnz >= 0, "fused_bwd: negative size");
  if (F == 0 || B == 0 || nnz == 0) return 0;
  TZK_REQUIRE(nnz < ((int64_t)1 << 31) && (int64_t)F * std::max(B, 1) < ((int64_t)1 << 31),
              "fused_bwd: nnz or F*B >= 2^31 not supported");
  TZK_REQUIRE(pw || (feat_rows && feat_key_base && offsets), "fused_bwd: NULL argument");
  TZK_REQUIRE(!(phases & 1) || ids || pw, "fused_bwd: ids is NULL");
  if (phases & 2) {
    TZK_REQUIRE((grad_out || grad_ptrs) && feat_w_off && feat_dim && weights && feat_rows && feat_key_base,
                "fused_bwd: NULL argument");
    TZK_REQUIRE(!pooled || (feat_col && feat_pool), "fused_bwd: pooled mode needs feat_col/feat_pool");
    TZK_REQUIRE(optimizer == TZK_OPT_SGD || state != nullptr || opt.interleaved, "fused_bwd: optimizer state is NULL");
    TZK_REQUIRE(!opt.interleaved || (optimizer == TZK_OPT_ADAGRAD && !opt.weights_f16),
                "fused_bwd: interleaved [weight | state] rows are implemented for fp32 tables with element-wise Adagrad");
    TZK_REQUIRE((optimizer != TZK_OPT_ADAM && optimizer != TZK_OPT_PARTIAL_ROWWISE_ADAM &&
                 optimizer != TZK_OPT_LAMB && optimizer != TZK_OPT_PARTIAL_ROWWISE_LAMB) || (opt.state2 && opt.step),
                "fused_bwd: Adam and LAMB variants need state2 and the device step counter");
    TZK_REQUIRE(optimizer != TZK_OPT_ROWWISE_ADAGRAD || (opt.weight_decay_mode >= 0 && opt.weight_decay_mode <= 2),
                "fused_bwd: weight_decay_mode %d is not NONE (0), L2 (1) or DECOUPLE (2)", opt.weight_decay_mode);
  }
  TZK_REQUIRE(F <= 2048, "fused_bwd: F=%d > 2048 keys per collection", F);
  TZK_REQUIRE(max_dim >= 1 && max_dim <= 1024, "fused_bwd: max_dim=%d out of range [1,1024]", max_dim);
  WsLayout L = ws_layout(nnz, total_keys, max_dim);
  const WsWeighted LW = ws_weighted(L, nnz);
  TZK_REQUIRE(!psw || (pooled && !pw), "fused_bwd: per-sample weights need the pooled local layout");
  const size_t ws_need = psw ? LW.total : L.total;
  TZK_REQUIRE(workspace && workspace_bytes >= ws_need, "fused_bwd: workspace too small (%zu < %zu)", workspace_bytes,
              ws_need);
  cudaStream_t st = as_stream(stream);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  float* sw = psw ? reinterpret_cast<float*>(ws + LW.sw) : nullptr;
  void* keys_in = ws + L.keys_in;
  void* keys_out = ws + L.keys_out;
  int32_t* vals_in = reinterpret_cast<int32_t*>(ws + L.vals_in);
  int32_t* vals_out = reinterpret_cast<int32_t*>(ws + L.vals_out);
  WorkLists wl;
  wl.items = reinterpret_cast<ChunkItem*>(ws + L.items);
  wl.run_done = reinterpret_cast<int32_t*>(ws + L.runs);
  wl.counters = reinterpret_cast<int32_t*>(ws + L.counters);
  wl.partials = reinterpret_cast<float*>(ws + L.partials);
  // short-run head list in the sort's dead INPUT buffers (n int32 positions in vals_in, n int32 lengths in keys_in).
  // Default on; TZK_BWD_HEADS=0: walk every position.
  // Both halves of a step read the switch, so it must not change between a sort and its apply.
  wl.head_pos = nullptr;
  wl.head_len = nullptr;
  const char* heads_env = getenv("TZK_BWD_HEADS");
  if (!(heads_env && heads_env[0] == '0')) {
    wl.head_pos = vals_in;
    wl.head_len = reinterpret_cast<int32_t*>(keys_in);
  }
  const bool k64 = total_keys >= ((int64_t)1 << 32);
  const int bits = bits_for(total_keys + 1);   // one spare value above the largest key = padding sentinel
  const uint64_t sentinel = ((uint64_t)1 << bits) - 1;

  if ((phases & 1) && pw) {
    size_t cub_bytes = L.cub_bytes;
    cudaError_t ce;
    const int grid_p = (int)std::min<int64_t>(ceil_div64(nnz, kThreads), kSmCountH100 * 8);
    if (k64) {
      peer_pull_linearize_kernel<uint64_t><<<grid_p, kThreads, 0, st>>>(*pw, (uint64_t)sentinel, (uint64_t*)keys_in,
                                                                         vals_in, overflow);
      TZK_CHECK_LAUNCH("peer_pull_linearize_kernel");
      ce = cub_sort<uint64_t>(ws + L.cub_tmp, cub_bytes, (const uint64_t*)keys_in, (uint64_t*)keys_out, vals_in,
                              vals_out, nnz, bits, st);
    } else {
      peer_pull_linearize_kernel<uint32_t><<<grid_p, kThreads, 0, st>>>(*pw, (uint32_t)sentinel, (uint32_t*)keys_in,
                                                                         vals_in, overflow);
      TZK_CHECK_LAUNCH("peer_pull_linearize_kernel");
      ce = cub_sort<uint32_t>(ws + L.cub_tmp, cub_bytes, (const uint32_t*)keys_in, (uint32_t*)keys_out, vals_in,
                              vals_out, nnz, bits, st);
    }
    TZK_REQUIRE(ce == cudaSuccess, "fused_bwd: radix sort failed: %s", cudaGetErrorString(ce));
  } else if (phases & 1) {
  const int64_t n_bags = (int64_t)F * B;
  int grid_lin = (int)std::min<int64_t>(ceil_div64(n_bags, kThreads), kSmCountH100 * 16);
  size_t cub_bytes = L.cub_bytes;
  cudaError_t ce;
  const size_t smem_lin = (size_t)(3 * F + 1) * sizeof(int64_t);   // 49 160 B at F = 2048: opt-in above 48 KB
  const int grid_seq = (int)std::min<int64_t>(ceil_div64(nnz, kThreads), kSmCountH100 * 16);
  if (!pooled && smem_lin > 48 * 1024) {
    if (k64) cudaFuncSetAttribute(linearize_seq_kernel<uint64_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_lin);
    else cudaFuncSetAttribute(linearize_seq_kernel<uint32_t>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_lin);
  }
  int32_t* bag_of = reinterpret_cast<int32_t*>(ws + LW.bag_of);
  if (k64) {
    if (psw)
      linearize_weighted_kernel<uint64_t><<<grid_lin, kThreads, 0, st>>>(
          ids, offsets, feat_rows, feat_key_base, F, B, (uint64_t)sentinel, (uint64_t*)keys_in, vals_in, bag_of);
    else if (pooled)
      linearize_kernel<uint64_t><<<grid_lin, kThreads, 0, st>>>(ids, offsets, feat_rows, feat_key_base, F, B,
                                                                pooled, (uint64_t)sentinel, (uint64_t*)keys_in, vals_in);
    else
      linearize_seq_kernel<uint64_t><<<grid_seq, kThreads, smem_lin, st>>>(
          ids, offsets, feat_rows, feat_key_base, F, B, nnz, (uint64_t)sentinel, (uint64_t*)keys_in, vals_in);
    TZK_CHECK_LAUNCH("linearize_kernel");
    ce = cub_sort<uint64_t>(ws + L.cub_tmp, cub_bytes, (const uint64_t*)keys_in, (uint64_t*)keys_out, vals_in,
                            vals_out, nnz, bits, st);
  } else {
    if (psw)
      linearize_weighted_kernel<uint32_t><<<grid_lin, kThreads, 0, st>>>(
          ids, offsets, feat_rows, feat_key_base, F, B, (uint32_t)sentinel, (uint32_t*)keys_in, vals_in, bag_of);
    else if (pooled)
      linearize_kernel<uint32_t><<<grid_lin, kThreads, 0, st>>>(ids, offsets, feat_rows, feat_key_base, F, B,
                                                                pooled, (uint32_t)sentinel, (uint32_t*)keys_in, vals_in);
    else
      linearize_seq_kernel<uint32_t><<<grid_seq, kThreads, smem_lin, st>>>(
          ids, offsets, feat_rows, feat_key_base, F, B, nnz, (uint32_t)sentinel, (uint32_t*)keys_in, vals_in);
    TZK_CHECK_LAUNCH("linearize_kernel");
    ce = cub_sort<uint32_t>(ws + L.cub_tmp, cub_bytes, (const uint32_t*)keys_in, (uint32_t*)keys_out, vals_in,
                            vals_out, nnz, bits, st);
  }
  TZK_REQUIRE(ce == cudaSuccess, "fused_bwd: radix sort failed: %s", cudaGetErrorString(ce));
  if (psw) {
    const int grid_w = (int)std::min<int64_t>(ceil_div64(nnz, kThreads), kSmCountH100 * 8);
    sorted_bag_weight_kernel<<<grid_w, kThreads, 0, st>>>(vals_out, bag_of, psw, nnz, sw);
    TZK_CHECK_LAUNCH("sorted_bag_weight_kernel");
  }
  }
  if (phases & 1) {   // work list of the long runs (tiny tables, hot ids) for the gradient half's chunk CTAs
    zero_counters<<<1, 1, 0, st>>>(wl.counters);
    const int grid_f = (int)std::min<int64_t>(ceil_div64(nnz, kThreads), kSmCountH100 * 8);
    if (k64) find_long_runs_kernel<uint64_t><<<grid_f, kThreads, 0, st>>>((const uint64_t*)keys_out, nnz, (uint64_t)sentinel, wl);
    else find_long_runs_kernel<uint32_t><<<grid_f, kThreads, 0, st>>>((const uint32_t*)keys_out, nnz, (uint32_t)sentinel, wl);
    TZK_CHECK_LAUNCH("find_long_runs_kernel");
  }
  if (!(phases & 2)) return 0;

  BwdArgs a;
  a.grad_out = grad_out; a.ld_grad = ld_grad; a.offsets = offsets; a.weights = weights; a.state = state;
  a.lr = lr; a.eps = eps; a.grad_scale = grad_scale; a.F = F; a.B = B; a.optimizer = optimizer;
  a.pooled = pooled; a.n = nnz; a.sentinel = sentinel;
  a.state2 = opt.state2; a.step = opt.step; a.beta1 = opt.beta1; a.beta2 = opt.beta2;
  a.weight_decay = opt.weight_decay; a.max_gradient = opt.max_gradient; a.bc1 = a.bc2 = 1.f;
  a.peer_w = 0; a.idx_span = 1; a.w_f16 = opt.weights_f16 ? 1 : 0; a.interleaved = opt.interleaved ? 1 : 0;
  a.div_b = make_fast_div(B); a.div_span = make_fast_div(1);
  TZK_REQUIRE(ld_grad >= 0 && ld_grad < ((int64_t)1 << 31), "fused_bwd: ld_grad out of range");
  a.ld32 = (int32_t)ld_grad; a.wd_mode = opt.weight_decay_mode;
  if (optimizer == TZK_OPT_LARS_SGD) { a.beta1 = opt.momentum; a.beta2 = opt.eta; }
  const int fam = norm_family(opt) ? kFamNorm : kFamClassic;
  PeerGrads gp;
  for (int r = 0; r < 16; ++r) gp.p[r] = 0ull;
  if (pw) {
    TZK_REQUIRE(grad_ptrs, "fused_bwd: peer mode needs the published gradient pointers");
    a.peer_w = pw->W; a.idx_span = pw->idx_span;
    a.div_span = make_fast_div(pw->idx_span);
    for (int r = 0; r < pw->W; ++r) gp.p[r] = grad_ptrs[r];
    a.grad_out = reinterpret_cast<const float*>(grad_ptrs[pw->me]);
  }

  bool peers_aligned = true;
  for (int r = 0; r < a.peer_w; ++r) peers_aligned = peers_aligned && (gp.p[r] % 16 == 0);
  const int vec = (vec_ok && peers_aligned && ((uintptr_t)weights % (a.w_f16 ? 8 : 16) == 0) &&
                   ((uintptr_t)a.grad_out % 16 == 0) &&
                   (ld_grad % 4 == 0) &&
                   (!elem_state_opt(optimizer) || opt.interleaved || (uintptr_t)state % 16 == 0) &&
                   ((optimizer != TZK_OPT_ADAM && optimizer != TZK_OPT_LAMB) || (uintptr_t)opt.state2 % 16 == 0))
                      ? 4 : 1;
  int need = (max_dim + vec - 1) / vec;  // chunks per row
  int G = 1;
  while (G < need && G < 32) G <<= 1;
  const int ch = (need + G - 1) / G;
  TZK_REQUIRE(ch <= 8, "fused_bwd: max_dim=%d needs %d chunks per lane (> 8); unaligned wide rows are not supported",
              max_dim, ch);
  const int NG = kThreads / G;
  int grid_s = (int)std::min<int64_t>(ceil_div64(nnz, NG), kSmCountH100 * 16);
  // TZK_BWD_TILE=1 selects the tile path.  Both paths are bound by the random 64-B weight/state/gradient accesses of
  // the gradient half, and the general kernels execute fewer instructions without the three barriers per tile, so
  // they stay the default.  The kFamNorm optimizers always take the general path.
  const char* tile_env = getenv("TZK_BWD_TILE");
  const bool tile_path = tile_env && tile_env[0] == '1' && !a.w_f16 && !a.interleaved && optimizer != TZK_OPT_ACCUM_OUT &&
                         fam == kFamClassic && !sw;   // (fp32 tables, real classic updates, unweighted bags)
  if (vec == 4 && ch == 1 && tile_path) {
    // tile path: every gradient / weight / state row of a tile is requested at once, runs are reduced in shared memory
    float* carry_first = reinterpret_cast<float*>(ws + L.carry);
    float* carry_last = carry_first + L.carry_floats;
#define TZK_TILE_LAUNCH(KeyT, G_)                                                                               \
  do {                                                                                                          \
    using C = TileCfg<G_>;                                                                                      \
    const int64_t n_tiles = ceil_div64(nnz, C::TP);                                                             \
    const size_t smem_t = align16((size_t)C::TP * C::ROWF * 4 + (C::TP + 2) * sizeof(KeyT) + C::TP * 4) +       \
                          (size_t)F * sizeof(BwdFeat);                                                          \
    if (smem_t > 48 * 1024)                                                                                     \
      cudaFuncSetAttribute(tile_update_kernel<KeyT, G_>, cudaFuncAttributeMaxDynamicSharedMemorySize,           \
                           (int)smem_t);                                                                        \
    const int grid_t = (int)std::min<int64_t>(n_tiles, kSmCountH100 * 8);                                       \
    tile_update_kernel<KeyT, G_><<<grid_t, kThreads, smem_t, st>>>(                                             \
        a, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, (const KeyT*)keys_out, vals_out, \
        carry_first, carry_last, gp);                                                                           \
    TZK_CHECK_LAUNCH("tile_update_kernel");                                                                     \
    if (n_tiles > 1) {                                                                                          \
      const size_t smem_c = (size_t)F * sizeof(BwdFeat);                                                        \
      if (smem_c > 48 * 1024)                                                                                   \
        cudaFuncSetAttribute(carry_combine_kernel<KeyT, G_>, cudaFuncAttributeMaxDynamicSharedMemorySize,       \
                             (int)smem_c);                                                                      \
      const int grid_c = (int)std::min<int64_t>(ceil_div64(n_tiles - 1, C::NG), kSmCountH100 * 8);              \
      carry_combine_kernel<KeyT, G_><<<grid_c, kThreads, smem_c, st>>>(                                         \
          a, feat_w_off, feat_rows, feat_key_base, feat_dim, feat_col, feat_pool, (const KeyT*)keys_out,        \
          vals_out, carry_first, carry_last);                                                                   \
      TZK_CHECK_LAUNCH("carry_combine_kernel");                                                                 \
    }                                                                                                           \
  } while (0)
#define TZK_TILE_DISPATCH(KeyT)                      \
  switch (G) {                                       \
    case 1: TZK_TILE_LAUNCH(KeyT, 1); break;         \
    case 2: TZK_TILE_LAUNCH(KeyT, 2); break;         \
    case 4: TZK_TILE_LAUNCH(KeyT, 4); break;         \
    case 8: TZK_TILE_LAUNCH(KeyT, 8); break;         \
    case 16: TZK_TILE_LAUNCH(KeyT, 16); break;       \
    default: TZK_TILE_LAUNCH(KeyT, 32); break;       \
  }
    if (k64) { TZK_TILE_DISPATCH(uint64_t) } else { TZK_TILE_DISPATCH(uint32_t) }
#undef TZK_TILE_DISPATCH
#undef TZK_TILE_LAUNCH
    return 0;
  }

  // general path: one launch — short runs by sorted position + the long-run list's chunk CTAs (CH compiled for 1, 2, 8)
  const int n_long = kSmCountH100 * 2;
  if (fam == kFamNorm) TZK_BWD_DISPATCH(kFamNorm);
  else TZK_BWD_DISPATCH(kFamClassic);
  return 0;
}

static tzk_opt_args classic_opt(int32_t optimizer, float* state, float lr, float eps) {
  tzk_opt_args o;
  o.optimizer = optimizer; o.lr = lr; o.eps = eps; o.beta1 = 0.9f; o.beta2 = 0.999f; o.weight_decay = 0.f;
  o.max_gradient = 0.f; o.state = state; o.state2 = nullptr; o.step = nullptr; o.weights_f16 = 0; o.interleaved = 0;
  o.momentum = 0.f; o.eta = 0.f; o.weight_decay_mode = 0; o.per_sample_weights = nullptr;
  return o;
}

extern "C" int tzk_fused_bwd(int32_t optimizer, int32_t pooled, const float* grad_out, int64_t ld_grad,
                             const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                             const int32_t* feat_col, const int32_t* feat_pool,
                             const int64_t* feat_key_base, const int64_t* ids, const int64_t* offsets,
                             int32_t F, int32_t B, int64_t nnz, int64_t total_keys, int32_t max_dim,
                             int32_t vec_ok, float* weights, float* state, float lr, float eps,
                             float grad_scale, void* workspace, size_t workspace_bytes,
                             tzk_stream_t stream) {
  TZK_REQUIRE(optimizer >= 0 && optimizer <= TZK_OPT_ROWWISE_ADAGRAD,
              "fused_bwd: optimizer %d needs tzk_fused_bwd_ex", optimizer);
  return fused_bwd_impl(3, classic_opt(optimizer, state, lr, eps), pooled, grad_out, ld_grad, feat_w_off, feat_rows,
                        feat_dim, feat_col, feat_pool, feat_key_base, ids, offsets, F, B, nnz, total_keys, max_dim,
                        vec_ok, weights, grad_scale, workspace, workspace_bytes, stream);
}

extern "C" int tzk_fused_bwd_ex(const tzk_opt_args* opt, int32_t pooled, const float* grad_out, int64_t ld_grad,
                                const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                                const int32_t* feat_col, const int32_t* feat_pool, const int64_t* feat_key_base,
                                const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int64_t nnz,
                                int64_t total_keys, int32_t max_dim, int32_t vec_ok, float* weights,
                                float grad_scale, void* workspace, size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(opt != nullptr, "fused_bwd_ex: opt is NULL");
  return fused_bwd_impl(3, *opt, pooled, grad_out, ld_grad, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool,
                        feat_key_base, ids, offsets, F, B, nnz, total_keys, max_dim, vec_ok, weights, grad_scale,
                        workspace, workspace_bytes, stream);
}

extern "C" int tzk_fused_bwd_sort(int32_t pooled, const int64_t* feat_rows, const int64_t* feat_key_base,
                                  const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int64_t nnz,
                                  int64_t total_keys, int32_t max_dim, void* workspace, size_t workspace_bytes,
                                  tzk_stream_t stream) {
  return fused_bwd_impl(1, classic_opt(TZK_OPT_SGD, nullptr, 0.f, 0.f), pooled, nullptr, 0, nullptr, feat_rows,
                        nullptr, nullptr, nullptr, feat_key_base, ids, offsets, F, B, nnz, total_keys, max_dim, 0,
                        nullptr, 0.f, workspace, workspace_bytes, stream);
}

// id half of a weighted update (workspace: tzk_fused_bwd_weighted_workspace_bytes); its gradient half is
// tzk_fused_bwd_apply_ex with opt->per_sample_weights non-NULL
extern "C" int tzk_fused_bwd_sort_weighted(int32_t pooled, const int64_t* feat_rows, const int64_t* feat_key_base,
                                           const int64_t* ids, const int64_t* offsets, const float* per_sample_weights,
                                           int32_t F, int32_t B, int64_t nnz, int64_t total_keys, int32_t max_dim,
                                           void* workspace, size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(per_sample_weights != nullptr || F == 0 || B == 0 || nnz == 0,
              "fused_bwd_sort_weighted: per_sample_weights is NULL");
  tzk_opt_args o = classic_opt(TZK_OPT_SGD, nullptr, 0.f, 0.f);
  o.per_sample_weights = per_sample_weights;
  return fused_bwd_impl(1, o, pooled, nullptr, 0, nullptr, feat_rows, nullptr, nullptr, nullptr, feat_key_base, ids,
                        offsets, F, B, nnz, total_keys, max_dim, 0, nullptr, 0.f, workspace, workspace_bytes, stream);
}

extern "C" int tzk_fused_bwd_apply(int32_t optimizer, int32_t pooled, const float* grad_out, int64_t ld_grad,
                                   const int64_t* feat_w_off, const int64_t* feat_rows, const int32_t* feat_dim,
                                   const int32_t* feat_col, const int32_t* feat_pool,
                                   const int64_t* feat_key_base, const int64_t* offsets, int32_t F, int32_t B,
                                   int64_t nnz, int64_t total_keys, int32_t max_dim, int32_t vec_ok, float* weights,
                                   float* state, float lr, float eps, float grad_scale, void* workspace,
                                   size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(optimizer >= 0 && optimizer <= TZK_OPT_ROWWISE_ADAGRAD,
              "fused_bwd_apply: optimizer %d needs tzk_fused_bwd_apply_ex", optimizer);
  return fused_bwd_impl(2, classic_opt(optimizer, state, lr, eps), pooled, grad_out, ld_grad, feat_w_off, feat_rows,
                        feat_dim, feat_col, feat_pool, feat_key_base, nullptr, offsets, F, B, nnz, total_keys,
                        max_dim, vec_ok, weights, grad_scale, workspace, workspace_bytes, stream);
}

extern "C" int tzk_fused_bwd_apply_ex(const tzk_opt_args* opt, int32_t pooled, const float* grad_out,
                                      int64_t ld_grad, const int64_t* feat_w_off, const int64_t* feat_rows,
                                      const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_pool,
                                      const int64_t* feat_key_base, const int64_t* offsets, int32_t F, int32_t B,
                                      int64_t nnz, int64_t total_keys, int32_t max_dim, int32_t vec_ok,
                                      float* weights, float grad_scale, void* workspace, size_t workspace_bytes,
                                      tzk_stream_t stream) {
  TZK_REQUIRE(opt != nullptr, "fused_bwd_apply_ex: opt is NULL");
  return fused_bwd_impl(2, *opt, pooled, grad_out, ld_grad, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool,
                        feat_key_base, nullptr, offsets, F, B, nnz, total_keys, max_dim, vec_ok, weights, grad_scale,
                        workspace, workspace_bytes, stream);
}

// ---- owner side of the small-table exchange ----------------------------------------------------------------------------
// Every rank reduced its own batch's gradients of the small tables into a dense per-row buffer psum_r [R_small, dim]
// (+ flags_r [R_small]: row touched this step) in symmetric memory.  The owner of a row adds the W partial sums in rank
// order — long sequential NVLink reads, a few MB in all — and applies ONE optimizer update to its arena row.
struct SmallTab {
  int64_t kb_small;    // key of the table's first row in the small key space (= row index into psum / flags)
  int64_t start;       // global row of this rank's first local row
  int64_t w_off;       // local arena offset of the shard
  int64_t psum_off;    // element offset of the table in psum
  int64_t key_base;    // local linearised key of the shard's first row (row-wise optimizer state)
  int32_t first;       // prefix sum of local rows over the small tables
  int32_t n_local;
  int32_t dim;
  int32_t pad;
};
struct SmallPeers { unsigned long long psum[16], flags[16]; };

template <int G, int FAM>
__global__ void __launch_bounds__(kThreads)
small_table_update_kernel(BwdArgs a, const __grid_constant__ SmallPeers sp, const SmallTab* __restrict__ tabs, int n_tabs,
                          int total_rows, int W) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SmallTab* st = reinterpret_cast<SmallTab*>(smem_raw);
  for (int i = threadIdx.x; i < n_tabs; i += blockDim.x) st[i] = tabs[i];
  __syncthreads();
  init_bias_correction<FAM>(a);
  constexpr int NG = kThreads / G;
  const int lane = threadIdx.x % G;
  for (int j = blockIdx.x * NG + threadIdx.x / G; j < total_rows; j += gridDim.x * NG) {
    int lo = 0, hi = n_tabs;
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (st[mid].first <= j) lo = mid; else hi = mid;
    }
    const SmallTab t = st[lo];
    const int64_t i = j - t.first;                      // local row
    const int64_t key_s = t.kb_small + t.start + i;     // row in the small key space
    float acc[1][4] = {{0.f, 0.f, 0.f, 0.f}};
    bool any = false;
    const int c = lane * 4;
    // all W flags, then all flagged partial sums, are requested before anything is consumed: two NVLink round trips per
    // row instead of 2 W dependent ones; the additions stay in rank order (the same sum on every run)
    int32_t fl[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) fl[r] = r < W ? reinterpret_cast<const int32_t*>(sp.flags[r])[key_s] : 0;
    float4 pv[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      pv[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (fl[r] && c < t.dim)
        pv[r] = ld_coh_f4(reinterpret_cast<const float*>(sp.psum[r]) + t.psum_off + (t.start + i) * t.dim + c);
    }
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      if (fl[r]) {
        any = true;
        acc[0][0] += pv[r].x; acc[0][1] += pv[r].y; acc[0][2] += pv[r].z; acc[0][3] += pv[r].w;
      }
    }
    if (!any) continue;                                 // (group-uniform: every lane read the same flags)
    BwdFeat d;
    d.w_off = t.w_off; d.rows = t.n_local; d.key_base = t.key_base; d.dim = t.dim; d.col = 0; d.pool = 0;
    d.stride = a.interleaved ? 2 * t.dim : t.dim;
    finish_run<G, 4, 1, FAM>(a, d, i, t.key_base + i, acc, lane);
  }
}

// psum_ptrs / flag_ptrs: HOST arrays [W] of device addresses (rank r's partial-sum buffer / flags as mapped here).
// tabs: device array of n_tabs descriptors {kb_small, start, w_off, psum_off, key_base, first, n_local, dim} (int64 x5,
// int32 x4 — struct SmallTab); total_rows = sum of n_local.  Dims must be multiples of 4 and <= 128.
extern "C" int tzk_peer_small_update(const tzk_opt_args* opt, const uint64_t* psum_ptrs, const uint64_t* flag_ptrs,
                                     int32_t W, const void* tabs, int32_t n_tabs, int32_t total_rows, int32_t max_dim,
                                     float* weights, tzk_stream_t stream) {
  TZK_REQUIRE(opt && psum_ptrs && flag_ptrs && W >= 1 && W <= 16 && n_tabs >= 0 && total_rows >= 0,
              "peer_small_update: bad argument");
  if (n_tabs == 0 || total_rows == 0) return 0;
  TZK_REQUIRE(tabs && weights && max_dim >= 4 && max_dim <= 128 && max_dim % 4 == 0 && n_tabs <= 1024,
              "peer_small_update: dims must be multiples of 4 and <= 128");
  TZK_REQUIRE(opt->optimizer >= 0 && opt->optimizer <= TZK_OPT_LARS_SGD, "peer_small_update: unsupported optimizer");
  TZK_REQUIRE(!opt->weights_f16 || !opt->interleaved, "peer_small_update: interleaved rows are fp32");
  TZK_REQUIRE(opt->optimizer == TZK_OPT_SGD || opt->state, "peer_small_update: optimizer state is NULL");
  TZK_REQUIRE(opt->per_sample_weights == nullptr, "peer_small_update: weighted bags are not supported on the peer step");
  TZK_REQUIRE(!norm_family(*opt) || !opt->interleaved, "peer_small_update: interleaved rows are Adagrad only");
  TZK_REQUIRE((opt->optimizer != TZK_OPT_ADAM && opt->optimizer != TZK_OPT_PARTIAL_ROWWISE_ADAM &&
               opt->optimizer != TZK_OPT_LAMB && opt->optimizer != TZK_OPT_PARTIAL_ROWWISE_LAMB) ||
                  (opt->state2 && opt->step),
              "peer_small_update: Adam and LAMB variants need state2 and the device step counter");
  BwdArgs a;
  a.grad_out = nullptr; a.ld_grad = 0; a.offsets = nullptr; a.weights = weights; a.state = opt->state;
  a.lr = opt->lr; a.eps = opt->eps; a.grad_scale = 1.f; a.F = 0; a.B = 1; a.optimizer = opt->optimizer; a.pooled = 0;
  a.n = total_rows; a.sentinel = 0; a.state2 = opt->state2; a.step = opt->step; a.beta1 = opt->beta1; a.beta2 = opt->beta2;
  a.weight_decay = opt->weight_decay; a.max_gradient = opt->max_gradient; a.bc1 = a.bc2 = 1.f;
  // weights_f16: the owner widens its half row, adds the W fp32 partial sums in rank order, updates in fp32 and rounds
  // the row back to nearest even (finish_run's FP16 path)
  a.peer_w = 0; a.idx_span = 1; a.w_f16 = opt->weights_f16 ? 1 : 0; a.interleaved = opt->interleaved ? 1 : 0;
  a.div_b = make_fast_div(1); a.div_span = make_fast_div(1); a.ld32 = 0; a.wd_mode = opt->weight_decay_mode;
  if (opt->optimizer == TZK_OPT_LARS_SGD) { a.beta1 = opt->momentum; a.beta2 = opt->eta; }
  const bool norm = norm_family(*opt);
  SmallPeers sp;
  for (int r = 0; r < 16; ++r) { sp.psum[r] = r < W ? psum_ptrs[r] : 0ull; sp.flags[r] = r < W ? flag_ptrs[r] : 0ull; }
  int G = 1;
  while (G * 4 < max_dim) G <<= 1;
  const int NG = kThreads / G;
  const int grid = (int)std::min<int64_t>(ceil_div64(total_rows, NG), kSmCountH100 * 8);
  const size_t smem = (size_t)n_tabs * sizeof(SmallTab);
  cudaStream_t st = as_stream(stream);
  const SmallTab* tp = static_cast<const SmallTab*>(tabs);
#define TZK_SMALL_LAUNCH(G_)                                                                                     \
  do {                                                                                                           \
    if (norm) small_table_update_kernel<G_, kFamNorm><<<grid, kThreads, smem, st>>>(a, sp, tp, n_tabs, total_rows, W); \
    else small_table_update_kernel<G_, kFamClassic><<<grid, kThreads, smem, st>>>(a, sp, tp, n_tabs, total_rows, W); \
  } while (0)
  switch (G) {
    case 1: TZK_SMALL_LAUNCH(1); break;
    case 2: TZK_SMALL_LAUNCH(2); break;
    case 4: TZK_SMALL_LAUNCH(4); break;
    case 8: TZK_SMALL_LAUNCH(8); break;
    case 16: TZK_SMALL_LAUNCH(16); break;
    default: TZK_SMALL_LAUNCH(32); break;
  }
#undef TZK_SMALL_LAUNCH
  TZK_CHECK_LAUNCH("small_table_update_kernel");
  return 0;
}

static int fill_wire(PeerWire* pw, const uint64_t* key_ptrs, const uint64_t* idx_ptrs, const uint64_t* count_ptrs,
                     int32_t me, int32_t W, int64_t cap, int32_t idx_span) {
  if (W < 1 || W > 16 || me < 0 || me >= W || cap < 1 || idx_span < 0) return 1;
  if ((int64_t)W * idx_span >= ((int64_t)1 << 31) || (int64_t)W * cap >= ((int64_t)1 << 31)) return 1;
  for (int r = 0; r < 16; ++r) {
    pw->key[r] = (r < W && key_ptrs) ? key_ptrs[r] : 0ull;
    pw->idx[r] = (r < W && idx_ptrs) ? idx_ptrs[r] : 0ull;
    pw->cnt[r] = (r < W && count_ptrs) ? count_ptrs[r] : 0ull;
  }
  pw->me = me; pw->W = W; pw->cap = cap; pw->idx_span = idx_span; pw->pad = 0;
  return 0;
}

// Owner side of the peer-memory backward, id half: pull this rank's chunk of every source's wire buffers
// (tzk_peer_bucketize) into the sort input and sort.  `*_ptrs`: HOST arrays [W] of device addresses (rank r's buffer as
// mapped in this process).  The workspace must be the one later handed to tzk_fused_bwd_apply_peer
// (tzk_fused_bwd_workspace_bytes(W * cap, total_keys, max_dim)).  `overflow` (device int32, may be NULL) is OR-ed with
// every source's overflow flag.
extern "C" int tzk_fused_bwd_sort_peer(const uint64_t* key_ptrs, const uint64_t* idx_ptrs, const uint64_t* count_ptrs,
                                       int32_t me, int32_t W, int64_t cap, int32_t idx_span, int64_t total_keys,
                                       int32_t max_dim, int32_t* overflow, void* workspace, size_t workspace_bytes,
                                       tzk_stream_t stream) {
  PeerWire pw;
  TZK_REQUIRE(key_ptrs && (idx_ptrs || idx_span == 0) && count_ptrs &&
                  fill_wire(&pw, key_ptrs, idx_ptrs, count_ptrs, me, W, cap, idx_span) == 0,
              "fused_bwd_sort_peer: bad wire description");
  return fused_bwd_impl(1, classic_opt(TZK_OPT_SGD, nullptr, 0.f, 0.f), 0, nullptr, 0, nullptr, nullptr, nullptr,
                        nullptr, nullptr, nullptr, nullptr, nullptr, 1, 1, (int64_t)W * cap, total_keys, max_dim, 0,
                        nullptr, 0.f, workspace, workspace_bytes, stream, &pw, nullptr, overflow);
}

// Owner side, gradient half: the run kernels of tzk_fused_bwd_apply over the W * cap sorted wire slots, every gradient
// slice fetched from the source rank's published gradient (grad_ptrs[src]: [B, ld_grad] pooled-output gradient, MEAN
// bags already divided by their length; or [nnz, ld_grad] rows for sequence collections).  B = bags per feature of a
// source batch (pooled) — every rank runs the same batch size.
extern "C" int tzk_fused_bwd_apply_peer(const tzk_opt_args* opt, int32_t pooled, const uint64_t* grad_ptrs,
                                        int64_t ld_grad, const int64_t* feat_w_off, const int64_t* feat_rows,
                                        const int32_t* feat_dim, const int32_t* feat_col, const int32_t* feat_pool,
                                        const int64_t* feat_key_base, int32_t F, int32_t B, int32_t me, int32_t W,
                                        int64_t cap, int32_t idx_span, int64_t total_keys, int32_t max_dim,
                                        int32_t vec_ok, float* weights, float grad_scale, void* workspace,
                                        size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(opt != nullptr && grad_ptrs != nullptr, "fused_bwd_apply_peer: NULL argument");
  TZK_REQUIRE(opt->per_sample_weights == nullptr, "fused_bwd_apply_peer: weighted bags are not supported on the peer step");
  PeerWire pw;
  TZK_REQUIRE(fill_wire(&pw, nullptr, nullptr, nullptr, me, W, cap, idx_span) == 0,
              "fused_bwd_apply_peer: bad wire description");
  TZK_REQUIRE(!pooled || (int64_t)F * B <= idx_span, "fused_bwd_apply_peer: idx_span smaller than F * B");
  return fused_bwd_impl(2, *opt, pooled, nullptr, ld_grad, feat_w_off, feat_rows, feat_dim, feat_col, feat_pool,
                        feat_key_base, nullptr, nullptr, F, B, (int64_t)W * cap, total_keys, max_dim, vec_ok, weights,
                        grad_scale, workspace, workspace_bytes, stream, &pw, grad_ptrs, nullptr);
}

extern "C" int tzk_bag_grad_expand(const float* grad_out, int64_t ld_grad, const int32_t* feat_col,
                                   const int32_t* feat_pool, const int64_t* offsets, const int32_t* slot,
                                   int32_t F, int32_t B, int32_t D, float* g_rows, tzk_stream_t stream) {
  TZK_REQUIRE(F >= 0 && B >= 0 && D >= 1, "bag_grad_expand: bad sizes");
  if (F == 0 || B == 0) return 0;
  TZK_REQUIRE(grad_out && feat_col && feat_pool && offsets && slot && g_rows, "bag_grad_expand: NULL argument");
  cudaStream_t st = as_stream(stream);
  const bool vec = (D % 4 == 0) && ((uintptr_t)grad_out % 16 == 0) && ((uintptr_t)g_rows % 16 == 0) && (ld_grad % 4 == 0);
  const int64_t items = (int64_t)F * B * (vec ? D / 4 : D);
  const int grid = (int)std::min<int64_t>(ceil_div64(items, kThreads), kSmCountH100 * 16);
  if (vec)
    bag_grad_expand_kernel<<<grid, kThreads, 0, st>>>(grad_out, ld_grad, feat_col, feat_pool, offsets, slot, F, B, D,
                                                       g_rows);
  else
    bag_grad_expand_scalar_kernel<<<grid, kThreads, 0, st>>>(grad_out, ld_grad, feat_col, feat_pool, offsets, slot,
                                                              F, B, D, g_rows);
  TZK_CHECK_LAUNCH("bag_grad_expand_kernel");
  return 0;
}
