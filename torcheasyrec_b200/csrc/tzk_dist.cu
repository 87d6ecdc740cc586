// tzk_dist.cu — K1 row-wise block bucketize and K2 KJT segment permute (integer work, bit-exact).
#include "tzk_common.cuh"

using namespace tzk;

namespace {
constexpr int kThreads = 256;
constexpr int kMaxW = 64;

// dest = owner + id / block (row-wise: owner 0, block = ceil(rows/W); table-wise: block >= rows so the
// quotient is 0 and dest = owner; table-row-wise: both).  ids are expected in [0, rows); anything else is
// clamped into a valid rank (fbgemm bounds WARNING mode would have remapped it to row 0 later anyway).
__device__ __forceinline__ int dest_of(int64_t id, int64_t block, int owner, int W, int64_t* local) {
  int64_t q = id < 0 ? 0 : id / block;
  int64_t r = owner + q;
  if (r >= W) { q -= r - (W - 1); r = W - 1; }
  *local = id - q * block;
  return (int)r;
}

__global__ void __launch_bounds__(kThreads)
bucketize_count_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                       const int64_t* __restrict__ feat_block, const int32_t* __restrict__ feat_owner, int F,
                       int B, int W, int32_t* __restrict__ out_lengths) {
  const int64_t n_bags = (int64_t)F * B;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t bag = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; bag < n_bags; bag += stride) {
    const int f = (int)(bag / B);
    const int b = (int)(bag - (int64_t)f * B);
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    const int64_t blk = __ldg(feat_block + f);
    const int own = feat_owner ? __ldg(feat_owner + f) : 0;
    int64_t loc;
    if (e - s == 1) {
      const int r = dest_of(__ldg(ids + s), blk, own, W, &loc);
      for (int w = 0; w < W; ++w) out_lengths[((int64_t)w * F + f) * B + b] = (w == r);
    } else {
      for (int w = 0; w < W; ++w) {
        int32_t c = 0;
        for (int64_t l = s; l < e; ++l) c += (dest_of(__ldg(ids + l), blk, own, W, &loc) == w);
        out_lengths[((int64_t)w * F + f) * B + b] = c;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
bucketize_scatter_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ offsets,
                         const int64_t* __restrict__ feat_block, const int32_t* __restrict__ feat_owner, int F,
                         int B, int W, const int64_t* __restrict__ out_offsets, int64_t* __restrict__ out_ids,
                         int32_t* __restrict__ out_pos, int32_t* __restrict__ out_inv, int64_t cap) {
  // cap > 0: destination r's ids start at r*cap instead of right after destination r-1 (fixed-capacity wire
  // layout of the graph-capturable exchange); slots beyond cap are dropped (the caller checks the counts).
  const int64_t n_bags = (int64_t)F * B;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t bag = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; bag < n_bags; bag += stride) {
    const int f = (int)(bag / B);
    const int b = (int)(bag - (int64_t)f * B);
    const int64_t s = __ldg(offsets + bag), e = __ldg(offsets + bag + 1);
    const int64_t blk = __ldg(feat_block + f);
    const int own = feat_owner ? __ldg(feat_owner + f) : 0;
    int64_t loc;
    if (e - s == 1) {
      const int r = dest_of(__ldg(ids + s), blk, own, W, &loc);
      int64_t o = __ldg(out_offsets + ((int64_t)r * F + f) * B + b);
      if (cap > 0) {
        o = o - __ldg(out_offsets + (int64_t)r * F * B);
        if (o >= cap) { if (out_inv) out_inv[s] = (int32_t)(r * cap); continue; }
        o += (int64_t)r * cap;
      }
      out_ids[o] = loc;
      if (out_pos) out_pos[o] = (int32_t)s;
      if (out_inv) out_inv[s] = (int32_t)o;
    } else if (e > s) {
      int32_t cnt[kMaxW];
      for (int w = 0; w < W; ++w) cnt[w] = 0;
      for (int64_t l = s; l < e; ++l) {
        const int r = dest_of(__ldg(ids + l), blk, own, W, &loc);
        int64_t o = __ldg(out_offsets + ((int64_t)r * F + f) * B + b) + cnt[r]++;
        if (cap > 0) {
          o = o - __ldg(out_offsets + (int64_t)r * F * B);
          if (o >= cap) { if (out_inv) out_inv[l] = (int32_t)(r * cap); continue; }
          o += (int64_t)r * cap;
        }
        out_ids[o] = loc;
        if (out_pos) out_pos[o] = (int32_t)l;
        if (out_inv) out_inv[l] = (int32_t)o;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
permute_lengths_kernel(const int32_t* __restrict__ lengths, const int32_t* __restrict__ perm, int S_out,
                       int B, int32_t* __restrict__ out) {
  const int64_t n = (int64_t)S_out * B;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const int s = (int)(i / B);
    const int b = (int)(i - (int64_t)s * B);
    out[i] = lengths[(int64_t)__ldg(perm + s) * B + b];
  }
}

// segment s of the output is one contiguous run of the input: memcpy-like, blockIdx.y = segment
__global__ void __launch_bounds__(kThreads)
permute_ids_kernel(const int64_t* __restrict__ ids, const int64_t* __restrict__ in_offsets,
                   const int64_t* __restrict__ out_offsets, const int32_t* __restrict__ perm, int B,
                   int64_t* __restrict__ out_ids) {
  const int s = blockIdx.y;
  const int64_t src0 = __ldg(in_offsets + (int64_t)__ldg(perm + s) * B);
  const int64_t dst0 = __ldg(out_offsets + (int64_t)s * B);
  const int64_t n = __ldg(out_offsets + (int64_t)(s + 1) * B) - dst0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out_ids[dst0 + i] = ids[src0 + i];
}

// the per-sample weights of a weighted KJT travel with its ids: the same segment copy over 4-B floats
__global__ void __launch_bounds__(kThreads)
permute_weights_kernel(const float* __restrict__ w, const int64_t* __restrict__ in_offsets,
                       const int64_t* __restrict__ out_offsets, const int32_t* __restrict__ perm, int B,
                       float* __restrict__ out_w) {
  const int s = blockIdx.y;
  const int64_t src0 = __ldg(in_offsets + (int64_t)__ldg(perm + s) * B);
  const int64_t dst0 = __ldg(out_offsets + (int64_t)s * B);
  const int64_t n = __ldg(out_offsets + (int64_t)(s + 1) * B) - dst0;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    out_w[dst0 + i] = w[src0 + i];
}
}  // namespace

extern "C" size_t tzk_bucketize_rw_workspace_bytes(int32_t F, int32_t B, int32_t W, int64_t nnz) {
  (void)nnz;
  return tzk_lengths_to_offsets_workspace_bytes((int64_t)F * B * W);
}

extern "C" int tzk_bucketize_rw(const int64_t* ids, const int64_t* offsets, int32_t F, int32_t B, int32_t W,
                                const int64_t* feat_block, const int32_t* feat_owner, int64_t nnz,
                                int64_t wire_capacity, int32_t* out_lengths, int64_t* out_offsets, int64_t* out_ids,
                                int32_t* out_pos, int32_t* out_inv, void* workspace, size_t workspace_bytes,
                                tzk_stream_t stream) {
  TZK_REQUIRE(wire_capacity >= 0 && wire_capacity * W < ((int64_t)1 << 31), "bucketize_rw: bad wire_capacity");
  TZK_REQUIRE(F >= 0 && B >= 0 && nnz >= 0, "bucketize_rw: negative size");
  TZK_REQUIRE(W >= 1 && W <= kMaxW, "bucketize_rw: W=%d out of range [1,%d]", W, kMaxW);
  TZK_REQUIRE(nnz < ((int64_t)1 << 31), "bucketize_rw: nnz >= 2^31");
  TZK_REQUIRE(out_offsets, "bucketize_rw: out_offsets is NULL");
  const int64_t n_bags = (int64_t)F * B;
  cudaStream_t st = as_stream(stream);
  if (n_bags == 0) return tzk_lengths_to_offsets(nullptr, 0, out_offsets, workspace, workspace_bytes, stream);
  TZK_REQUIRE(offsets && feat_block && out_lengths && (nnz == 0 || (ids && out_ids)),
              "bucketize_rw: NULL argument");
  int grid = (int)(ceil_div64(n_bags, kThreads) < kSmCountH100 * 16 ? ceil_div64(n_bags, kThreads)
                                                                   : kSmCountH100 * 16);
  bucketize_count_kernel<<<grid, kThreads, 0, st>>>(ids, offsets, feat_block, feat_owner, F, B, W, out_lengths);
  TZK_CHECK_LAUNCH("bucketize_count_kernel");
  int rc = tzk_lengths_to_offsets(out_lengths, n_bags * W, out_offsets, workspace, workspace_bytes, stream);
  if (rc) return rc;
  if (nnz > 0) {
    bucketize_scatter_kernel<<<grid, kThreads, 0, st>>>(ids, offsets, feat_block, feat_owner, F, B, W,
                                                        out_offsets, out_ids, out_pos, out_inv, wire_capacity);
    TZK_CHECK_LAUNCH("bucketize_scatter_kernel");
  }
  return 0;
}

extern "C" int tzk_permute_lengths(const int32_t* lengths, const int32_t* perm, int32_t S_out, int32_t B,
                                   int32_t* out_lengths, tzk_stream_t stream) {
  TZK_REQUIRE(S_out >= 0 && B >= 0, "permute_lengths: negative size");
  const int64_t n = (int64_t)S_out * B;
  if (n == 0) return 0;
  TZK_REQUIRE(lengths && perm && out_lengths, "permute_lengths: NULL argument");
  int grid = (int)(ceil_div64(n, kThreads) < kSmCountH100 * 16 ? ceil_div64(n, kThreads) : kSmCountH100 * 16);
  permute_lengths_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(lengths, perm, S_out, B, out_lengths);
  TZK_CHECK_LAUNCH("permute_lengths_kernel");
  return 0;
}

extern "C" int tzk_permute_ids(const int64_t* ids, const int64_t* in_offsets, const int64_t* out_offsets,
                               const int32_t* perm, int32_t S_out, int32_t B, int64_t* out_ids,
                               tzk_stream_t stream) {
  TZK_REQUIRE(S_out >= 0 && B >= 0, "permute_ids: negative size");
  if (S_out == 0 || B == 0) return 0;
  TZK_REQUIRE(S_out <= 65535, "permute_ids: S_out=%d > 65535", S_out);
  TZK_REQUIRE(in_offsets && out_offsets && perm, "permute_ids: NULL argument");
  // grid.x sized for the typical segment (B ids); longer segments loop
  int gx = (int)(ceil_div64(B, kThreads) < 64 ? ceil_div64(B, kThreads) : 64);
  dim3 grid(gx, S_out);
  permute_ids_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(ids, in_offsets, out_offsets, perm, B, out_ids);
  TZK_CHECK_LAUNCH("permute_ids_kernel");
  return 0;
}

extern "C" int tzk_permute_weights(const float* weights, const int64_t* in_offsets, const int64_t* out_offsets,
                                   const int32_t* perm, int32_t S_out, int32_t B, float* out_weights,
                                   tzk_stream_t stream) {
  TZK_REQUIRE(S_out >= 0 && B >= 0, "permute_weights: negative size");
  if (S_out == 0 || B == 0) return 0;
  TZK_REQUIRE(S_out <= 65535, "permute_weights: S_out=%d > 65535", S_out);
  TZK_REQUIRE(in_offsets && out_offsets && perm, "permute_weights: NULL argument");
  int gx = (int)(ceil_div64(B, kThreads) < 64 ? ceil_div64(B, kThreads) : 64);
  dim3 grid(gx, S_out);
  permute_weights_kernel<<<grid, kThreads, 0, as_stream(stream)>>>(weights, in_offsets, out_offsets, perm, B,
                                                                    out_weights);
  TZK_CHECK_LAUNCH("permute_weights_kernel");
  return 0;
}
