// tzk_core.cu — error plumbing, device query, K3 lengths->offsets scan.
#include <stdarg.h>
#include <string.h>

#include "tzk_common.cuh"

namespace tzk {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace tzk

using namespace tzk;

extern "C" int tzk_abi_version(void) { return TZK_ABI_VERSION; }
extern "C" const char* tzk_last_error(void) { return tzk::g_err; }
extern "C" int tzk_sm_count(void) {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return n;
}

// ----------------------------------------------------------------------------------------------------
// K3: lengths (int32) -> offsets (int64), exclusive scan with a trailing total.
// Three small kernels (tile sums, scan of tile sums, tile scan + carry).  The input is F*B int32
// (6.8 MB at cfg2) and is read twice; the scan is < 1% of the step's bytes, so no decoupled look-back.
// ----------------------------------------------------------------------------------------------------
namespace {
constexpr int kScanThreads = 256;
constexpr int kScanItems = 16;  // per thread
constexpr int kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ int64_t warp_incl_scan(int64_t v, int lane) {
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    int64_t o = __shfl_up_sync(0xffffffffu, v, d);
    if (lane >= d) v += o;
  }
  return v;
}

// block-wide exclusive scan of one int64 per thread; returns exclusive prefix, total in *total
__device__ __forceinline__ int64_t block_excl_scan(int64_t v, int64_t* total) {
  __shared__ int64_t warp_tot[kScanThreads / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int64_t incl = warp_incl_scan(v, lane);
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    int64_t t = lane < kScanThreads / 32 ? warp_tot[lane] : 0;
    int64_t ti = warp_incl_scan(t, lane);
    if (lane < kScanThreads / 32) warp_tot[lane] = ti - t;  // exclusive warp base
    if (lane == kScanThreads / 32 - 1) *total = ti;
  }
  __syncthreads();
  int64_t r = warp_tot[wid] + incl - v;
  return r;
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_sums(const int32_t* __restrict__ len, int64_t n,
                                                                int64_t* __restrict__ tile_sum) {
  __shared__ int64_t total;
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
  int64_t s = 0;
  // coalesced: thread t reads base + k*256 + t
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    int64_t i = base + (int64_t)k * kScanThreads + threadIdx.x;
    if (i < n) s += len[i];
  }
  (void)block_excl_scan(s, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// single block: exclusive scan of the tile sums in place
__global__ void __launch_bounds__(kScanThreads) scan_tile_offsets(int64_t* __restrict__ tile_sum,
                                                                   int64_t n_tiles) {
  __shared__ int64_t total;
  __shared__ int64_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  for (int64_t base = 0; base < n_tiles; base += kScanThreads) {
    int64_t i = base + threadIdx.x;
    int64_t v = i < n_tiles ? tile_sum[i] : 0;
    int64_t ex = block_excl_scan(v, &total);
    int64_t carry = carry_s;
    if (i < n_tiles) tile_sum[i] = carry + ex;
    __syncthreads();
    if (threadIdx.x == 0) carry_s = carry + total;
    __syncthreads();
  }
}

// STAGED: the offsets leave through shared memory as full-line stores (TZK_SCAN_STAGED); otherwise every thread writes
// its 16 results directly (128-B stride between neighbouring lanes)
template <bool STAGED>
__global__ void __launch_bounds__(kScanThreads) scan_tiles(const int32_t* __restrict__ len, int64_t n,
                                                            const int64_t* __restrict__ tile_off,
                                                            int64_t* __restrict__ offsets) {
  __shared__ int64_t total;
  // one staging buffer, two uses: the tile's lengths (int32, coalesced in), then its offsets (int64, coalesced out)
  __shared__ __align__(16) int64_t stage[kScanTile];
  int32_t* vals = reinterpret_cast<int32_t*>(stage);
  const int64_t base = (int64_t)blockIdx.x * kScanTile;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    int64_t i = base + (int64_t)k * kScanThreads + threadIdx.x;
    vals[k * kScanThreads + threadIdx.x] = i < n ? len[i] : 0;
  }
  __syncthreads();
  // thread t owns items [t*16, t*16+16) of the tile
  int64_t loc[kScanItems];
  int64_t s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    loc[k] = s;
    s += vals[threadIdx.x * kScanItems + k];
  }
  int64_t ex = block_excl_scan(s, &total) + tile_off[blockIdx.x];   // (its barriers also fence the reads of `vals`)
  if (STAGED) {
    // a thread's 16 results are 128 B apart from its neighbour's: through shared memory, then full-line stores
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) stage[threadIdx.x * kScanItems + k] = ex + loc[k];
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      const int j = k * kScanThreads + threadIdx.x;
      if (base + j < n) offsets[base + j] = stage[j];
    }
  } else {
#pragma unroll
    for (int k = 0; k < kScanItems; ++k) {
      int64_t i = base + threadIdx.x * kScanItems + k;
      if (i < n) offsets[i] = ex + loc[k];
    }
  }
  if (base + kScanTile >= n && threadIdx.x == 0) {
    // last tile: trailing total
    offsets[n] = tile_off[blockIdx.x] + total;
  }
}
__global__ void scan_empty(int64_t* offsets) { offsets[0] = 0; }
}  // namespace

extern "C" size_t tzk_lengths_to_offsets_workspace_bytes(int64_t n) {
  int64_t tiles = n <= 0 ? 1 : ceil_div64(n, kScanTile);
  return (size_t)tiles * sizeof(int64_t);
}

extern "C" int tzk_lengths_to_offsets(const int32_t* lengths, int64_t n, int64_t* offsets, void* workspace,
                                      size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(n >= 0, "lengths_to_offsets: n < 0");
  TZK_REQUIRE(offsets != nullptr, "lengths_to_offsets: offsets is NULL");
  cudaStream_t st = as_stream(stream);
  if (n == 0) {
    scan_empty<<<1, 1, 0, st>>>(offsets);
    TZK_CHECK_LAUNCH("scan_empty");
    return 0;
  }
  TZK_REQUIRE(lengths != nullptr, "lengths_to_offsets: lengths is NULL");
  TZK_REQUIRE(workspace_bytes >= tzk_lengths_to_offsets_workspace_bytes(n) && workspace != nullptr,
              "lengths_to_offsets: workspace too small (%zu < %zu)", workspace_bytes,
              tzk_lengths_to_offsets_workspace_bytes(n));
  int64_t tiles = ceil_div64(n, kScanTile);
  int64_t* tile_sum = static_cast<int64_t*>(workspace);
  scan_tile_sums<<<(unsigned)tiles, kScanThreads, 0, st>>>(lengths, n, tile_sum);
  TZK_CHECK_LAUNCH("scan_tile_sums");
  scan_tile_offsets<<<1, kScanThreads, 0, st>>>(tile_sum, tiles);
  TZK_CHECK_LAUNCH("scan_tile_offsets");
  const char* staged_env = getenv("TZK_SCAN_STAGED");      // default on; 0: direct stores
  if (!(staged_env && staged_env[0] == '0')) scan_tiles<true><<<(unsigned)tiles, kScanThreads, 0, st>>>(lengths, n, tile_sum, offsets);
  else scan_tiles<false><<<(unsigned)tiles, kScanThreads, 0, st>>>(lengths, n, tile_sum, offsets);
  TZK_CHECK_LAUNCH("scan_tiles");
  return 0;
}
