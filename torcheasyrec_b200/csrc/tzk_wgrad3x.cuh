// tzk_wgrad3x.cuh — the weight gradient of the wide tower layer,  dW[n, k] = sum_m dZ[m, n] * X[m, k]  (n < 64, m < M =
// batch), on mma.sync m16n8k8 with the 3xTF32 split.  Shared by tzk_gemm3x.cu (tzk_wgrad3x: X is one tensor) and
// tzk_interact_wide.cu (tzk_interact_wide_wgrad: X = [pairs | dense | sparse] of DLRM-Criteo's interaction, never
// materialised; its own wgmma kernel on these work items, partials and reduction).  Included inside the includer's
// anonymous namespace after tzk_sm90_ptx.h (or sm90_cpu_emu.h) and tzk_tma.h; the includer provides TZK_DYN_SMEM /
// TZK_LAUNCH.
//
// X is read as 32-column TMA boxes.  Box b belongs to source s (first[s] <= b < first[s + 1]) and covers its columns
// col0[s] + 32 (b - first[s]) ..; its dW columns are dst[s] + 32 (b - first[s]) .., those below width[s] are written.
// dW columns are independent sums over the batch, so where a box comes from changes no bit of any column.
//
// Work item = (column tile j of 4 boxes = 128 columns, row slab s); each CTA owns one item and computes the [64 x 128]
// block dZ[slab]^T X[slab, tile] with A = dZ^T and B = X straight from the row-major boxes, streaming the slab in chunks
// of 32 rows (4 k-steps of 8).  Warp w: n rows 16 (w % 4) .. +16, X columns 64 (w / 4) .. +64.  The partial block goes
// to `partial`; wgrad_reduce_kernel adds the slabs in a fixed order and scatters the columns to dW.  X is read exactly
// once over all items (tiles read disjoint boxes); dZ is re-read by the column tiles from L2.
// Per stage: X (4 boxes of 32 rows x 128 B = 16 KB) | dZ (2 boxes = 8 KB).
#pragma once

constexpr int WG_THREADS = 256;
constexpr int WG_ROWS = 32;                         // batch rows per chunk = 4 k-steps
constexpr int WG_BOX = WG_ROWS * 128;               // one TMA box: 32 rows x 32 floats = 4 KB
constexpr int WG_A = 4 * WG_BOX, WG_B = 2 * WG_BOX; // 16 KB, 8 KB
constexpr int WG_STAGE = WG_A + WG_B;               // 24 KB
constexpr int WG_STAGES = 4;                        // 96 KB: two CTAs per SM
constexpr int WG_SRC = 3;                           // X sources at most

struct WgSources {
  int first[WG_SRC + 1];   // box ranges, first[0] = 0; first[WG_SRC] = boxes
  int col0[WG_SRC];        // source column of the range's first box
  int dst[WG_SRC];         // dW column of the range's first column
  int width[WG_SRC];       // source columns that reach dW
};

struct WgParams {
  float* partial;      // [slabs, k_tiles * 128, 64]
  int64_t M;           // batch rows
  int64_t slab_rows;   // multiple of 32
  int k_tiles;         // ceil(boxes / 4)
  WgSources src;
  const float* dz_scale;   // nullable: dZ is read times *dz_scale (interact_wide_wgrad_kernel; wgrad3x_kernel: null)
};

__device__ __forceinline__ int wg_source(const WgSources& s, int box) {
  return box >= s.first[2] ? 2 : box >= s.first[1] ? 1 : 0;
}
// v[s] by selects (a dynamically indexed parameter array would go through local memory)
__device__ __forceinline__ int wg_pick(const int* v, int s) { return s == 0 ? v[0] : s == 1 ? v[1] : v[2]; }

__global__ void __launch_bounds__(WG_THREADS, 2)
wgrad3x_kernel(const __grid_constant__ CUtensorMap map_x0, const __grid_constant__ CUtensorMap map_x1,
               const __grid_constant__ CUtensorMap map_x2, const __grid_constant__ CUtensorMap map_dz, WgParams p) {
  TZK_DYN_SMEM(uint8_t, smem);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + WG_STAGES * WG_STAGE);
  // this tile's boxes: source [0 .. 4), column [4 .. 8).  Thread 0 reads them back in every load: kept in registers
  // across the main loop they would be spilled.
  int* boxes = reinterpret_cast<int*>(full + WG_STAGES);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int jt = blockIdx.x % p.k_tiles;                  // column tile of X
  const int64_t slab = blockIdx.x / p.k_tiles;
  const int64_t row0 = slab * p.slab_rows;
  const int64_t rows = (p.M - row0 < p.slab_rows) ? p.M - row0 : p.slab_rows;
  const int num_c = (int)((rows + WG_ROWS - 1) / WG_ROWS);  // rows past M are zero-filled by the TMA

  if (threadIdx.x == 0) {
    for (int s = 0; s < WG_STAGES; ++s) mbar_init(full + s, 1);
    fence_mbarrier_init();
    for (int b = 0; b < 4; ++b) {
      const int box = jt * 4 + b, s = wg_source(p.src, box);
      boxes[b] = s;
      boxes[4 + b] = wg_pick(p.src.col0, s) + 32 * (box - wg_pick(p.src.first, s));
    }
  }
  __syncthreads();
  auto load = [&](int c) {                                // thread 0 only
    uint8_t* sb = smem + (c % WG_STAGES) * WG_STAGE;
    uint64_t* bar = full + c % WG_STAGES;
    const int r = (int)(row0 + (int64_t)c * WG_ROWS);
    mbar_expect_tx(bar, WG_A + WG_B);
#pragma unroll 1
    for (int b = 0; b < 4; ++b) {
      const int s = *reinterpret_cast<volatile int*>(boxes + b), col = *reinterpret_cast<volatile int*>(boxes + 4 + b);
      tma_load_2d(sb + b * WG_BOX, s == 0 ? &map_x0 : s == 1 ? &map_x1 : &map_x2, bar, col, r);
    }
#pragma unroll
    for (int b = 0; b < 2; ++b) tma_load_2d(sb + WG_A + b * WG_BOX, &map_dz, bar, b * 32, r);
  };
  if (threadIdx.x == 0)
    for (int c = 0; c < WG_STAGES && c < num_c; ++c) load(c);

  const int n0 = (warp & 3) * 16 + g;                     // this lane's n rows n0 and n0 + 8
  const int kc0 = (warp >> 2) * 64 + g;                   // this lane's X column in n8 tile nt: kc0 + 8 nt
  float acc[8][4], part[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int q = 0; q < 4; ++q) acc[nt][q] = 0.f;
  for (int c = 0; c < num_c; ++c) {
    const int s = c % WG_STAGES;
    mbar_wait(full + s, (uint32_t)(c / WG_STAGES) & 1u);
    const float* xs = reinterpret_cast<const float*>(smem + s * WG_STAGE);
    const float* zs = reinterpret_cast<const float*>(smem + s * WG_STAGE + WG_A);
    // element (m, col) of a [32 rows x 128 floats] operand held as 32-column boxes
    auto at = [](const float* base, int m, int col) { return base[(col >> 5) * (WG_BOX / 4) + swz(m, col & 31)]; };
#pragma unroll
    for (int ks = 0; ks < WG_ROWS / 8; ++ks) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) part[nt][q] = 0.f;
      const int m = ks * 8 + t;                           // batch rows m (a0, a1, b0) and m + 4 (a2, a3, b1)
      const float a[4] = {at(zs, m, n0), at(zs, m, n0 + 8), at(zs, m + 4, n0), at(zs, m + 4, n0 + 8)};
      uint32_t ah[4], al[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        ah[i] = tf32_bits(a[i]);
        al[i] = tf32_bits(a[i] - __uint_as_float(ah[i]));
      }
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        const float b[2] = {at(xs, m, kc0 + 8 * nt), at(xs, m + 4, kc0 + 8 * nt)};
        uint32_t bh[2], bl[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          bh[i] = tf32_bits(b[i]);
          bl[i] = tf32_bits(b[i] - __uint_as_float(bh[i]));
        }
        mma_tf32(part[nt], al, bh);
        mma_tf32(part[nt], ah, bl);
        mma_tf32(part[nt], ah, bh);
      }
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[nt][q] += part[nt][q];
    }
    __syncthreads();
    if (threadIdx.x == 0 && c + WG_STAGES < num_c) load(c + WG_STAGES);
  }
  // c0/c1: n row n0, X columns 2t, 2t+1 of the n8 tile; c2/c3: n row n0 + 8
  float* out = p.partial + ((int64_t)slab * p.k_tiles + jt) * 128 * 64;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int kcol = (warp >> 2) * 64 + nt * 8 + 2 * t;
#pragma unroll
    for (int q = 0; q < 4; ++q) out[(int64_t)(kcol + (q & 1)) * 64 + n0 + 8 * (q >> 1)] = acc[nt][q];
  }
}

// dW[n, dst(k)] = sum over slabs (fixed order) of partial[s, k, n] for the partial columns k that reach dW; one thread
// per (k, n), n fastest for the reads
__global__ void wgrad_reduce_kernel(const float* __restrict__ partial, int slabs, int k_pad, WgSources src,
                                    float* __restrict__ dw, int64_t ld_dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= k_pad * 64) return;
  const int k = i >> 6, n = i & 63;
  const int s = wg_source(src, k >> 5);
  const int c = k - 32 * wg_pick(src.first, s);           // column within the source's range
  if (c >= wg_pick(src.width, s)) return;
  float acc = 0.f;
  for (int sl = 0; sl < slabs; ++sl) acc += partial[((int64_t)sl * k_pad + k) * 64 + n];
  dw[(int64_t)n * ld_dw + wg_pick(src.dst, s) + c] = acc;
}

// dw (columns as `src` maps them) = dz[M, 64]^T @ X, X given by up to WG_SRC tensor maps of [rows x 32] boxes
// (WG_ROWS rows); partial: slabs * k_tiles * 128 * 64 floats, k_tiles = ceil(src.first[WG_SRC] / 4).  Kernel: one with
// wgrad3x_kernel's parameters, work items and partial layout, using `extra_smem` bytes past the stages.
template <auto Kernel = wgrad3x_kernel>
inline int wgrad3x_launch(const CUtensorMap (&mx)[WG_SRC], const CUtensorMap& mz, const WgSources& src, int64_t M,
                          int32_t slabs, float* partial, float* dw, int64_t ld_dw, cudaStream_t st,
                          size_t extra_smem = 0, const float* dz_scale = nullptr) {
  WgParams p;
  p.partial = partial;
  p.dz_scale = dz_scale;
  p.M = M;
  p.k_tiles = (src.first[WG_SRC] + 3) / 4;
  p.slab_rows = ((M + slabs - 1) / slabs + WG_ROWS - 1) / WG_ROWS * WG_ROWS;
  p.src = src;
  const int used = (int)((M + p.slab_rows - 1) / p.slab_rows);           // slabs that hold rows (<= slabs)
  const size_t smem = (size_t)WG_STAGES * WG_STAGE + extra_smem + WG_STAGES * 8 + 8 * 4;
#ifndef TZK_CPU_SHIM
  static bool configured = false;     // once: nothing but the launches happens inside a stream capture
  if (!configured) {
    cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    configured = true;
  }
#endif
  TZK_LAUNCH((Kernel), used * p.k_tiles, WG_THREADS, smem, st, mx[0], mx[1], mx[2], mz, p);
  TZK_LAUNCH((wgrad_reduce_kernel), (p.k_tiles * 128 * 64 + 255) / 256, 256, 0, st, partial, used, p.k_tiles * 128, src,
             dw, ld_dw);
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}
