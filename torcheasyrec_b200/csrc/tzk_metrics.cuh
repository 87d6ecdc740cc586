// tzk_metrics.cuh — the update of the binned binary AUROC (torchmetrics.AUROC(task="binary", thresholds=T), the `auc`
// metric of tzrec/models/rank_model.py:296-302 and :392-398).
//
// torchmetrics keeps a [T, 2, 2] confusion matrix: sample (p, y) counts as predicted positive at threshold k iff
// p >= thr[k].  With thr nondecreasing that matrix is a function of a histogram: bin(p) = #{k : p >= thr[k]} in 0..T,
// and tps[k] = #{positives with bin > k}, fps[k] the same over negatives (fns / tns are the complements).  This kernel
// builds that histogram, counts[(T + 1)][2] (label-minor), accumulating into an int64 buffer:
//   - bin(p) is a branchless binary search over the thresholds themselves (never floor(p * (T - 1)): that arithmetic
//     form disagrees with p >= thr[k] at float32 linspace values);
//   - a label outside {0, 1}, or a prediction that is NaN or outside [0, 1], is not binned: it adds 1 to *invalid;
//   - grid from the SM count, grid-stride loop over 16-B vectors of predictions (4 fp32 or 8 bf16) and the matching
//     labels, scalar tail;
//   - the thresholds and a uint32 histogram live in shared memory (12 T bytes + 8), updated with shared atomics; each CTA
//     then adds its non-zero bins to the global counts.  A T whose tables do not fit in shared memory takes the
//     instantiation that reads the thresholds from global memory and adds to the global counts directly.
// Integer atomics only: the counts do not depend on the order in which threads arrive.
//
// Plain CUDA (no PTX): the includer provides TZK_DYN_SMEM / TZK_LAUNCH (nvcc: tzk_metrics.cu; g++ +
// tests/native/cuda_cpu_shim.h: tests/test_binned_auc_cpu.py runs this source on the host against a numpy restatement).
#pragma once
#include <stdint.h>

namespace tzk_auc {
constexpr int kThreads = 512;
constexpr int kMaxCtasPerSm = 4;                        // 4 x 512 threads = the 2048 an sm_90 SM holds
constexpr size_t kSmemPerSm = 227 * 1024;               // largest shared memory one CTA may opt into (sm_90)
constexpr size_t kSmemPerCtaReserved = 1024;            // the runtime's own share per resident CTA
// dynamic budget: the opt-in maximum less room for the kernel's static shared memory (s_bad: 16 B in ptxas -v)
constexpr size_t kDynSmemMax = kSmemPerSm - 256;

__host__ __device__ inline size_t thr_bytes(int T) { return ((size_t)T * sizeof(float) + 15) / 16 * 16; }
inline size_t smem_bytes(int T) { return thr_bytes(T) + (size_t)(T + 1) * 2 * sizeof(uint32_t); }
inline bool fits_shared(int T) { return smem_bytes(T) <= kDynSmemMax; }

__device__ __forceinline__ float pred_f32(float p) { return p; }
__device__ __forceinline__ float pred_f32(uint16_t h) { return __uint_as_float((uint32_t)h << 16); }   // bf16 bits
__device__ __forceinline__ int label_bit(float y) { return y == 0.0f ? 0 : (y == 1.0f ? 1 : -1); }
__device__ __forceinline__ int label_bit(int64_t y) { return y == 0 ? 0 : (y == 1 ? 1 : -1); }

// #{k < T : thr[k] <= p} for a nondecreasing thr, T >= 1: ceil(log2 T) selects, no data-dependent branch.
// (NaN compares false everywhere; it is counted invalid before it gets here)
__device__ __forceinline__ int bin_of(const float* thr, int T, float p) {
  const float* b = thr;
  int len = T;
  while (len > 1) {
    const int half = len >> 1;
    b += (b[half] <= p) ? half : 0;
    len -= half;
  }
  return (int)(b - thr) + (*b <= p ? 1 : 0);
}

template <typename P> struct alignas(16) PredVec { P v[16 / sizeof(P)]; };
template <typename L, int V> struct alignas(16) LabelVec { L v[V]; };

template <bool kShared, typename P, typename L>
__global__ void __launch_bounds__(kThreads) binned_auc_kernel(const P* __restrict__ pred, const L* __restrict__ label,
                                                              int64_t n, int vec, const float* __restrict__ thr_g, int T,
                                                              unsigned long long* counts, unsigned long long* invalid) {
  constexpr int V = 16 / sizeof(P);
  TZK_DYN_SMEM(float, smem);
  __shared__ unsigned s_bad;
  float* s_thr = smem;
  uint32_t* s_hist = reinterpret_cast<uint32_t*>(reinterpret_cast<unsigned char*>(smem) + thr_bytes(T));
  const int nb = 2 * (T + 1);
  if (kShared) {
    for (int i = threadIdx.x; i < T; i += blockDim.x) s_thr[i] = thr_g[i];
    for (int i = threadIdx.x; i < nb; i += blockDim.x) s_hist[i] = 0u;
  }
  if (threadIdx.x == 0) s_bad = 0u;
  __syncthreads();
  const float* thr = kShared ? s_thr : thr_g;
  unsigned bad = 0;
  auto add = [&](float p, int y) {
    if (y < 0 || !(p >= 0.0f && p <= 1.0f)) {
      ++bad;
      return;
    }
    const int slot = bin_of(thr, T, p) * 2 + y;
    if (kShared) atomicAdd(&s_hist[slot], 1u);
    else atomicAdd(&counts[slot], 1ull);
  };
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t done = 0;
  if (vec) {
    const int64_t nv = n / V;
    const PredVec<P>* pv = reinterpret_cast<const PredVec<P>*>(pred);
    const LabelVec<L, V>* lv = reinterpret_cast<const LabelVec<L, V>*>(label);
    for (int64_t c = t0; c < nv; c += stride) {
      const PredVec<P> p = pv[c];
      const LabelVec<L, V> y = lv[c];
#pragma unroll
      for (int j = 0; j < V; ++j) add(pred_f32(p.v[j]), label_bit(y.v[j]));
    }
    done = nv * V;
  }
  for (int64_t i = done + t0; i < n; i += stride) add(pred_f32(pred[i]), label_bit(label[i]));
  if (bad) atomicAdd(&s_bad, bad);
  __syncthreads();
  if (kShared) {
    for (int i = threadIdx.x; i < nb; i += blockDim.x) {
      const uint32_t c = s_hist[i];
      if (c) atomicAdd(&counts[i], (unsigned long long)c);
    }
  }
  if (threadIdx.x == 0 && s_bad) atomicAdd(invalid, (unsigned long long)s_bad);
}

template <bool kShared, typename P, typename L>
inline int launch(const void* pred, const void* label, int64_t n, const float* thr, int T, int64_t* counts,
                  int64_t* invalid, int sm_count, cudaStream_t st) {
  const bool vec = (reinterpret_cast<uintptr_t>(pred) % 16 == 0) && (reinterpret_cast<uintptr_t>(label) % 16 == 0);
  const int64_t items = vec ? n / (int64_t)(16 / sizeof(P)) + n % (int64_t)(16 / sizeof(P)) : n;
  const size_t smem = kShared ? smem_bytes(T) : 0;
  // CTAs per SM: as many as can be resident at once (registers, shared memory), so the grid is one wave
#ifdef TZK_CPU_SHIM
  int per_sm = kShared ? (int)(kSmemPerSm / (smem + kSmemPerCtaReserved)) : kMaxCtasPerSm;
#else
  if (smem > 48 * 1024 &&
      cudaFuncSetAttribute(binned_auc_kernel<kShared, P, L>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) !=
          cudaSuccess) {
    cudaGetLastError();
    return 4;                          // the tables do not fit after all: the caller takes the global-atomic kernel
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, binned_auc_kernel<kShared, P, L>, kThreads, smem) !=
      cudaSuccess) {
    cudaGetLastError();
    per_sm = 1;
  }
#endif
  per_sm = per_sm < 1 ? 1 : (per_sm > kMaxCtasPerSm ? kMaxCtasPerSm : per_sm);
  int64_t grid = (items + kThreads - 1) / kThreads;
  const int64_t cap = (int64_t)(sm_count > 0 ? sm_count : 132) * per_sm;
  grid = grid < 1 ? 1 : (grid > cap ? cap : grid);
  TZK_LAUNCH((binned_auc_kernel<kShared, P, L>), (unsigned)grid, kThreads, smem, st, static_cast<const P*>(pred),
             static_cast<const L*>(label), n, (int)vec, thr, T, reinterpret_cast<unsigned long long*>(counts),
             reinterpret_cast<unsigned long long*>(invalid));
  return cudaGetLastError() == cudaSuccess ? 0 : 3;
}

// pred_dtype 0 = fp32, 1 = bf16 (16-bit patterns); label_dtype 0 = fp32, 1 = int64.  Returns 0, 1 (bad argument) or 3
// (launch failure).  A shared-memory instantiation whose opt-in is refused is replaced by the global-atomic one.
inline int run(const void* pred, int pred_dtype, const void* label, int label_dtype, int64_t n, const float* thr, int T,
               int64_t* counts, int64_t* invalid, cudaStream_t st) {
  if (n < 0 || T < 1 || pred_dtype < 0 || pred_dtype > 1 || label_dtype < 0 || label_dtype > 1) return 1;
  if (!thr || !counts || !invalid || (n > 0 && (!pred || !label))) return 1;
  if (n == 0) return 0;
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    sms = 0;
  const bool sh = fits_shared(T);
#define TZK_AUC_PL(P_, L_)                                                                                            \
  do {                                                                                                                \
    const int rc_ = sh ? launch<true, P_, L_>(pred, label, n, thr, T, counts, invalid, sms, st) : 4;                  \
    return rc_ == 4 ? launch<false, P_, L_>(pred, label, n, thr, T, counts, invalid, sms, st) : rc_;                  \
  } while (0)
  if (pred_dtype == 0) {
    if (label_dtype == 0) TZK_AUC_PL(float, float);
    TZK_AUC_PL(float, int64_t);
  }
  if (label_dtype == 0) TZK_AUC_PL(uint16_t, float);
  TZK_AUC_PL(uint16_t, int64_t);
#undef TZK_AUC_PL
}
}  // namespace tzk_auc
