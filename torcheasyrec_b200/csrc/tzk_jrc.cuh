// tzk_jrc.cuh — the JRC loss (tzrec/loss/jrc_loss.py, https://arxiv.org/abs/2208.06164) and its gradient in O(B), for
// two-class logits l = (l0, l1), labels y in {0, 1} and one session id per sample:
//
//   ce_i = logsumexp(l0_i, l1_i) - l_{y_i, i}
//   y_i = 1: ge_i = log(exp(l1_i) + sum_{j in s(i), y_j = 0} exp(l1_j)) - l1_i
//   y_i = 0: ge_i = log(exp(l0_i) + sum_{j in s(i), y_j = 1} exp(l0_j)) - l0_i
//   loss = (1 / B) sum_i w_i (alpha ce_i + (1 - alpha) ge_i),  w_i = 1 (mean) or the caller's per-sample weight
//
// The samples arrive sorted by session (tzk_jrc.cu's radix sort: perm[k] is the k-th sample in session order, skey[k]
// its session id), so every session is a run of consecutive positions.  Each per-session quantity is a segmented
// reduction of pairs (m, s) = (max, sum of exp(x - max)), combined as (m, s) + (m', s') = (M, s e^(m-M) + s' e^(m'-M)):
//   pass 1  per session: (M1, S1) over the negatives' l1 and (M0, S0) over the positives' l0;
//   pass 2  per sample:  Z_i = exp(x_i - m_i) + S e^(M - m_i) (x_i = l1_i, (M, S) = (M1, S1) for a positive; l0_i and
//           (M0, S0) for a negative; m_i = max(x_i, M)), ce_i, ge_i, the loss term and the sample's own gradient;
//           per session: T1 = sum over positives of c_i e^(M1 - m_i) / Z_i, T0 = the same over negatives with M0
//           (c_i = w_i / B; plain sums, carried as pairs with m = 0);
//   pass 3  the cross terms: a negative j gets (1 - alpha) e^(l1_j - M1) T1 on dl1, a positive j gets
//           (1 - alpha) e^(l0_j - M0) T0 on dl0.
// Every exponent is <= 0 after its shift.
//
// A CTA owns a chunk of kChunk consecutive positions and reduces it with a segmented Hillis-Steele scan in shared
// memory, so a run of any length costs log2(kChunk) steps per chunk.  A session that crosses chunks is completed by
// carry_kernel: one CTA scans the chunks' first and last pieces the same way, kChunk chunks per step, and gives each
// crossing session one total.  No float atomics: every sum has a fixed order, so a graph replay gives the eager call's
// bits.
//
// The loss is NaN where the reference's is: B = 0, and in mean mode a batch without a positive or without a negative
// (an empty cross-entropy mean times 0); the gradient stays finite there.  A label outside {0, 1} (the reference raises
// inside CrossEntropyLoss) makes the loss and that sample's gradient row NaN, with no device assert.
//
// fp32.  Plain CUDA (no PTX): nvcc builds it in tzk_jrc.cu; g++ + tests/native/cuda_cpu_shim.h:
// tests/test_dbmtl_cpu.py runs this source on the host against float64.
#pragma once
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "tzk_launch.cuh"

namespace tzk_jrc {
constexpr int kChunk = 256;   // positions per CTA, one per thread

struct Pair {
  float m, s;
};
struct Val {                  // two independent pairs: (a) for the negatives' side, (b) for the positives' side
  Pair a, b;
};
struct ChunkSum {             // one chunk of a segmented reduction: its first and last piece, and whether it is one piece
  Val first, last;
  int single, pad_[3];
};

__device__ __forceinline__ Pair pair_id() { return Pair{-INFINITY, 0.f}; }
__device__ __forceinline__ Pair pair_add(Pair x, Pair y) {
  if (x.m == -INFINITY) return y;
  if (y.m == -INFINITY) return x;
  const float M = fmaxf(x.m, y.m);
  return Pair{M, x.s * expf(x.m - M) + y.s * expf(y.m - M)};
}
__device__ __forceinline__ Val val_id() { return Val{pair_id(), pair_id()}; }
__device__ __forceinline__ Val val_add(const Val& x, const Val& y) { return Val{pair_add(x.a, y.a), pair_add(x.b, y.b)}; }

__host__ __device__ inline int64_t chunks(int64_t B) { return (B + kChunk - 1) / kChunk; }

// ---- workspace: the sort's buffers, per-position scratch, per-chunk sums and CUB's scratch (last) ---------------------
struct Layout {
  size_t vals_in, perm, keys, e, q, sums1, tot1, sums2, tot2, partials, cub, total;
};
inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
inline Layout layout(int64_t B, size_t cub_bytes) {
  const size_t n = (size_t)(B < 1 ? 1 : B), G = (size_t)chunks(B < 1 ? 1 : B);
  Layout L;
  size_t o = 0;
  L.vals_in = o;  o = align256(o + n * 4);
  L.perm = o;     o = align256(o + n * 4);
  L.keys = o;     o = align256(o + n * 8);
  L.e = o;        o = align256(o + n * 4);
  L.q = o;        o = align256(o + n * 4);
  L.sums1 = o;    o = align256(o + G * sizeof(ChunkSum));
  L.tot1 = o;     o = align256(o + 2 * G * sizeof(Val));
  L.sums2 = o;    o = align256(o + G * sizeof(ChunkSum));
  L.tot2 = o;     o = align256(o + 2 * G * sizeof(Val));
  L.partials = o; o = align256(o + G * 4 * sizeof(float));
  L.cub = o;      o = align256(o + cub_bytes);
  L.total = o;
  return L;
}

__global__ void __launch_bounds__(256) iota_kernel(int32_t* __restrict__ v, int64_t B) {
  const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
  if (i < B) v[i] = (int32_t)i;
}

// ---- the chunk's segmented reduction -----------------------------------------------------------------------------------
struct Scratch {
  Val v[kChunk];
  int f[kChunk], h[kChunk], e[kChunk];
};

// v: this thread's element (the identity past the chunk's n positions); head: its position starts a session.  Returns
// the total of the thread's session: its piece's total when the session lies inside the chunk, else the carry's total
// (tot: [G] totals of the sessions of each chunk's first position, then [G] of each chunk's last position).  With `sum`
// (tot == nullptr), thread 0 writes the chunk's ChunkSum instead.
__device__ __forceinline__ Val session_total(Val v, bool head, int n, Scratch& sh, ChunkSum* sum, const Val* tot,
                                             int64_t G) {
  const int t = threadIdx.x;
  int f = (t == 0 || t >= n || head) ? 1 : 0;   // past the end: a piece of its own
  sh.v[t] = v;
  sh.f[t] = f;
  sh.h[t] = f;
  __syncthreads();
  for (int d = 1; d < kChunk; d <<= 1) {        // inclusive segmented scan, left to right
    Val o = v;
    int of = 1;
    if (t >= d) {
      o = sh.v[t - d];
      of = sh.f[t - d];
    }
    __syncthreads();
    if (t >= d && !f) {
      v = val_add(o, v);
      f = of;
    }
    sh.v[t] = v;
    sh.f[t] = f;
    __syncthreads();
  }
  int e = (t == kChunk - 1 || sh.h[t + 1]) ? t : kChunk;   // the last position of this thread's piece: suffix min
  sh.e[t] = e;
  __syncthreads();
  for (int d = 1; d < kChunk; d <<= 1) {
    const int o = (t + d < kChunk) ? sh.e[t + d] : kChunk;
    __syncthreads();
    e = o < e ? o : e;
    sh.e[t] = e;
    __syncthreads();
  }
  const int e0 = sh.e[0];
  Val r = sh.v[e];
  if (sum != nullptr && t == 0) {
    sum->first = sh.v[e0];
    sum->last = sh.v[n - 1];
    sum->single = (e0 == n - 1) ? 1 : 0;
  }
  if (tot != nullptr && t < n) {
    if (e == e0) r = tot[blockIdx.x];
    else if (e == n - 1) r = tot[G + blockIdx.x];
  }
  __syncthreads();
  return r;
}

__device__ __forceinline__ bool is_head(const int64_t* skey, int64_t p) { return p == 0 || skey[p] != skey[p - 1]; }

// pass 1: per session, (max, sum exp) of the negatives' l1 (a) and of the positives' l0 (b)
__global__ void __launch_bounds__(kChunk) pass1_kernel(const float* __restrict__ logits, int64_t ld,
                                                       const float* __restrict__ labels, const int32_t* __restrict__ perm,
                                                       const int64_t* __restrict__ skey, int64_t B,
                                                       ChunkSum* __restrict__ sums) {
  __shared__ Scratch sh;
  const int t = threadIdx.x;
  const int64_t p = (int64_t)blockIdx.x * kChunk + t;
  const int n = (int)((B - (int64_t)blockIdx.x * kChunk) < kChunk ? (B - (int64_t)blockIdx.x * kChunk) : kChunk);
  Val v = val_id();
  bool head = false;
  if (t < n) {
    const int64_t i = perm[p];
    const float y = labels[i];
    if (y == 0.f) v.a = Pair{logits[i * ld + 1], 1.f};
    else if (y == 1.f) v.b = Pair{logits[i * ld], 1.f};
    head = is_head(skey, p);
  }
  session_total(v, head, n, sh, sums + blockIdx.x, nullptr, 0);
}

__device__ __forceinline__ bool continues(const int64_t* skey, int64_t c) {   // chunk c's first session began earlier
  return c > 0 && skey[c * kChunk] == skey[c * kChunk - 1];
}

// one CTA: the totals of the sessions that touch a chunk boundary (tot[c]: of chunk c's first position, tot[G + c]: of
// its last), over tiles of kChunk chunks.
//   forward   acc_last[c] = acc_last[c - 1] + last[c] while chunk c is one piece that continues the previous chunk's
//             last session, else last[c]: a segmented scan over the chunks; acc_first[c] = acc_last[c - 1] + first[c]
//             when chunk c continues, else first[c]
//   backward  the last session of chunk c ends at chunk T(c) = the first j >= c whose last session does not run on
//             through chunk j + 1 as a whole (a suffix min); its total is acc_first[T + 1] when it ends inside chunk
//             T + 1, else acc_last[T]; a one-piece chunk's first session is its last
// Every chunk of a session reads the one stored total, so all its positions see the same bits.  With `loss`, also the
// loss from the [G][4] partials of pass 2 (sum of w L, positives, negatives, invalid labels): each thread adds its
// chunks g = t, t + kChunk, ... in order, then a fixed tree over the threads.
__global__ void __launch_bounds__(kChunk) carry_kernel(const ChunkSum* __restrict__ sums,
                                                       const int64_t* __restrict__ skey, int64_t G,
                                                       Val* __restrict__ tot, const float* __restrict__ partials,
                                                       int64_t B, int mean_mode, float* __restrict__ loss) {
  __shared__ Scratch sh;
  const int t = threadIdx.x;
  Val run = val_id();                           // acc_last of the chunk before the tile
  for (int64_t t0 = 0; t0 < G; t0 += kChunk) {
    const int64_t c = t0 + t;
    const bool in = c < G;
    const bool cont = in && continues(skey, c);
    Val v = in ? sums[c].last : val_id();
    int f = (!in || !(cont && sums[c].single)) ? 1 : 0;
    if (t == 0 && !f) {
      v = val_add(run, v);
      f = 1;
    }
    sh.v[t] = v;
    sh.f[t] = f;
    __syncthreads();
    for (int d = 1; d < kChunk; d <<= 1) {      // inclusive segmented scan, left to right
      Val o = v;
      int of = 1;
      if (t >= d) {
        o = sh.v[t - d];
        of = sh.f[t - d];
      }
      __syncthreads();
      if (t >= d && !f) {
        v = val_add(o, v);
        f = of;
      }
      sh.v[t] = v;
      sh.f[t] = f;
      __syncthreads();
    }
    if (in) {
      const Val prev = t > 0 ? sh.v[t - 1] : run;
      tot[c] = cont ? val_add(prev, sums[c].first) : sums[c].first;
      tot[G + c] = v;
    }
    run = sh.v[(G - t0 < kChunk ? G - t0 : kChunk) - 1];
    __syncthreads();
  }
  int64_t t_next = G;                           // T of the first chunk of the tile after this one
  for (int64_t t0 = G > 0 ? (G - 1) / kChunk * kChunk : -1; t0 >= 0; t0 -= kChunk) {
    const int64_t c = t0 + t;
    const bool in = c < G;
    const bool brk = in && !(c + 1 < G && continues(skey, c + 1) && sums[c + 1].single);
    int e = brk ? t : kChunk;
    sh.e[t] = e;
    __syncthreads();
    for (int d = 1; d < kChunk; d <<= 1) {      // suffix min of the chunks where a session ends
      const int o = (t + d < kChunk) ? sh.e[t + d] : kChunk;
      __syncthreads();
      e = o < e ? o : e;
      sh.e[t] = e;
      __syncthreads();
    }
    const int64_t T = e < kChunk ? t0 + e : t_next;
    Val tl = val_id(), tf = val_id();
    if (in) {
      tl = (T + 1 < G && continues(skey, T + 1)) ? tot[T + 1] : tot[G + T];
      tf = sums[c].single ? tl : tot[c];
    }
    t_next = sh.e[0] < kChunk ? t0 + sh.e[0] : t_next;
    __syncthreads();                            // every read of the tile's totals before its writes
    if (in) {
      tot[c] = tf;
      tot[G + c] = tl;
    }
    __syncthreads();
  }
  if (loss == nullptr) return;
  Val a = Val{Pair{0.f, 0.f}, Pair{0.f, 0.f}};
  for (int64_t g = t; g < G; g += kChunk) {
    a.a.m += partials[4 * g];
    a.a.s += partials[4 * g + 1];
    a.b.m += partials[4 * g + 2];
    a.b.s += partials[4 * g + 3];
  }
  sh.v[t] = a;
  __syncthreads();
  for (int s = kChunk / 2; s > 0; s >>= 1) {
    if (t < s) {
      Val x = sh.v[t];
      const Val y = sh.v[t + s];
      x.a.m += y.a.m;
      x.a.s += y.a.s;
      x.b.m += y.b.m;
      x.b.s += y.b.s;
      sh.v[t] = x;
    }
    __syncthreads();
  }
  if (t == 0) {
    const Val r = sh.v[0];
    float l = r.a.m / (float)B;
    if (B == 0 || r.b.s > 0.f || (mean_mode && (r.a.s == 0.f || r.b.m == 0.f))) l = NAN;
    *loss = l;
  }
}

// pass 2: per sample ce, ge, the loss term and the own-row gradient; e and q for pass 3; per session T1 (a) / T0 (b)
__global__ void __launch_bounds__(kChunk) pass2_kernel(const float* __restrict__ logits, int64_t ld,
                                                       const float* __restrict__ labels, const float* __restrict__ weights,
                                                       const int32_t* __restrict__ perm, const int64_t* __restrict__ skey,
                                                       int64_t B, float alpha, const Val* __restrict__ tot1,
                                                       float* __restrict__ e_out, float* __restrict__ q_out,
                                                       float* __restrict__ dlogits, ChunkSum* __restrict__ sums2,
                                                       float* __restrict__ partials) {
  __shared__ Scratch sh;
  const int t = threadIdx.x;
  const int64_t G = chunks(B);
  const int64_t p = (int64_t)blockIdx.x * kChunk + t;
  const int n = (int)((B - (int64_t)blockIdx.x * kChunk) < kChunk ? (B - (int64_t)blockIdx.x * kChunk) : kChunk);
  Val v = val_id();
  bool head = false;
  int64_t i = 0;
  float l0 = 0.f, l1 = 0.f, y = 0.f;
  if (t < n) {
    i = perm[p];
    y = labels[i];
    l0 = logits[i * ld];
    l1 = logits[i * ld + 1];
    if (y == 0.f) v.a = Pair{l1, 1.f};
    else if (y == 1.f) v.b = Pair{l0, 1.f};
    head = is_head(skey, p);
  }
  const Val st = session_total(v, head, n, sh, nullptr, tot1, G);
  Val v2 = val_id();
  float wl = 0.f, pos = 0.f, neg = 0.f, inv = 0.f;
  if (t < n) {
    const float w = weights ? weights[i] : 1.f;
    const float c = w / (float)B;
    const float mx = fmaxf(l0, l1);
    const float lse = mx + logf(expf(l0 - mx) + expf(l1 - mx));
    const float p0 = expf(l0 - lse), p1 = expf(l1 - lse);
    float d0, d1, L, e = 0.f, q = 0.f;
    if (y == 1.f || y == 0.f) {
      const bool P = y == 1.f;
      const float x = P ? l1 : l0;
      const Pair o = P ? st.a : st.b;           // the other class's pair of the session
      const float m = fmaxf(x, o.m);
      const float Z = expf(x - m) + o.s * expf(o.m - m);
      const float ge = m - x + logf(Z);
      const float self = expf(x - m) / Z - 1.f;
      q = c * expf(o.m - m) / Z;
      L = alpha * (lse - x) + (1.f - alpha) * ge;
      if (P) {
        d0 = c * alpha * p0;
        d1 = c * alpha * (p1 - 1.f) + c * (1.f - alpha) * self;
        e = expf(l0 - st.b.m);
        v2.a = Pair{0.f, q};
        v2.b = Pair{0.f, 0.f};
        pos = 1.f;
      } else {
        d0 = c * alpha * (p0 - 1.f) + c * (1.f - alpha) * self;
        d1 = c * alpha * p1;
        e = expf(l1 - st.a.m);
        v2.a = Pair{0.f, 0.f};
        v2.b = Pair{0.f, q};
        neg = 1.f;
      }
    } else {
      L = d0 = d1 = NAN;
      v2.a = v2.b = Pair{0.f, 0.f};
      inv = 1.f;
    }
    wl = w * L;
    dlogits[2 * i] = d0;
    dlogits[2 * i + 1] = d1;
    e_out[p] = e;
    q_out[p] = q;
  }
  session_total(v2, head, n, sh, sums2 + blockIdx.x, nullptr, 0);
  // the chunk's [sum w L, positives, negatives, invalid], a fixed tree over the threads
  sh.v[t] = Val{Pair{wl, pos}, Pair{neg, inv}};
  __syncthreads();
  for (int s = kChunk / 2; s > 0; s >>= 1) {
    if (t < s) {
      Val a = sh.v[t];
      const Val b = sh.v[t + s];
      a.a.m += b.a.m;
      a.a.s += b.a.s;
      a.b.m += b.b.m;
      a.b.s += b.b.s;
      sh.v[t] = a;
    }
    __syncthreads();
  }
  if (t == 0) {
    float* out = partials + 4 * (int64_t)blockIdx.x;
    out[0] = sh.v[0].a.m;
    out[1] = sh.v[0].a.s;
    out[2] = sh.v[0].b.m;
    out[3] = sh.v[0].b.s;
  }
}

// pass 3: the cross terms, from the session's T1 (a, for negatives) and T0 (b, for positives)
__global__ void __launch_bounds__(kChunk) pass3_kernel(const float* __restrict__ labels, const int32_t* __restrict__ perm,
                                                       const int64_t* __restrict__ skey, int64_t B, float alpha,
                                                       const Val* __restrict__ tot2, const float* __restrict__ e_in,
                                                       const float* __restrict__ q_in, float* __restrict__ dlogits) {
  __shared__ Scratch sh;
  const int t = threadIdx.x;
  const int64_t G = chunks(B);
  const int64_t p = (int64_t)blockIdx.x * kChunk + t;
  const int n = (int)((B - (int64_t)blockIdx.x * kChunk) < kChunk ? (B - (int64_t)blockIdx.x * kChunk) : kChunk);
  Val v = val_id();
  bool head = false;
  int64_t i = 0;
  float y = -1.f;
  if (t < n) {
    i = perm[p];
    y = labels[i];
    const float q = q_in[p];
    v.a = Pair{0.f, y == 1.f ? q : 0.f};
    v.b = Pair{0.f, y == 0.f ? q : 0.f};
    head = is_head(skey, p);
  }
  const Val st = session_total(v, head, n, sh, nullptr, tot2, G);
  if (t < n) {
    if (y == 1.f) dlogits[2 * i] += (1.f - alpha) * e_in[p] * st.b.s;
    else if (y == 0.f) dlogits[2 * i + 1] += (1.f - alpha) * e_in[p] * st.a.s;
  }
}

// the passes over samples already sorted by session (perm and the sorted keys at L.perm / L.keys of ws).  weights:
// nullptr for the mean reduction.  dlogits: [B, 2] contiguous.
inline void run_sorted(const float* logits, int64_t ld, const float* labels, const float* weights, int64_t B,
                       float alpha, float* loss, float* dlogits, unsigned char* ws, const Layout& L,
                       cudaStream_t stream) {
  const int64_t G = chunks(B);
  const int32_t* perm = reinterpret_cast<const int32_t*>(ws + L.perm);
  const int64_t* skey = reinterpret_cast<const int64_t*>(ws + L.keys);
  float* e = reinterpret_cast<float*>(ws + L.e);
  float* q = reinterpret_cast<float*>(ws + L.q);
  ChunkSum* sums1 = reinterpret_cast<ChunkSum*>(ws + L.sums1);
  ChunkSum* sums2 = reinterpret_cast<ChunkSum*>(ws + L.sums2);
  Val* tot1 = reinterpret_cast<Val*>(ws + L.tot1);
  Val* tot2 = reinterpret_cast<Val*>(ws + L.tot2);
  float* partials = reinterpret_cast<float*>(ws + L.partials);
  if (G > 0) {
    TZK_LAUNCH((pass1_kernel), (unsigned)G, kChunk, 0, stream, logits, ld, labels, perm, skey, B, sums1);
    TZK_LAUNCH((carry_kernel), 1, kChunk, 0, stream, sums1, skey, G, tot1, nullptr, B, 0, nullptr);
    TZK_LAUNCH((pass2_kernel), (unsigned)G, kChunk, 0, stream, logits, ld, labels, weights, perm, skey, B, alpha, tot1,
               e, q, dlogits, sums2, partials);
  }
  TZK_LAUNCH((carry_kernel), 1, kChunk, 0, stream, sums2, skey, G, tot2, partials, B, weights == nullptr ? 1 : 0, loss);
  if (G > 0)
    TZK_LAUNCH((pass3_kernel), (unsigned)G, kChunk, 0, stream, labels, perm, skey, B, alpha, tot2, e, q, dlogits);
}
}  // namespace tzk_jrc
