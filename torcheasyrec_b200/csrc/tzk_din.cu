// tzk_din.cu — DIN target attention over JAGGED sequence rows (SURVEY §8f N3).
//
// The reference pads the looked-up sequence rows to [B, T, Ds] with T = the longest sequence of the batch (a
// device->host sync: tzrec/modules/embedding.py:1468), broadcasts the query over T and runs the attention MLP over all
// B*T positions, padding included (tzrec/modules/sequence.py:65-128).  Here the rows stay where the un-pooled gather
// put them — [N, Ds], N = sum of the sequence lengths, sample b owns rows offsets[b] .. offsets[b+1] — and only these
// two steps around the (dense, library) attention MLP are kernels:
//   din_attn_input   : row n of sample b -> [q_b | k_n | q_b - k_n | q_b * k_n]  (the MLP's input, [N, 4*Ds]);
//                      backward: d_k and the per-sample sum d_q, rows visited in order (deterministic)
//   jagged_softmax_wsum : p = softmax over the sample's first min(len, max_len) scores, out_b = sum_n p_n k_n;
//                      a sample without rows gives zeros — what the reference's masked softmax over an all-padding
//                      row times zero rows gives; backward: d_score, d_k
// No padded tensor, no host read of the longest length; work and bytes scale with N instead of B*T.
// One warp per sample, lanes over the columns, rows in order: HBM-bound streaming, no atomics.
#include "tzk_common.cuh"

using namespace tzk;

namespace {
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int d = 16; d >= 1; d >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, d));
  return v;
}

__global__ void __launch_bounds__(kThreads)
din_attn_input_fwd_kernel(const float* __restrict__ query, int64_t ld_q, int Dq, const float* __restrict__ seq,
                          const int64_t* __restrict__ offsets, int B, int Ds, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int b = blockIdx.x * kWarps + (threadIdx.x >> 5); b < B; b += gridDim.x * kWarps) {
    const int64_t s = __ldg(offsets + b), e = __ldg(offsets + b + 1);
    for (int c = lane; c < Ds; c += 32) {
      const float q = c < Dq ? __ldg(query + (int64_t)b * ld_q + c) : 0.f;     // the query is zero-padded to Ds
      for (int64_t n = s; n < e; ++n) {
        const float k = __ldg(seq + n * Ds + c);
        float* o = out + n * 4 * Ds + c;
        o[0] = q;
        o[Ds] = k;
        o[2 * Ds] = q - k;
        o[3 * Ds] = q * k;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads)
din_attn_input_bwd_kernel(const float* __restrict__ d_in, const float* __restrict__ query, int64_t ld_q, int Dq,
                          const float* __restrict__ seq, const int64_t* __restrict__ offsets, int B, int Ds,
                          float* __restrict__ d_query, float* __restrict__ d_seq) {
  const int lane = threadIdx.x & 31;
  for (int b = blockIdx.x * kWarps + (threadIdx.x >> 5); b < B; b += gridDim.x * kWarps) {
    const int64_t s = __ldg(offsets + b), e = __ldg(offsets + b + 1);
    for (int c = lane; c < Ds; c += 32) {
      const float q = c < Dq ? __ldg(query + (int64_t)b * ld_q + c) : 0.f;
      float dq = 0.f;
      for (int64_t n = s; n < e; ++n) {
        const float* g = d_in + n * 4 * Ds + c;
        const float g1 = __ldg(g), g2 = __ldg(g + Ds), g3 = __ldg(g + 2 * Ds), g4 = __ldg(g + 3 * Ds);
        const float k = __ldg(seq + n * Ds + c);
        dq += g1 + g3 + g4 * k;
        d_seq[n * Ds + c] = g2 - g3 + g4 * q;
      }
      if (c < Dq) d_query[(int64_t)b * Dq + c] = dq;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
jagged_softmax_wsum_fwd_kernel(const float* __restrict__ scores, const float* __restrict__ seq,
                               const int64_t* __restrict__ offsets, int B, int Ds, int max_len,
                               float* __restrict__ probs, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int b = blockIdx.x * kWarps + (threadIdx.x >> 5); b < B; b += gridDim.x * kWarps) {
    const int64_t s = __ldg(offsets + b), e_all = __ldg(offsets + b + 1);
    const int64_t e = (max_len > 0 && e_all - s > max_len) ? s + max_len : e_all;
    float m = -INFINITY;
    for (int64_t n = s + lane; n < e; n += 32) m = fmaxf(m, __ldg(scores + n));
    m = warp_max(m);
    float z = 0.f;
    for (int64_t n = s + lane; n < e; n += 32) z += expf(__ldg(scores + n) - m);
    z = warp_sum(z);
    const float inv = e > s ? 1.f / z : 0.f;
    for (int64_t n = s + lane; n < e_all; n += 32) probs[n] = n < e ? expf(__ldg(scores + n) - m) * inv : 0.f;
    __syncwarp();
    for (int c = lane; c < Ds; c += 32) {
      float acc = 0.f;
      for (int64_t n = s; n < e; ++n) acc += probs[n] * __ldg(seq + n * Ds + c);
      out[(int64_t)b * Ds + c] = acc;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
jagged_softmax_wsum_bwd_kernel(const float* __restrict__ d_out, const float* __restrict__ probs,
                               const float* __restrict__ seq, const int64_t* __restrict__ offsets, int B, int Ds,
                               int max_len, float* __restrict__ d_scores, float* __restrict__ d_seq) {
  const int lane = threadIdx.x & 31;
  for (int b = blockIdx.x * kWarps + (threadIdx.x >> 5); b < B; b += gridDim.x * kWarps) {
    const int64_t s = __ldg(offsets + b), e_all = __ldg(offsets + b + 1);
    const int64_t e = (max_len > 0 && e_all - s > max_len) ? s + max_len : e_all;
    // d_p[n] = <d_out_b, k_n>  (kept in d_scores until the second pass); t = sum_n p_n d_p[n]
    float t = 0.f;
    for (int64_t n = s; n < e; ++n) {
      float dot = 0.f;
      for (int c = lane; c < Ds; c += 32) dot += __ldg(d_out + (int64_t)b * Ds + c) * __ldg(seq + n * Ds + c);
      dot = warp_sum(dot);
      const float p = __ldg(probs + n);
      t += p * dot;
      if (lane == 0) d_scores[n] = dot;
    }
    __syncwarp();
    for (int64_t n = s + lane; n < e_all; n += 32) d_scores[n] = n < e ? __ldg(probs + n) * (d_scores[n] - t) : 0.f;
    for (int c = lane; c < Ds; c += 32) {
      const float g = __ldg(d_out + (int64_t)b * Ds + c);
      for (int64_t n = s; n < e_all; ++n) d_seq[n * Ds + c] = n < e ? __ldg(probs + n) * g : 0.f;
    }
  }
}

inline int grid_for(int B) {
  const int64_t ctas = ceil_div64(B, kWarps);
  return (int)(ctas < kSmCountH100 * 8 ? (ctas > 0 ? ctas : 1) : kSmCountH100 * 8);
}
}  // namespace

extern "C" int tzk_din_attn_input_fwd(const float* query, int64_t ld_q, int32_t Dq, const float* seq,
                                      const int64_t* offsets, int32_t B, int32_t Ds, int64_t N, float* out,
                                      tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && Ds >= 1 && Dq >= 0 && Dq <= Ds && N >= 0, "din_attn_input_fwd: bad sizes");
  if (B == 0 || N == 0) return 0;
  TZK_REQUIRE(query && seq && offsets && out, "din_attn_input_fwd: NULL argument");
  din_attn_input_fwd_kernel<<<grid_for(B), kThreads, 0, as_stream(stream)>>>(query, ld_q, Dq, seq, offsets, B, Ds, out);
  TZK_CHECK_LAUNCH("din_attn_input_fwd_kernel");
  return 0;
}

extern "C" int tzk_din_attn_input_bwd(const float* d_in, const float* query, int64_t ld_q, int32_t Dq, const float* seq,
                                      const int64_t* offsets, int32_t B, int32_t Ds, int64_t N, float* d_query,
                                      float* d_seq, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && Ds >= 1 && Dq >= 0 && Dq <= Ds && N >= 0, "din_attn_input_bwd: bad sizes");
  if (B == 0) return 0;
  TZK_REQUIRE(query && offsets && d_query && (N == 0 || (d_in && seq && d_seq)), "din_attn_input_bwd: NULL argument");
  din_attn_input_bwd_kernel<<<grid_for(B), kThreads, 0, as_stream(stream)>>>(d_in, query, ld_q, Dq, seq, offsets, B, Ds,
                                                                              d_query, d_seq);
  TZK_CHECK_LAUNCH("din_attn_input_bwd_kernel");
  return 0;
}

extern "C" int tzk_jagged_softmax_wsum_fwd(const float* scores, const float* seq, const int64_t* offsets, int32_t B,
                                           int32_t Ds, int32_t max_len, int64_t N, float* probs, float* out,
                                           tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && Ds >= 1 && N >= 0, "jagged_softmax_wsum_fwd: bad sizes");
  if (B == 0) return 0;
  TZK_REQUIRE(offsets && out && (N == 0 || (scores && seq && probs)), "jagged_softmax_wsum_fwd: NULL argument");
  jagged_softmax_wsum_fwd_kernel<<<grid_for(B), kThreads, 0, as_stream(stream)>>>(scores, seq, offsets, B, Ds, max_len,
                                                                                   probs, out);
  TZK_CHECK_LAUNCH("jagged_softmax_wsum_fwd_kernel");
  return 0;
}

extern "C" int tzk_jagged_softmax_wsum_bwd(const float* d_out, const float* probs, const float* seq,
                                           const int64_t* offsets, int32_t B, int32_t Ds, int32_t max_len, int64_t N,
                                           float* d_scores, float* d_seq, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && Ds >= 1 && N >= 0, "jagged_softmax_wsum_bwd: bad sizes");
  if (B == 0 || N == 0) return 0;
  TZK_REQUIRE(d_out && probs && seq && offsets && d_scores && d_seq, "jagged_softmax_wsum_bwd: NULL argument");
  jagged_softmax_wsum_bwd_kernel<<<grid_for(B), kThreads, 0, as_stream(stream)>>>(d_out, probs, seq, offsets, B, Ds,
                                                                                   max_len, d_scores, d_seq);
  TZK_CHECK_LAUNCH("jagged_softmax_wsum_bwd_kernel");
  return 0;
}
