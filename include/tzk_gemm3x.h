/* tzk_gemm3x.h — C-ABI of libtzk_gemm3x.so (torcheasyrec_b200/csrc/tzk_gemm3x.cu): the one wide tower layer of the
 * rank models (tzrec/modules/mlp.py:20-84 Perceptron; DLRM's final MLP input, tzrec/models/dlrm.py:113-131, 783 wide,
 * travelling as [B, 784]) on hand-written sm_90a tensor-core kernels: mma.sync m16n8k8 TF32 with the 3xTF32 split
 * (fp32-level accuracy), TMA-fed through mbarrier-guarded shared-memory stages.  Replaces the three library GEMMs of
 * that layer (forward, input gradient, weight gradient).  Plain pointers and sizes; caller-owned memory and stream;
 * returns 0 or 1 bad argument / 2 tensor-map encoding failed / 3 launch failure.  Rows must be 16-B aligned
 * (ld % 4 == 0).
 *
 *   tzk_gemm3x   y[M,N] = act(x[M,K] @ w[N,K]^T + bias)   N = 64 (forward, K = 784; bias / relu optional) or a
 *                multiple of 112 (input gradient: x = dZ [M,64], w = W^T [784,64]).  K columns beyond the tensor read
 *                as zeros up to the next multiple of 32.  w_hi / w_lo: [N, ld_w] scratch (the TF32 split of w).
 *   tzk_wgrad3x  dw[64,K] = dz[M,64]^T @ x[M,K], reduction over the batch split into `slabs` row slabs whose partial
 *                results (scratch `partial`, tzk_wgrad3x_partial_floats(K, slabs) floats) are added in a fixed order:
 *                bit-repeatable.
 * Accuracy note: the tensor core's fp32 accumulation is not round-to-nearest; the kernels accumulate every k-step
 * (8 columns of K) in fresh registers and add them in round-to-nearest (see the comment at the top of the source). */
#ifndef TZK_GEMM3X_H_
#define TZK_GEMM3X_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
int tzk_gemm3x(const float* x, int64_t ld_x, const float* w, int64_t ld_w, const float* bias, int64_t M, int32_t N,
               int32_t K, int32_t relu, float* y, int64_t ld_y, float* w_hi, float* w_lo, void* stream);
int64_t tzk_wgrad3x_partial_floats(int32_t K, int32_t slabs);
int tzk_wgrad3x(const float* x, int64_t ld_x, const float* dz, int64_t ld_dz, int64_t M, int32_t K, int32_t slabs,
                float* partial, float* dw, int64_t ld_dw, void* stream);
#ifdef __cplusplus
}
#endif
#endif /* TZK_GEMM3X_H_ */
