// tzk_interact_bf16.cu — C entry points of the BF16 DLRM-Criteo interaction (tzk_interact_bf16.cuh).  A translation unit
// of its own, so the fp32 kernels of tzk_dense.cu are compiled exactly as before.
#include <cuda_bf16.h>

#include "tzk_common.cuh"

using namespace tzk;

#include "tzk_launch.cuh"
namespace tzk_ib16 {
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);       // .x (low half) = lo
  return *reinterpret_cast<const uint32_t*>(&v);
}
__device__ __forceinline__ uint16_t bf16_rn(float x) { return __bfloat16_as_ushort(__float2bfloat16_rn(x)); }
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
}  // namespace tzk_ib16
#include "tzk_interact_bf16.cuh"

namespace {
int bf16_check(const char* who, const void* dense, int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t B,
               const void* x, int64_t ld_x) {
  TZK_REQUIRE(B >= 0, "%s: negative batch size", who);
  TZK_REQUIRE(dense && sparse && x, "%s: NULL argument", who);
  TZK_REQUIRE((uintptr_t)dense % 8 == 0 && ld_dense % 4 == 0 && ld_dense >= tzk_ib16::kD,
              "%s: dense must be [B, 16] bf16 with 8-B aligned rows", who);
  TZK_REQUIRE((uintptr_t)sparse % 16 == 0 && ld_sparse % 4 == 0 && ld_sparse >= (tzk_ib16::kN - 1) * tzk_ib16::kD,
              "%s: sparse must be [B, 416] fp32 with 16-B aligned rows", who);
  TZK_REQUIRE((uintptr_t)x % 16 == 0 && ld_x % 8 == 0 && ld_x >= tzk_ib16::kRow,
              "%s: the interaction row must be [B, 784] bf16 with 16-B aligned rows", who);
  return 0;
}
}  // namespace

extern "C" int tzk_dot_interact27_fwd_bf16(const uint16_t* dense, int64_t ld_dense, const float* sparse,
                                           int64_t ld_sparse, int64_t B, uint16_t* out, int64_t ld_out,
                                           tzk_stream_t stream) {
  int rc = bf16_check("dot_interact27_fwd_bf16", dense, ld_dense, sparse, ld_sparse, B, out, ld_out);
  if (rc) return rc;
  if (B == 0) return 0;
  tzk_ib16::dot_interact27_fwd_bf16_kernel<<<tzk_ib16::grid_for(B, kSmCountH100 * 8), tzk_ib16::kWarps * 32,
                                             tzk_ib16::fwd_smem(), as_stream(stream)>>>(dense, ld_dense, sparse,
                                                                                        ld_sparse, B, out, ld_out);
  TZK_CHECK_LAUNCH("dot_interact27_fwd_bf16_kernel");
  return 0;
}

extern "C" int tzk_dot_interact27_bwd_bf16(const uint16_t* d_out, int64_t ld_dout, const uint16_t* dense,
                                           int64_t ld_dense, const float* sparse, int64_t ld_sparse, int64_t B,
                                           uint16_t* d_dense, int64_t ld_ddense, float* d_sparse, int64_t ld_dsparse,
                                           tzk_stream_t stream) {
  int rc = bf16_check("dot_interact27_bwd_bf16", dense, ld_dense, sparse, ld_sparse, B, d_out, ld_dout);
  if (rc) return rc;
  TZK_REQUIRE(d_dense && d_sparse, "dot_interact27_bwd_bf16: NULL gradient output");
  TZK_REQUIRE((uintptr_t)d_dense % 8 == 0 && ld_ddense % 4 == 0 && ld_ddense >= tzk_ib16::kD,
              "dot_interact27_bwd_bf16: d_dense must be [B, 16] bf16 with 8-B aligned rows");
  TZK_REQUIRE((uintptr_t)d_sparse % 16 == 0 && ld_dsparse % 4 == 0 && ld_dsparse >= (tzk_ib16::kN - 1) * tzk_ib16::kD,
              "dot_interact27_bwd_bf16: d_sparse must be [B, 416] fp32 with 16-B aligned rows");
  if (B == 0) return 0;
  tzk_ib16::dot_interact27_bwd_bf16_kernel<<<tzk_ib16::grid_for(B, kSmCountH100 * 8), tzk_ib16::kWarps * 32,
                                             tzk_ib16::bwd_smem(), as_stream(stream)>>>(
      dense, ld_dense, sparse, ld_sparse, d_out, ld_dout, B, d_dense, ld_ddense, d_sparse, ld_dsparse);
  TZK_CHECK_LAUNCH("dot_interact27_bwd_bf16_kernel");
  return 0;
}
