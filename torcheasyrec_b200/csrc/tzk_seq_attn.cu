// tzk_seq_attn.cu — C entry points of the fused sequence encoders over jagged rows (tzk_seq_attn.cuh).  A translation
// unit of its own, so no existing kernel is recompiled by it.
#include "tzk_common.cuh"

#include "tzk_seq_attn.cuh"

using namespace tzk;

#define SEQ_ATTN_COVER "description outside the kernels' cover (H >= 1, 1 <= hd <= 128, row strides >= H hd)"

extern "C" int64_t tzk_seq_attn_smem_bytes(const tzk_seq_attn_args* args_host) {
  if (args_host == nullptr) return 0;
  tzk_seq_attn_args a = *args_host;
  a.B = 0;                          // the shapes alone
  if (tzk_seq_attn::check(a, false) != 0) return 0;
  return (int64_t)tzk_seq_attn::smem_bytes(a);
}

extern "C" int tzk_self_attn_pool_fwd(const tzk_seq_attn_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_seq_attn::check(*args_host, false) == 0, "self_attn_pool_fwd: " SEQ_ATTN_COVER);
  TZK_REQUIRE(grid >= 1, "self_attn_pool_fwd: need grid >= 1");
  tzk_seq_attn::fwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("self_attn_pool_fwd_kernel");
  return 0;
}

extern "C" int tzk_self_attn_pool_bwd(const tzk_seq_attn_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_seq_attn::check(*args_host, true) == 0, "self_attn_pool_bwd: " SEQ_ATTN_COVER);
  TZK_REQUIRE(grid >= 1, "self_attn_pool_bwd: need grid >= 1");
  tzk_seq_attn::bwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("self_attn_pool_bwd_kernel");
  return 0;
}

extern "C" int tzk_jagged_pool_fwd(const tzk_jagged_pool_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_seq_attn::check_pool(*args_host, false) == 0,
              "jagged_pool_fwd: need D >= 1, max_len >= 0, mean 0 or 1 and the buffers");
  TZK_REQUIRE(grid >= 1, "jagged_pool_fwd: need grid >= 1");
  tzk_seq_attn::pool_fwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("jagged_pool_fwd_kernel");
  return 0;
}

extern "C" int tzk_jagged_pool_bwd(const tzk_jagged_pool_args* args_host, int32_t grid, tzk_stream_t stream) {
  TZK_REQUIRE(args_host != nullptr && tzk_seq_attn::check_pool(*args_host, true) == 0,
              "jagged_pool_bwd: need D >= 1, max_len >= 0, mean 0 or 1 and the buffers");
  TZK_REQUIRE(grid >= 1, "jagged_pool_bwd: need grid >= 1");
  tzk_seq_attn::pool_bwd(*args_host, grid, as_stream(stream));
  TZK_CHECK_LAUNCH("jagged_pool_bwd_kernel");
  return 0;
}
