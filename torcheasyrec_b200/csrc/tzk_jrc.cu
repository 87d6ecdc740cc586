// tzk_jrc.cu — C entry points of the JRC loss (tzk_jrc.cuh): the radix sort by session, then the header's passes.  A
// translation unit of its own, so no existing kernel is recompiled by it.
#include <cub/cub.cuh>

#include "tzk_common.cuh"

#include "tzk_jrc.cuh"

using namespace tzk;

namespace {
size_t cub_sort_bytes(int64_t B) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const int64_t*)nullptr, (int64_t*)nullptr, (const int32_t*)nullptr,
                                  (int32_t*)nullptr, (int)(B < 1 ? 1 : B), 0, 64);
  return bytes;
}
}  // namespace

extern "C" size_t tzk_jrc_loss_workspace_bytes(int64_t B) {
  if (B < 0 || B >= ((int64_t)1 << 31)) return 0;
  return tzk_jrc::layout(B, cub_sort_bytes(B)).total;
}

extern "C" int tzk_jrc_loss(const float* logits, int64_t ld, const float* labels, const int64_t* session_ids,
                            const float* weights, int64_t B, float alpha, int32_t key_bits, float* loss,
                            float* dlogits, void* workspace, size_t workspace_bytes, tzk_stream_t stream) {
  TZK_REQUIRE(B >= 0 && B < ((int64_t)1 << 31), "jrc_loss: need 0 <= B < 2^31");
  TZK_REQUIRE(key_bits >= 1 && key_bits <= 64, "jrc_loss: need 1 <= key_bits <= 64");
  TZK_REQUIRE(loss != nullptr, "jrc_loss: NULL loss");
  TZK_REQUIRE(B == 0 || (logits && labels && session_ids && dlogits && ld >= 2), "jrc_loss: NULL argument or ld < 2");
  const size_t cub_bytes = cub_sort_bytes(B);
  const tzk_jrc::Layout L = tzk_jrc::layout(B, cub_bytes);
  TZK_REQUIRE(workspace != nullptr && workspace_bytes >= L.total, "jrc_loss: workspace too small");
  cudaStream_t st = as_stream(stream);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  if (B > 0) {
    int32_t* vals_in = reinterpret_cast<int32_t*>(ws + L.vals_in);
    tzk_jrc::iota_kernel<<<(unsigned)((B + 255) / 256), 256, 0, st>>>(vals_in, B);
    TZK_CHECK_LAUNCH("jrc iota_kernel");
    size_t tmp = cub_bytes;
    const cudaError_t e = cub::DeviceRadixSort::SortPairs(
        ws + L.cub, tmp, session_ids, reinterpret_cast<int64_t*>(ws + L.keys), vals_in,
        reinterpret_cast<int32_t*>(ws + L.perm), (int)B, 0, key_bits, st);
    TZK_REQUIRE(e == cudaSuccess, "jrc_loss: session sort failed: %s", cudaGetErrorString(e));
  }
  tzk_jrc::run_sorted(logits, ld, labels, weights, B, alpha, loss, dlogits, ws, L, st);
  TZK_CHECK_LAUNCH("jrc pass kernels");
  return 0;
}
