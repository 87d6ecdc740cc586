// tzk_metrics.cu — C entry point of the evaluation metrics' device update (tzk_metrics.cuh).  A translation unit of its
// own, so no kernel of the training step is recompiled by it.
#include "tzk_common.cuh"

#define TZK_DYN_SMEM(type, name) extern __shared__ __align__(16) type name[]
#define TZK_UNPAREN(...) __VA_ARGS__
#define TZK_LAUNCH(kernel, grid, block, smem, stream, ...) TZK_UNPAREN kernel<<<grid, block, smem, stream>>>(__VA_ARGS__)
#include "tzk_metrics.cuh"

using namespace tzk;

extern "C" int tzk_binned_auc_update(const void* preds, int32_t pred_dtype, const void* labels, int32_t label_dtype,
                                     int64_t n, const float* thresholds, int32_t T, int64_t* counts, int64_t* invalid,
                                     tzk_stream_t stream) {
  TZK_REQUIRE(n >= 0, "binned_auc_update: negative sample count");
  TZK_REQUIRE(T >= 1, "binned_auc_update: need at least one threshold");
  TZK_REQUIRE(pred_dtype == 0 || pred_dtype == 1, "binned_auc_update: predictions must be fp32 (0) or bf16 (1)");
  TZK_REQUIRE(label_dtype == 0 || label_dtype == 1, "binned_auc_update: labels must be fp32 (0) or int64 (1)");
  TZK_REQUIRE(thresholds && counts && invalid, "binned_auc_update: NULL thresholds / counts / invalid counter");
  TZK_REQUIRE(n == 0 || (preds && labels), "binned_auc_update: NULL predictions or labels");
  const int rc = tzk_auc::run(preds, pred_dtype, labels, label_dtype, n, thresholds, T, counts, invalid,
                              as_stream(stream));
  if (rc == 3) {
    set_error("binned_auc_kernel: launch failed");
    return 2;
  }
  TZK_REQUIRE(rc == 0, "binned_auc_update: bad argument");
  return 0;
}
