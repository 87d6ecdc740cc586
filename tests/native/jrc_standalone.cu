// jrc_standalone.cu — host build of torcheasyrec_b200/csrc/tzk_jrc.cuh (tests/test_dbmtl_cpu.py).  std::stable_sort
// stands in for the radix sort of tzk_jrc.cu (both order by session id and keep the sample order inside a session).
#ifndef TZK_CPU_SHIM
#error "host-only test build"
#endif
#include "cuda_cpu_shim.h"
#include <math.h>
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "../../torcheasyrec_b200/csrc/tzk_jrc.cuh"

extern "C" int jrc_loss(const float* logits, int64_t ld, const float* labels, const int64_t* session_ids,
                        const float* weights, int64_t B, float alpha, float* loss, float* dlogits) {
  const tzk_jrc::Layout L = tzk_jrc::layout(B, 0);
  std::vector<unsigned char> ws(L.total);
  int32_t* perm = reinterpret_cast<int32_t*>(ws.data() + L.perm);
  int64_t* keys = reinterpret_cast<int64_t*>(ws.data() + L.keys);
  for (int64_t i = 0; i < B; ++i) perm[i] = (int32_t)i;
  std::stable_sort(perm, perm + B, [&](int32_t a, int32_t b) { return session_ids[a] < session_ids[b]; });
  for (int64_t i = 0; i < B; ++i) keys[i] = session_ids[perm[i]];
  tzk_jrc::run_sorted(logits, ld, labels, weights, B, alpha, loss, dlogits, ws.data(), L, nullptr);
  return 0;
}
