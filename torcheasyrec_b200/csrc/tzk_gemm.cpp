// tzk_gemm.cpp — fp32-accurate tensor-core GEMMs for the dense towers (library GEMM, not a hot-path row).
//
// The reference runs its MLP towers as plain fp32 cuBLAS GEMMs with TF32 off (train.proto field 14), i.e. on the
// CUDA cores.  cuBLASLt 12.9 can run the same fp32 GEMM on the tensor cores of GPUs that support the BF16x9 split
// (CUBLAS_COMPUTE_32F_EMULATED_16BFX9: every fp32 operand is split into three bf16 values, nine products,
// fp32-equivalent accuracy); where it offers no algorithm for that compute type the plain fp32 GEMM runs.  PyTorch 2.11+cu128 bundles cuBLAS 12.8, which lacks it, so this file loads the
// toolkit's own libcublasLt.so.12.9 by absolute path (dlopen, RTLD_LOCAL — it coexists with torch's copy) and
// exposes one row-major GEMM entry point.  If the library or the emulated algorithm is unavailable the caller
// keeps using torch's GEMM; nothing here is required for correctness.
#include <cublasLt.h>
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <mutex>
#include <tuple>

namespace {
char g_err[512] = "";
void set_err(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

struct Api {
  void* dl = nullptr;
  cublasLtHandle_t handle = nullptr;
  decltype(&cublasLtCreate) create;
  decltype(&cublasLtGetVersion) version;
  decltype(&cublasLtMatmulDescCreate) desc_create;
  decltype(&cublasLtMatmulDescDestroy) desc_destroy;
  decltype(&cublasLtMatmulDescSetAttribute) desc_set;
  decltype(&cublasLtMatrixLayoutCreate) layout_create;
  decltype(&cublasLtMatrixLayoutDestroy) layout_destroy;
  decltype(&cublasLtMatrixLayoutSetAttribute) layout_set;
  decltype(&cublasLtMatmulPreferenceCreate) pref_create;
  decltype(&cublasLtMatmulPreferenceDestroy) pref_destroy;
  decltype(&cublasLtMatmulPreferenceSetAttribute) pref_set;
  decltype(&cublasLtMatmulAlgoGetHeuristic) heuristic;
  decltype(&cublasLtMatmul) matmul;
} api;

struct Plan {
  cublasLtMatmulDesc_t op = nullptr;
  cublasLtMatrixLayout_t a = nullptr, b = nullptr, c = nullptr;
  cublasLtMatmulAlgo_t algo;
  size_t ws = 0;
  int emulated = 0;
};
using Key = std::tuple<int, int, int, int, int, int, int, int, int>;
std::map<Key, Plan> g_plans;
std::mutex g_mu;

template <typename T>
bool sym(T& fn, const char* name) {
  fn = reinterpret_cast<T>(dlsym(api.dl, name));
  if (!fn) set_err("tzg: missing symbol %s", name);
  return fn != nullptr;
}

bool make_layout(cublasLtMatrixLayout_t* l, int rows, int cols, int ld) {
  if (api.layout_create(l, CUDA_R_32F, rows, cols, ld) != CUBLAS_STATUS_SUCCESS) return false;
  cublasLtOrder_t order = CUBLASLT_ORDER_ROW;
  return api.layout_set(*l, CUBLASLT_MATRIX_LAYOUT_ORDER, &order, sizeof(order)) == CUBLAS_STATUS_SUCCESS;
}
}  // namespace

extern "C" const char* tzg_last_error(void) { return g_err; }

// returns the cuBLASLt version (e.g. 120901) or 0 on failure
extern "C" long tzg_init(const char* path) {
  std::lock_guard<std::mutex> lock(g_mu);
  if (api.handle) return (long)api.version();
  api.dl = dlopen(path, RTLD_NOW | RTLD_LOCAL);
  if (!api.dl) {
    set_err("tzg: dlopen(%s) failed: %s", path, dlerror());
    return 0;
  }
  bool ok = sym(api.create, "cublasLtCreate") && sym(api.version, "cublasLtGetVersion") &&
            sym(api.desc_create, "cublasLtMatmulDescCreate") && sym(api.desc_destroy, "cublasLtMatmulDescDestroy") &&
            sym(api.desc_set, "cublasLtMatmulDescSetAttribute") &&
            sym(api.layout_create, "cublasLtMatrixLayoutCreate") &&
            sym(api.layout_destroy, "cublasLtMatrixLayoutDestroy") &&
            sym(api.layout_set, "cublasLtMatrixLayoutSetAttribute") &&
            sym(api.pref_create, "cublasLtMatmulPreferenceCreate") &&
            sym(api.pref_destroy, "cublasLtMatmulPreferenceDestroy") &&
            sym(api.pref_set, "cublasLtMatmulPreferenceSetAttribute") &&
            sym(api.heuristic, "cublasLtMatmulAlgoGetHeuristic") && sym(api.matmul, "cublasLtMatmul");
  if (!ok) return 0;
  if (api.create(&api.handle) != CUBLAS_STATUS_SUCCESS) {
    set_err("tzg: cublasLtCreate failed");
    api.handle = nullptr;
    return 0;
  }
  return (long)api.version();
}

// Row-major: C[M,N] = alpha * op(A) * op(B) + beta * C ; op(A) is [M,K] (A stored [K,M] if transA), op(B) is [K,N]
// (B stored [N,K] if transB).  emulate != 0 asks for BF16x9; falls back to plain fp32 if no algorithm exists.
// Returns 0 on success; *used_emulation (nullable) reports which path ran.
extern "C" int tzg_matmul(int transA, int transB, int M, int N, int K, const float* A, int lda, const float* B,
                          int ldb, float* C, int ldc, float alpha, float beta, int emulate, void* workspace,
                          size_t workspace_bytes, void* stream, int* used_emulation) {
  if (!api.handle) {
    set_err("tzg: not initialised");
    return 1;
  }
  Plan plan;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    Key key{transA, transB, M, N, K, lda, ldb, ldc, emulate};
    auto it = g_plans.find(key);
    if (it == g_plans.end()) {
      Plan p;
      bool found = false;
      for (int attempt = emulate ? 0 : 1; attempt < 2 && !found; ++attempt) {
        const cublasComputeType_t ct = attempt == 0 ? CUBLAS_COMPUTE_32F_EMULATED_16BFX9 : CUBLAS_COMPUTE_32F;
        if (api.desc_create(&p.op, ct, CUDA_R_32F) != CUBLAS_STATUS_SUCCESS) continue;
        cublasOperation_t ta = transA ? CUBLAS_OP_T : CUBLAS_OP_N, tb = transB ? CUBLAS_OP_T : CUBLAS_OP_N;
        api.desc_set(p.op, CUBLASLT_MATMUL_DESC_TRANSA, &ta, sizeof(ta));
        api.desc_set(p.op, CUBLASLT_MATMUL_DESC_TRANSB, &tb, sizeof(tb));
        bool ok = make_layout(&p.a, transA ? K : M, transA ? M : K, lda) &&
                  make_layout(&p.b, transB ? N : K, transB ? K : N, ldb) && make_layout(&p.c, M, N, ldc);
        cublasLtMatmulPreference_t pref = nullptr;
        ok = ok && api.pref_create(&pref) == CUBLAS_STATUS_SUCCESS;
        if (ok) {
          api.pref_set(pref, CUBLASLT_MATMUL_PREF_MAX_WORKSPACE_BYTES, &workspace_bytes, sizeof(workspace_bytes));
          cublasLtMatmulHeuristicResult_t res[4];
          int n = 0;
          if (api.heuristic(api.handle, p.op, p.a, p.b, p.c, p.c, pref, 4, res, &n) == CUBLAS_STATUS_SUCCESS && n > 0) {
            p.algo = res[0].algo;
            p.ws = res[0].workspaceSize;
            p.emulated = attempt == 0;
            found = true;
          }
          api.pref_destroy(pref);
        }
        if (!found) {
          if (p.a) api.layout_destroy(p.a);
          if (p.b) api.layout_destroy(p.b);
          if (p.c) api.layout_destroy(p.c);
          api.desc_destroy(p.op);
          p = Plan();
        }
      }
      if (!found) {
        set_err("tzg: no cublasLt algorithm for %dx%dx%d (transA=%d transB=%d)", M, N, K, transA, transB);
        return 2;
      }
      it = g_plans.emplace(key, p).first;
    }
    plan = it->second;
  }
  if (plan.ws > workspace_bytes) {
    set_err("tzg: workspace too small (%zu < %zu)", workspace_bytes, plan.ws);
    return 3;
  }
  cublasStatus_t st = api.matmul(api.handle, plan.op, &alpha, A, plan.a, B, plan.b, &beta, C, plan.c, C, plan.c,
                                 &plan.algo, workspace, plan.ws, reinterpret_cast<cudaStream_t>(stream));
  if (st != CUBLAS_STATUS_SUCCESS) {
    set_err("tzg: cublasLtMatmul failed with status %d", (int)st);
    return 4;
  }
  if (used_emulation) *used_emulation = plan.emulated;
  return 0;
}
