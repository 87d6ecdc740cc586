// tzk_tma.h — the SWIZZLE_128B box layout and the 2-D tensor maps that tzk_gemm3x.cu and tzk_interact_wide.cu load
// through TMA: boxes of [box_rows x 32 floats] (one 128-B row each).  Under TZK_CPU_SHIM make_map only records the
// tensor for tests/native/sm90_cpu_emu.h.  (Included inside the includer's anonymous namespace, after <cuda.h>.)
#pragma once

// element (row, col) of a [rows x 32 floats] SWIZZLE_128B box: the 16-B chunk index is XOR-ed with row % 8
__device__ __forceinline__ int swz(int row, int col) { return row * 32 + ((((col >> 2) ^ row) & 7) << 2) + (col & 3); }

// ---- host: tensor maps -------------------------------------------------------------------------------------
#ifdef TZK_CPU_SHIM
int make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  map->base = base; map->rows = rows; map->cols = cols; map->ld = ld; map->box_rows = box_rows;
  return 0;
}
#else
typedef CUresult (*EncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// box [32 floats x box_rows], SWIZZLE_128B
int make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  static EncodeTiled encode = nullptr;
  if (!encode) {
    cudaDriverEntryPointQueryResult q;
    void* fn = nullptr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn) return 1;
    encode = reinterpret_cast<EncodeTiled>(fn);
  }
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};          // innermost first
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};                       // bytes, dims 1..rank-1
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS ? 0 : 2;
}
#endif

