// Host-side CUtensorMap construction. The driver entry point is resolved through the runtime
// (cudaGetDriverEntryPoint) so the library has no link-time dependency on libcuda.
#pragma once
#include <cuda.h>
#include <mutex>
#include <cuda_runtime.h>

#include "common.cuh"

namespace mc {

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
      set_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s", cudaGetErrorString(e));
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

// 2-D bf16 row-major tensor [rows, cols] with row pitch ld (elements); box = [box_rows, box_cols] with box_cols*2 == 128 B,
// 128-byte swizzle. Out-of-bounds box elements are filled with zeros.
// A tensor map is a pure function of (base, shape, pitch, box): the engines call the same few hundred (buffer, shape) pairs every
// forward, so encoded maps are kept in a small direct-mapped cache instead of re-running the driver's encoder per launch.
struct TmapKey {
  const void* base;
  uint64_t rows, cols, ld;
  uint32_t box_rows, box_cols;
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && box_rows == o.box_rows && box_cols == o.box_cols;
  }
};
struct TmapCacheEntry {
  TmapKey key;
  CUtensorMap map;
  bool valid;
};
constexpr int kTmapCacheSize = 1024;
TmapCacheEntry* tmap_cache();          // defined in gemm_wgmma.cu (one table per process; entries are device-pointer keyed)
std::mutex& tmap_cache_mutex();

inline int32_t make_tmap_bf16_2d_uncached(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                                          uint32_t box_cols);

inline int32_t make_tmap_bf16_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                                 uint32_t box_cols) {
  const TmapKey key{base, rows, cols, ld, box_rows, box_cols};
  uint64_t h = reinterpret_cast<uint64_t>(base) >> 4;
  h ^= rows * 0x9E3779B97F4A7C15ull;
  h ^= (cols << 20) ^ (ld << 40) ^ (static_cast<uint64_t>(box_rows) << 8) ^ box_cols;
  h ^= h >> 29;
  h *= 0xBF58476D1CE4E5B9ull;
  h ^= h >> 32;
  TmapCacheEntry& e = tmap_cache()[h % kTmapCacheSize];
  {
    std::lock_guard<std::mutex> g(tmap_cache_mutex());
    if (e.valid && e.key == key) {
      *map = e.map;
      return MC_OK;
    }
  }
  const int32_t rc = make_tmap_bf16_2d_uncached(map, base, rows, cols, ld, box_rows, box_cols);
  if (rc == MC_OK) {
    std::lock_guard<std::mutex> g(tmap_cache_mutex());
    e.key = key;
    e.map = *map;
    e.valid = true;
  }
  return rc;
}

inline int32_t make_tmap_bf16_2d_uncached(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                                          uint32_t box_cols) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return MC_ERR_CUDA;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * 2};  // bytes, dimension 1
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d): base=%p rows=%llu cols=%llu ld=%llu box=[%u,%u]", static_cast<int>(r), base,
              static_cast<unsigned long long>(rows), static_cast<unsigned long long>(cols), static_cast<unsigned long long>(ld), box_rows,
              box_cols);
    return MC_ERR_CUDA;
  }
  return MC_OK;
}

}  // namespace mc
