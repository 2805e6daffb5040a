// plip_b200 — host runtime helpers: error string, TMA tensor-map encoding.
#include "common.cuh"

#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

namespace plip {

static thread_local char g_last_error[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

const char* get_last_error() { return g_last_error; }

// cuTensorMapEncodeTiled is a driver-API symbol; resolve it through the runtime so the library
// does not link against libcuda.so (absent on the build box).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || p == nullptr) {
    set_last_error("cudaGetDriverEntryPoint(cuTensorMapEncodeTiled) failed: %s",
                   cudaGetErrorString(e));
    return nullptr;
  }
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

// A forward pass needs ~200 tensor maps and they repeat from call to call (same workspace, same weights, same
// micro-batch): encoded maps are cached by their full description.  cuTensorMapEncodeTiled costs ~1-2 us of
// host time each, which is what bounds small-batch latency once the GPU side is a few hundred microseconds.
namespace {
struct TmapKey {
  uint64_t base, rows, cols, stride, box;
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && stride == o.stride && box == o.box;
  }
};
struct TmapHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = k.base * 0x9E3779B97F4A7C15ull;
    h ^= (k.rows + 0x632BE59BD9B4E019ull) + (h << 6) + (h >> 2);
    h ^= (k.cols * 0xC2B2AE3D27D4EB4Full) + (h << 6) + (h >> 2);
    h ^= (k.stride * 0x165667B19E3779F9ull) + (h << 6) + (h >> 2);
    h ^= (k.box + 0x27D4EB2F165667C5ull) + (h << 6) + (h >> 2);
    return (size_t)h;
  }
};
std::mutex g_tmap_mu;
std::unordered_map<TmapKey, CUtensorMap, TmapHash> g_tmap_cache;
}  // namespace

static int encode_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                               uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols);

int make_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  const TmapKey key{reinterpret_cast<uint64_t>(base), rows, cols, row_stride_bytes,
                    (static_cast<uint64_t>(box_rows) << 32) | box_cols};
  {
    std::lock_guard<std::mutex> lk(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *out = it->second;
      return 0;
    }
  }
  if (int rc = encode_tmap_bf16_2d(out, base, rows, cols, row_stride_bytes, box_rows, box_cols)) return rc;
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  if (g_tmap_cache.size() >= 8192) g_tmap_cache.clear();  // callers with ever-changing buffers: bounded memory
  g_tmap_cache.emplace(key, *out);
  return 0;
}

// Not cached: one launch of the long-sequence attention kernel encodes two.
int make_tmap_bf16_3d(CUtensorMap* out, const void* base, uint64_t mats, uint64_t rows, uint64_t cols,
                      uint64_t row_stride_bytes, uint64_t mat_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = resolve_encode();
  if (!enc) return -1;
  cuuint64_t gdim[3] = {cols, rows, mats};
  cuuint64_t gstr[2] = {row_stride_bytes, mat_stride_bytes};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled (3-D) failed (%d): base=%p mats=%llu rows=%llu cols=%llu box=%ux%u",
                   (int)r, base, (unsigned long long)mats, (unsigned long long)rows, (unsigned long long)cols,
                   box_rows, box_cols);
    return -1;
  }
  return 0;
}

static int encode_tmap_bf16_2d(CUtensorMap* out, const void* base, uint64_t rows, uint64_t cols,
                               uint64_t row_stride_bytes, uint32_t box_rows, uint32_t box_cols) {
  EncodeTiledFn enc = resolve_encode();
  if (!enc) return -1;
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstr[1] = {row_stride_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (%d): base=%p rows=%llu cols=%llu stride=%llu box=%ux%u",
                   (int)r, base, (unsigned long long)rows, (unsigned long long)cols,
                   (unsigned long long)row_stride_bytes, box_rows, box_cols);
    return -1;
  }
  return 0;
}

}  // namespace plip
