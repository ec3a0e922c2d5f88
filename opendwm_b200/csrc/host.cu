// Host-side plumbing shared by all entry points: error string, TMA descriptor
// encoding (driver entry point resolved at run time, no link dependency on
// libcuda), device properties.
#include <stdarg.h>
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "common.cuh"
#include "../../include/dwm_b200.h"

namespace dwm {

static thread_local char g_last_error[1024] = "";

void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_last_error, sizeof(g_last_error), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

static int encode_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                          uint32_t box_rows, uint32_t box_cols, int elem_bytes);

// Descriptor cache: the step launches the same (pointer, shape, box) GEMM operands every
// iteration (weights are packed once, activations live in one workspace), so each distinct
// descriptor is encoded once per process instead of twice per launch (VERDICT r01 item 3,
// SURVEY.md §8(b) threading row).  A descriptor only encodes address + geometry, so a recycled
// address with the same geometry yields the identical descriptor: entries never go stale.
namespace {
struct TmapKey {
  const void* base;
  uint64_t rows, cols, ld;
  uint64_t items, item_ld;   // 0, 0 for a 2-D map
  uint32_t box_rows, box_cols;
  int elem;
  bool operator==(const TmapKey& o) const {
    return base == o.base && rows == o.rows && cols == o.cols && ld == o.ld && items == o.items &&
           item_ld == o.item_ld && box_rows == o.box_rows && box_cols == o.box_cols && elem == o.elem;
  }
};
struct TmapHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = reinterpret_cast<uint64_t>(k.base) * 0x9E3779B97F4A7C15ull;
    h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.cols * 0xC2B2AE3D27D4EB4Full + (h << 6) + (h >> 2));
    h ^= (k.items * 0x165667B19E3779F9ull + k.item_ld + (h << 6) + (h >> 2));
    h ^= (k.ld + (static_cast<uint64_t>(k.box_rows) << 40) + (static_cast<uint64_t>(k.box_cols) << 20) +
          static_cast<uint64_t>(k.elem) + (h << 6) + (h >> 2));
    return static_cast<size_t>(h);
  }
};
std::mutex g_tmap_mu;
std::unordered_map<TmapKey, CUtensorMap, TmapHash> g_tmap_cache;
}  // namespace

static bool tmap_cached(const TmapKey& key, CUtensorMap* map) {
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  auto it = g_tmap_cache.find(key);
  if (it == g_tmap_cache.end()) return false;
  memcpy(map, &it->second, sizeof(CUtensorMap));
  return true;
}

static void tmap_cache_put(const TmapKey& key, const CUtensorMap* map) {
  std::lock_guard<std::mutex> lk(g_tmap_mu);
  if (g_tmap_cache.size() > 8192) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *map);
}

int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                 uint32_t box_rows, uint32_t box_cols, int elem_bytes) {
  const TmapKey key{base, rows, cols, ld, 0, 0, box_rows, box_cols, elem_bytes};
  if (tmap_cached(key, map)) return 0;
  const int rc = encode_tmap_2d(map, base, rows, cols, ld, box_rows, box_cols, elem_bytes);
  if (rc) return rc;
  tmap_cache_put(key, map);
  return 0;
}

int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t items, uint64_t rows, uint64_t cols,
                 uint64_t ld, uint64_t item_ld, uint32_t box_rows, uint32_t box_cols, int elem_bytes) {
  const TmapKey key{base, rows, cols, ld, items, item_ld, box_rows, box_cols, elem_bytes};
  if (tmap_cached(key, map)) return 0;
  const uint64_t dims[3] = {cols, rows, items};
  const uint64_t strides[2] = {ld * static_cast<uint64_t>(elem_bytes), item_ld * static_cast<uint64_t>(elem_bytes)};
  const uint32_t box[3] = {box_cols, box_rows, 1};
  const int rc = make_tmap_nd(map, base, 3, dims, strides, box, elem_bytes);
  if (rc) return rc;
  tmap_cache_put(key, map);
  return 0;
}

static int encode_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t ld,
                          uint32_t box_rows, uint32_t box_cols, int elem_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled not available (no CUDA driver / GPU?)");
    return -3;
  }
  cuuint64_t gdim[2] = {cols, rows};
  cuuint64_t gstride[1] = {ld * static_cast<uint64_t>(elem_bytes)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  // the element type only sets the element size (copies are bitwise; OOB fill is zero bytes)
  CUtensorMapDataType dt = elem_bytes == 2   ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                           : elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                             : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(map, dt, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed (CUresult %d) rows=%llu cols=%llu ld=%llu box=%ux%u",
                   (int)r, (unsigned long long)rows, (unsigned long long)cols,
                   (unsigned long long)ld, box_rows, box_cols);
    return -3;
  }
  return 0;
}

int make_tmap_nd(CUtensorMap* map, const void* base, int rank, const uint64_t* dims,
                 const uint64_t* strides_bytes, const uint32_t* box, int elem_bytes) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) {
    set_last_error("cuTensorMapEncodeTiled not available (no CUDA driver / GPU?)");
    return -3;
  }
  cuuint64_t gdim[5];
  cuuint64_t gstride[4];
  cuuint32_t bx[5], estr[5];
  for (int i = 0; i < rank; ++i) { gdim[i] = dims[i]; bx[i] = box[i]; estr[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gstride[i] = strides_bytes[i];
  CUtensorMapDataType dt = elem_bytes == 2   ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                           : elem_bytes == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8
                                             : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(map, dt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstride, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled (rank %d) failed (CUresult %d)", rank, (int)r);
    return -3;
  }
  return 0;
}

int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

}  // namespace dwm

extern "C" const char* dwm_b200_version(void) { return "dwm_b200 0.1 (sm_90a)"; }
extern "C" const char* dwm_b200_last_error(void) { return dwm::g_last_error; }
