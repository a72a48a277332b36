// C-ABI plumbing: error strings, version, launch counter, TMA tensor-map cache.
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "common.cuh"
#include "host_util.h"

namespace cb {

static thread_local char t_err[512] = "";
std::atomic<int64_t> g_launches{0};
static int pdl_default() {
  const char* e = getenv("CB_PDL");
  return (e && e[0] == '1') ? 1 : ((e && e[0] == '2') ? 2 : 0);
}
std::atomic<int> g_pdl{pdl_default()};
static std::atomic<const uint64_t*> g_drop_offset{nullptr};
const uint64_t* drop_offset_ptr() { return g_drop_offset.load(std::memory_order_relaxed); }

// ++*counter; *snapshot = *counter  (one thread; see cb_dropout_offset_advance)
__global__ void drop_offset_advance_kernel(unsigned long long* counter, unsigned long long* snapshot) {
  pdl_wait();
  pdl_trigger();
  const unsigned long long v = *counter + 1ull;
  *counter = v;
  if (snapshot) *snapshot = v;
}

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(t_err, sizeof(t_err), fmt, ap);
  va_end(ap);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q);
    if (e == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

struct TmapKey {
  uint64_t base, inner, rows, ld;
  uint32_t box_inner, box_rows;
  bool operator==(const TmapKey& o) const {
    return base == o.base && inner == o.inner && rows == o.rows && ld == o.ld &&
           box_inner == o.box_inner && box_rows == o.box_rows;
  }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    uint64_t h = k.base * 0x9E3779B97F4A7C15ull;
    h ^= (k.inner + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.rows + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= (k.ld + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2));
    h ^= ((static_cast<uint64_t>(k.box_inner) << 32 | k.box_rows) + (h << 6) + (h >> 2));
    return static_cast<size_t>(h);
  }
};

// The caches hold the encoded maps BY VALUE and hand out copies (made under the lock): a caller keeps its maps in its own
// launch arguments, so evicting the cache can never invalidate a map another call is about to launch with.
bool get_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t ld,
                 uint32_t box_inner, uint32_t box_rows) {
  static std::mutex mu;
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey key{reinterpret_cast<uint64_t>(base), inner, rows, ld, box_inner, box_rows};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    return true;
  }

  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled driver entry point not available");
    return false;
  }
  if ((reinterpret_cast<uint64_t>(base) & 15) != 0 || ((ld * 2) & 15) != 0) {
    set_error("TMA operand must be 16-byte aligned (base %p, row pitch %llu elements)", base,
              (unsigned long long)ld);
    return false;
  }
  alignas(64) CUtensorMap tm;
  CUtensorMap* m = &tm;
  cuuint64_t dims[2] = {inner, rows};
  cuuint64_t strides[1] = {ld * 2};
  cuuint32_t box[2] = {box_inner, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d) inner=%llu rows=%llu ld=%llu box=%ux%u", (int)r,
              (unsigned long long)inner, (unsigned long long)rows, (unsigned long long)ld, box_inner,
              box_rows);
    return false;
  }
  if (cache.size() > 65536) cache.clear();   // unbounded growth guard (base addresses churn under a caching allocator)
  cache.emplace(key, tm);
  *out = tm;
  return true;
}

// The same [rows, cols] row-major bf16 matrix seen as 3-D {64 columns, rows, cols / 64 column blocks}: ONE box of
// {64, box_rows, nblk} lands as nblk consecutive 128B-swizzled [box_rows x 64] slabs - exactly what nblk separate 2-D boxes of an
// MN-major wgmma operand produce - so the producer issues one cp.async.bulk.tensor instead of nblk. cols must be a multiple of 64.
bool get_tmap_3d_mn(CUtensorMap* out, const void* base, uint64_t cols, uint64_t rows, uint64_t ld, uint32_t box_rows, uint32_t nblk) {
  static std::mutex mu;
  static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> cache;
  TmapKey key{reinterpret_cast<uint64_t>(base), cols, rows, ld, 0x80000000u | (nblk << 16) | 64u, box_rows};
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if (it != cache.end()) {
    *out = it->second;
    return true;
  }
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled driver entry point not available");
    return false;
  }
  if ((reinterpret_cast<uint64_t>(base) & 15) != 0 || ((ld * 2) & 15) != 0 || (cols & 63) != 0 || nblk == 0 || nblk > 8) {
    set_error("3-D MN-major tensor map: base %p, row pitch %llu, cols %llu (must be a multiple of 64), %u blocks", base,
              (unsigned long long)ld, (unsigned long long)cols, nblk);
    return false;
  }
  alignas(64) CUtensorMap tm;
  CUtensorMap* m = &tm;
  cuuint64_t dims[3] = {64, rows, cols / 64};
  cuuint64_t strides[2] = {ld * 2, 128};             // bytes: next row, next 64-column block
  cuuint32_t box[3] = {64, box_rows, nblk};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (3-D) failed (%d) cols=%llu rows=%llu ld=%llu box=64x%ux%u", (int)r, (unsigned long long)cols,
              (unsigned long long)rows, (unsigned long long)ld, box_rows, nblk);
    return false;
  }
  if (cache.size() > 65536) cache.clear();
  cache.emplace(key, tm);
  *out = tm;
  return true;
}

}  // namespace cb

extern "C" {
const char* cb_last_error(void) { return cb::t_err; }
int cb_version(void) { return 100; }
int cb_sm_arch(void) { return 90; }
int64_t cb_launch_count(void) { return cb::g_launches.load(std::memory_order_relaxed); }
int cb_set_pdl(int enable) { return cb::g_pdl.exchange(enable == 2 ? 2 : (enable ? 1 : 0), std::memory_order_relaxed); }
int cb_dropout_offset_bind(const uint64_t* device_word) {
  cb::g_drop_offset.store(device_word, std::memory_order_relaxed);
  return CB_OK;
}
int cb_dropout_offset_advance(uint64_t* counter, uint64_t* snapshot, void* stream) {
  CB_REQUIRE(counter != nullptr, "cb_dropout_offset_advance: null counter");
  cb::launch_k(cb::drop_offset_advance_kernel, dim3(1), dim3(1), 0, static_cast<cudaStream_t>(stream),
               reinterpret_cast<unsigned long long*>(counter), reinterpret_cast<unsigned long long*>(snapshot));
  return cb::check_launch("cb_dropout_offset_advance");
}
}
