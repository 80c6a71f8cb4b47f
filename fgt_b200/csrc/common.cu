// Error plumbing, device probing, launch helpers and TMA descriptor encoding (driver entry point fetched at run time,
// so the library links against the CUDA runtime only and loads on hosts without a driver).
#include <stdlib.h>

#include "common.h"

#include <cudaTypedefs.h>
#include <stdarg.h>

#include <mutex>
#include <set>
#include <unordered_map>
#include <utility>

namespace fgt {

static thread_local char g_err[512] = "";

char* err_buf() { return g_err; }

int set_err(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int check_act16(const char* who, const void* hi, long long plane, int vec, bool f16_ok) {
  if (!hi || (reinterpret_cast<uintptr_t>(hi) % (2 * vec) == 0 && plane % vec == 0 && plane >= (f16_ok ? 0 : 1)))
    return FGT_OK;
  return set_err(FGT_ERR_ARG, "%s: 16-bit buffer misaligned or plane offset %lld not a %s multiple of %d", who, plane,
                 f16_ok ? "non-negative" : "positive", vec);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(ptr);
    (void)cudaGetLastError();
  }
  return fn;
}

// Descriptor cache: eager-mode callers (RAFT's 20-iteration loop, the pipeline) launch the same (pointer, shape)
// combinations over and over; encoding is a driver call per map (2-19 maps per GEMM launch). Keyed by every encode
// argument; bounded (cleared when full); thread-safe.
namespace {
struct MapKey {
  uint64_t v[16];
  bool operator==(const MapKey& o) const { return memcmp(v, o.v, sizeof(v)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    uint64_t h = 1469598103934665603ull;
    for (uint64_t x : k.v) {
      h ^= x;
      h *= 1099511628211ull;
    }
    return static_cast<size_t>(h);
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_map_cache;
constexpr size_t kMapCacheMax = 8192;
}  // namespace

static int encode_map_uncached(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank,
                               const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box);

static int encode_map_any(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                          const uint64_t* strides_bytes, const uint32_t* box) {
  if (rank < 1 || rank > 5) return set_err(FGT_ERR_ARG, "tensor map: rank=%d", rank);
  MapKey key;
  memset(&key, 0, sizeof(key));
  key.v[0] = reinterpret_cast<uint64_t>(base);
  key.v[1] = (static_cast<uint64_t>(dtype) << 8) | static_cast<uint64_t>(rank);
  for (int i = 0; i < rank; ++i) key.v[2 + i] = dims[i];
  for (int i = 0; i < rank - 1; ++i) key.v[7 + i] = strides_bytes[i];
  for (int i = 0; i < rank; ++i) key.v[11 + i] = box[i];
  {
    std::lock_guard<std::mutex> lk(g_map_mu);
    auto it = g_map_cache.find(key);
    if (it != g_map_cache.end()) {
      *out = it->second;
      return FGT_OK;
    }
  }
  const int rc = encode_map_uncached(out, dtype, base, rank, dims, strides_bytes, box);
  if (rc == FGT_OK) {
    std::lock_guard<std::mutex> lk(g_map_mu);
    if (g_map_cache.size() >= kMapCacheMax) g_map_cache.clear();
    g_map_cache.emplace(key, *out);
  }
  return rc;
}

static int encode_map_uncached(CUtensorMap* out, CUtensorMapDataType dtype, const void* base, int rank,
                               const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return set_err(FGT_ERR_DEVICE, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (box[i] == 0 || box[i] > 256) return set_err(FGT_ERR_ARG, "tensor map: box[%d]=%u", i, box[i]);
  }
  for (int i = 0; i < rank - 1; ++i) {
    gstr[i] = strides_bytes[i];
    if (gstr[i] % 16 != 0 || gstr[i] == 0)
      return set_err(FGT_ERR_ARG, "tensor map: stride[%d]=%llu not a positive multiple of 16 bytes", i,
                     (unsigned long long)gstr[i]);
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_err(FGT_ERR_ARG, "tensor map: base misaligned");
  CUresult r = fn(out, dtype, static_cast<cuuint32_t>(rank), const_cast<void*>(base),
                  gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_err(FGT_ERR_CUDA,
                   "cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u,%u]",
                   (int)r, rank, (unsigned long long)gdim[0], (unsigned long long)(rank > 1 ? gdim[1] : 0),
                   (unsigned long long)(rank > 2 ? gdim[2] : 0), (unsigned long long)(rank > 3 ? gdim[3] : 0),
                   (unsigned long long)(rank > 4 ? gdim[4] : 0), bx[0], rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0,
                   rank > 3 ? bx[3] : 0, rank > 4 ? bx[4] : 0);
  return FGT_OK;
}

int encode_map_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box) {
  return encode_map_any(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box);
}

bool pdl_enabled() {
  static int on = -1;
  if (on < 0) {
    const char* e = getenv("FGT_PDL");
    on = (e && e[0] == '1') ? 1 : 0;
  }
  return on == 1;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 1;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return 1;
    n = prop.multiProcessorCount;
  }
  return n;
}

int grid_stride(long long items, int block) {
  const long long g = (items + block - 1) / block, cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<int>(g > cap ? cap : (g < 1 ? 1 : g));
}

int allow_dynamic_smem(const void* kernel, size_t bytes, const char* name) {
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) {
    std::lock_guard<std::mutex> lk(mu);
    if (done.count({kernel, dev})) return FGT_OK;
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    if (e == cudaSuccess) {
      done.insert({kernel, dev});
      return FGT_OK;
    }
  }
  return set_err(FGT_ERR_CUDA, "%s: allowing %zu bytes of dynamic shared memory failed: %s", name, bytes,
                 cudaGetErrorString(e));
}

int launch_failed(const char* name, cudaError_t e, dim3 grid, dim3 block, size_t smem) {
  (void)cudaGetLastError();
  return set_err(FGT_ERR_CUDA, "launching %s (grid %ux%ux%u, block %ux%ux%u, %zu bytes of shared memory) failed: %s",
                 name, grid.x, grid.y, grid.z, block.x, block.y, block.z, smem, cudaGetErrorString(e));
}

}  // namespace fgt

extern "C" int fgt_version(void) { return 100; }
extern "C" const char* fgt_last_error(void) { return fgt::err_buf(); }
