// vsb200 -- C-ABI plumbing: error text, device check, tensor-map encoding, PAB integer gate.
#include <string.h>

#include <mutex>
#include <unordered_map>

#include "vsb_host.h"

namespace vsbs {
thread_local char g_err[512] = "";
std::atomic<unsigned long long> g_launches{0};
static EncodeTiledFn g_encode = nullptr;
static int g_sms = 0;

EncodeTiledFn encode_tiled() { return g_encode; }

int num_sms() {
  if (g_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_sms <= 0) g_sms = 132;
  }
  return g_sms;
}

static int load_encode() {
  if (g_encode) return VSB_OK;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
  if (e != cudaSuccess || qres != cudaDriverEntryPointSuccess || fn == nullptr)
    return fail(VSB_ERR_CUDA, "cuTensorMapEncodeTiled not available: %s", cudaGetErrorString(e));
  g_encode = reinterpret_cast<EncodeTiledFn>(fn);
  return VSB_OK;
}

// ---- tensor-map cache ------------------------------------------------------------------------------------------
// cuTensorMapEncodeTiled costs ~1-2 us of host time; a denoising step makes hundreds of such calls (3 per GEMM).  torch's caching allocator hands the same addresses back every step, so (base, shape, strides,
// box, swizzle) repeats: an encoded map is a pure function of that key.  Bounded: cleared when it reaches kTmapCacheMax.
struct TmapKey {
  const void* base;
  unsigned long long dims[5], strides[4];
  unsigned box[5], estr[5];
  int rank, swz;
  int dtype, pad_;
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapKeyHash {
  size_t operator()(const TmapKey& k) const {
    const unsigned long long* w = reinterpret_cast<const unsigned long long*>(&k);
    unsigned long long h = 0x9E3779B97F4A7C15ull;
    for (size_t i = 0; i < sizeof(TmapKey) / 8; ++i) {
      h ^= w[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    }
    return (size_t)h;
  }
};
static_assert(sizeof(TmapKey) % 8 == 0, "TmapKey is hashed as 64-bit words");
constexpr size_t kTmapCacheMax = 8192;
static std::unordered_map<TmapKey, CUtensorMap, TmapKeyHash> g_tmap_cache;
static std::mutex g_tmap_mu;
static std::atomic<unsigned long long> g_tmap_hits{0}, g_tmap_misses{0};
static int g_opt_tmap_cache = 1;

static int make_tmap_bf16_uncached(int dtype, CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
                                   const unsigned long long* strides_bytes, const unsigned* box, CUtensorMapSwizzle swz,
                                   const unsigned* elem_strides);

int make_tmap_elem(int dtype, CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box, CUtensorMapSwizzle swz,
                   const unsigned* elem_strides) {
  if (!g_opt_tmap_cache || rank < 1 || rank > 5)
    return make_tmap_bf16_uncached(dtype, m, base, rank, dims, strides_bytes, box, swz, elem_strides);
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base;
  key.rank = rank;
  key.swz = (int)swz;
  key.dtype = dtype;
  for (int i = 0; i < rank; ++i) {
    key.dims[i] = dims[i];
    key.box[i] = box[i];
    key.estr[i] = elem_strides ? elem_strides[i] : 1;
    if (i > 0) key.strides[i - 1] = strides_bytes[i - 1];
  }
  {
    std::lock_guard<std::mutex> g(g_tmap_mu);
    auto it = g_tmap_cache.find(key);
    if (it != g_tmap_cache.end()) {
      *m = it->second;
      g_tmap_hits.fetch_add(1, std::memory_order_relaxed);
      return VSB_OK;
    }
  }
  int rc = make_tmap_bf16_uncached(dtype, m, base, rank, dims, strides_bytes, box, swz, elem_strides);
  if (rc) return rc;
  g_tmap_misses.fetch_add(1, std::memory_order_relaxed);
  std::lock_guard<std::mutex> g(g_tmap_mu);
  if (g_tmap_cache.size() >= kTmapCacheMax) g_tmap_cache.clear();
  g_tmap_cache.emplace(key, *m);
  return VSB_OK;
}

static int make_tmap_bf16_uncached(int dtype, CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
                                   const unsigned long long* strides_bytes, const unsigned* box, CUtensorMapSwizzle swz,
                                   const unsigned* elem_strides) {
  int rc = load_encode();
  if (rc) return rc;
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = elem_strides ? elem_strides[i] : 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i - 1];
      if (gstr[i - 1] % 16) return fail(VSB_ERR_UNSUPPORTED, "tensor map stride %llu not a multiple of 16 bytes", (unsigned long long)gstr[i - 1]);
    }
  }
  CUresult r = g_encode(m, dtype == kTmapDtypeU8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : dtype ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gdim, gstr, bdim,
                        estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(VSB_ERR_CUDA, "cuTensorMapEncodeTiled failed: CUresult %d", (int)r);
  return VSB_OK;
}
}  // namespace vsbs

using namespace vsbs;

extern "C" int vsb_version(void) { return 100; }
extern "C" const char* vsb_last_error(void) { return g_err; }
extern "C" unsigned long long vsb_launch_count(void) { return g_launches.load(); }
extern "C" unsigned long long vsb_tmap_cache_stats(int which) { return which ? g_tmap_misses.load() : g_tmap_hits.load(); }

extern "C" int vsb_init(int device) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) {
    cudaGetLastError();
    return fail(VSB_ERR_NO_DEVICE, "no CUDA device: vsb200 has no CPU fallback");
  }
  if (device < 0 || device >= n) return fail(VSB_ERR_INVALID, "device %d out of range (%d devices)", device, n);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return fail(VSB_ERR_CUDA, "cudaGetDeviceProperties failed");
  if (prop.major != 9 || prop.minor != 0)
    return fail(VSB_ERR_NO_DEVICE, "device %d is sm_%d%d; vsb200 kernels are sm_90a only", device, prop.major, prop.minor);
  // cuTensorMapEncodeTiled needs a current context on some device, not on `device`: the caller's current device is
  // left untouched (the first version called cudaSetDevice(device) and silently changed it)
  g_sms = prop.multiProcessorCount;
  return load_encode();
}

extern "C" int vsb_set_option(const char* name, int value) {
  if (!name) return fail(VSB_ERR_INVALID, "set_option: null name");
  if (!strcmp(name, "tmap_cache")) {
    g_opt_tmap_cache = value;
    return VSB_OK;
  }
  return fail(VSB_ERR_INVALID, "set_option: unknown option '%s'", name);
}

// core/pab/pab_mgr.py:54-91: flag = on && t is not None && count % range != 0 && lo < t < hi; count = (count+1) % steps
extern "C" int vsb_pab_gate(int broadcast_on, int has_timestep, int timestep, int* count, int range, int lo, int hi,
                            int steps) {
  if (!count || steps <= 0) return fail(VSB_ERR_INVALID, "pab_gate: bad args");
  int flag = 0;
  if (broadcast_on && has_timestep) {
    if (range <= 0) return fail(VSB_ERR_INVALID, "pab_gate: range must be positive");
    flag = ((*count % range) != 0) && (lo < timestep) && (timestep < hi);
  }
  *count = (*count + 1) % steps;
  return flag;
}
