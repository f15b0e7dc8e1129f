// vsb200 -- host-side helpers shared by the translation units behind the C-ABI.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>

#include <atomic>

#include "../../include/vsb200.h"

// Host state shared by the bf16 build and its fp16 twin (namespace vsbs is never renamed; api.cu defines it once).
namespace vsbs {
extern thread_local char g_err[512];
extern std::atomic<unsigned long long> g_launches;

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(VSB_ERR_CUDA, "%s: %s", what, cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return VSB_OK;
}
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// cuTensorMapEncodeTiled, resolved at run time through the runtime API (no link against libcuda).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled();

// Tensor map (dtype 0 = bf16, 1 = fp16, kTmapDtypeU8 = 1-byte), rank <= 5; dims/strides innermost first; strides in BYTES for dims
// 1..rank-1.  elem_strides (null: all 1) are TMA traversal strides: dimension i loads box[i] / elem_strides[i] elements,
// every elem_strides[i]-th one.  Cached by (dtype, base, shape, strides, box, traversal strides, swizzle).
int make_tmap_elem(int dtype, CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box, CUtensorMapSwizzle swz,
                   const unsigned* elem_strides = nullptr);
int num_sms();
constexpr int kTmapDtypeU8 = 2;  // make_tmap_elem dtype of 1-byte elements (e4m3 codes)
}  // namespace vsbs

#ifndef VSB_TMAP_DTYPE
#define VSB_TMAP_DTYPE 0
#endif
#define make_tmap_bf16(...) make_tmap_elem(VSB_TMAP_DTYPE, __VA_ARGS__)

#ifdef VSB_HALF
namespace vsbh { using namespace vsbs; }
#else
namespace vsb { using namespace vsbs; }
#endif
