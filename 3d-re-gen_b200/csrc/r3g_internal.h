// Internal (non-ABI) declarations shared by the .cu translation units of libr3g.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/r3g.h"

typedef CUresult (*r3g_pfn_encode_tiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                         const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                         CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                         CUtensorMapFloatOOBfill);

struct r3g_ctx {
  int device;
  int num_sms;
  int64_t launches;
  char err[1024];
  r3g_pfn_encode_tiled encode_tiled;
  // pinned host scratch for small device->host results (mc counts)
  int64_t* pinned;
  // per-device lazy state (function attributes and occupancy queries are per device, a context is per device)
  unsigned attr_done;          // R3G_ATTR_* bits: cudaFuncSetAttribute already applied on this context's device
  int pdl;                     // -1 = environment not read yet; R3G_PDL=0 disables programmatic dependent launch
};
enum { R3G_ATTR_ATTENTION = 1, R3G_ATTR_LINEAR128 = 4, R3G_ATTR_LINEAR256 = 8,
       R3G_ATTR_MISC0 = 32, R3G_ATTR_MISC1 = 64, R3G_ATTR_MISC2 = 128, R3G_ATTR_MOE_GEMM = 256 };

// Every ABI entry point runs with the context's device current (a kernel cannot be launched into a stream of
// another device) and restores the caller's device on return.
struct r3g_device_guard {
  int prev = -1;
  bool switched = false;
  explicit r3g_device_guard(const r3g_ctx* ctx) {
    if (ctx && ctx->encode_tiled && cudaGetDevice(&prev) == cudaSuccess && prev != ctx->device)
      switched = cudaSetDevice(ctx->device) == cudaSuccess;
  }
  ~r3g_device_guard() {
    if (switched) cudaSetDevice(prev);
  }
  r3g_device_guard(const r3g_device_guard&) = delete;
  r3g_device_guard& operator=(const r3g_device_guard&) = delete;
};

static inline int r3g_fail(r3g_ctx* ctx, int code, const char* fmt, ...) {
  if (ctx) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(ctx->err, sizeof(ctx->err), fmt, ap);
    va_end(ap);
  }
  return code;
}

// First statement of every compute entry point: refuse a NULL or device-less context (there is no CPU fallback), then
// make the context's device current for the rest of the call.  Argument checks come after it.
#define R3G_ENTRY(ctx, name)                                                                           \
  if (!(ctx) || !(ctx)->encode_tiled)                                                                  \
    return r3g_fail((ctx), R3G_E_CUDA, name ": no CUDA device (there is no CPU fallback)");            \
  r3g_device_guard r3g_guard_(ctx)

// host-side test of the 16-byte alignment that 128-bit accesses and tensor-map bases need (a null pointer passes)
static inline bool r3g_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Layout of a caller-supplied workspace: buffers in the order they are taken, each rounded up to 256 bytes.  A null
// base only measures: every take returns nullptr, and `off` ends as the bytes the workspace needs either way.
struct r3g_carver {
  char* base;
  size_t off = 0;
  template <typename T>
  T* take(size_t count) {
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += (count * sizeof(T) + 255) & ~(size_t)255;
    return p;
  }
};

#define R3G_CUDA_OK(ctx, expr)                                                                         \
  do {                                                                                                 \
    cudaError_t _e = (expr);                                                                           \
    if (_e != cudaSuccess)                                                                             \
      return r3g_fail((ctx), R3G_E_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
  } while (0)

#define R3G_LAUNCH_OK(ctx)                                                                             \
  do {                                                                                                 \
    cudaError_t _e = cudaGetLastError();                                                               \
    if (_e != cudaSuccess)                                                                             \
      return r3g_fail((ctx), R3G_E_CUDA, "%s:%d launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
    (ctx)->launches++;                                                                                 \
  } while (0)

// Launch of a kernel that calls pdl_wait() before its first access to memory another kernel produces (r3g_ptx.cuh):
// with R3G_PDL != 0 it carries the programmatic-stream-serialization attribute, so its prologue overlaps the tail of
// the previous kernel in the stream (also inside CUDA-graph capture, where the edge becomes a programmatic dependency).
#ifdef __CUDACC__
#include <stdlib.h>
#include <utility>
template <typename... KArgs, typename... Args>
inline cudaError_t r3g_launch_pdl(r3g_ctx* ctx, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                                  cudaStream_t s, Args&&... args) {
  if (ctx->pdl < 0) {
    const char* e = getenv("R3G_PDL");
    ctx->pdl = (e && e[0] == '0') ? 0 : 1;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = ctx->pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
#endif

// Connected components of a triangle mesh (mesh.cu): labels[v] = smallest vertex index of v's component, launched on `s`
// without a synchronise.  An index outside [0, nv) sets *bad_dev; skip_dead ignores faces whose first index is negative.
int r3g_launch_components(r3g_ctx* ctx, const int32_t* faces, int64_t nf, int64_t nv, int32_t* labels, int* bad_dev,
                          bool skip_dead, cudaStream_t s);

// 2D..4D fp16 tensor map with 128B swizzle; dims/strides innermost first, strides in BYTES for dims >= 1.
int r3g_make_tmap_f16(r3g_ctx* ctx, CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box);
