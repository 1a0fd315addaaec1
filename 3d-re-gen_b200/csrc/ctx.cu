// Context, error reporting, TMA descriptor creation.
#include <stdlib.h>
#include <string.h>

#include "r3g_internal.h"

extern "C" int r3g_version(void) { return 100; }

extern "C" int r3g_create(int device, r3g_ctx** out) {
  if (!out) return R3G_E_INVALID;
  *out = nullptr;
  r3g_ctx* ctx = (r3g_ctx*)calloc(1, sizeof(r3g_ctx));
  if (!ctx) return R3G_E_INVALID;
  ctx->device = device;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || device < 0 || device >= n) {
    // No CPU fallback: the context is still returned so the caller can read the message.
    snprintf(ctx->err, sizeof(ctx->err), "r3g_create: no usable CUDA device %d (%s, %d devices)", device,
             cudaGetErrorString(e), n);
    *out = ctx;
    return R3G_E_CUDA;
  }
  *out = ctx;
  ctx->pdl = -1;
  // the caller's current device is left as it was (the entry points switch to ctx->device for their own duration)
  struct Restore {
    int prev = -1;
    ~Restore() { if (prev >= 0) cudaSetDevice(prev); }
  } restore;
  if (cudaGetDevice(&restore.prev) != cudaSuccess) restore.prev = -1;
  R3G_CUDA_OK(ctx, cudaSetDevice(device));
  cudaDeviceProp prop;
  R3G_CUDA_OK(ctx, cudaGetDeviceProperties(&prop, device));
  ctx->num_sms = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) {
    return r3g_fail(ctx, R3G_E_CUDA, "r3g_create: device %d is sm_%d%d; this library is sm_90a only", device,
                    prop.major, prop.minor);
  }
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  R3G_CUDA_OK(ctx, cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
  if (!fn || qres != cudaDriverEntryPointSuccess)
    return r3g_fail(ctx, R3G_E_CUDA, "r3g_create: cuTensorMapEncodeTiled not available");
  ctx->encode_tiled = (r3g_pfn_encode_tiled)fn;
  R3G_CUDA_OK(ctx, cudaMallocHost((void**)&ctx->pinned, 64 * sizeof(int64_t)));
  return R3G_OK;
}

extern "C" void r3g_destroy(r3g_ctx* ctx) {
  if (!ctx) return;
  r3g_device_guard guard(ctx);
  if (ctx->pinned) cudaFreeHost(ctx->pinned);
  free(ctx);
}

extern "C" const char* r3g_last_error(r3g_ctx* ctx) { return ctx ? ctx->err : "null context"; }
extern "C" int64_t r3g_launch_count(r3g_ctx* ctx) { return ctx ? ctx->launches : 0; }

int r3g_make_tmap_f16(r3g_ctx* ctx, CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                      const uint64_t* strides_bytes, const uint32_t* box) {
  cuuint64_t gdim[5];
  cuuint64_t gstr[5];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    if (i > 0) {
      gstr[i - 1] = strides_bytes[i];
      if (strides_bytes[i] % 16 != 0)
        return r3g_fail(ctx, R3G_E_INVALID, "tensor-map stride %d = %llu bytes is not a multiple of 16", i,
                        (unsigned long long)strides_bytes[i]);
    }
  }
  if (!r3g_aligned16(base)) return r3g_fail(ctx, R3G_E_INVALID, "tensor-map base not 16-byte aligned");
  CUresult r = ctx->encode_tiled(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, (void*)base, gdim, gstr, bx,
                                 estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                 CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return r3g_fail(ctx, R3G_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return R3G_OK;
}
