// Convolution support for VGGT's DPT depth head (vggt/vggt/heads/dpt_head.py:172-291): every convolution runs as a
// GEMM on the wgmma linear kernel (gemm.cu) over channels-last (NHWC) fp16 feature maps --
//   1x1 convolution, ConvTranspose2d with kernel == stride : r3g_linear directly on the [N*H*W, C] rows,
//   3x3 convolution (padding 1, stride 1 or 2)              : r3g_im2col3x3 -> [N*Ho*Wo, 9*C] rows -> r3g_linear,
// and the align_corners=True bilinear resampling between the fusion stages (custom_interpolate, dpt_head.py:459-484) is
// r3g_bilinear_nhwc.  Both kernels here are pure data movement: HBM-bound, 16-byte accesses.
#include <cuda_fp16.h>

#include "r3g_internal.h"
#include "r3g_ptx.cuh"

namespace {

using namespace r3g;

// cols[(n, yo, xo), (ky*3 + kx) * C + c] = x[n, yo*s + ky - 1, xo*s + kx - 1, c]  (0 outside), optionally relu'd
__global__ void __launch_bounds__(256) im2col3x3_kernel(const __half* __restrict__ x, __half* __restrict__ cols, int N, int H,
                                                        int W, int C, int Ho, int Wo, int stride, int relu_in) {
  pdl_wait();
  pdl_trigger();
  const int c8 = C >> 3;
  const int64_t total = (int64_t)N * Ho * Wo * 9 * c8;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % c8);
    int64_t r = i / c8;
    const int tap = (int)(r % 9);
    r /= 9;                                    // output pixel index (n, yo, xo)
    const int xo = (int)(r % Wo);
    const int yo = (int)((r / Wo) % Ho);
    const int n = (int)(r / ((int64_t)Wo * Ho));
    const int yi = yo * stride + tap / 3 - 1, xi = xo * stride + tap % 3 - 1;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (yi >= 0 && yi < H && xi >= 0 && xi < W) {
      v = *reinterpret_cast<const uint4*>(x + (((int64_t)n * H + yi) * W + xi) * C + 8 * c);
      if (relu_in) {
        __half2* h = reinterpret_cast<__half2*>(&v);
        const __half2 z = __float2half2_rn(0.f);
#pragma unroll
        for (int k = 0; k < 4; ++k) h[k] = __hmax2(h[k], z);
      }
    }
    *reinterpret_cast<uint4*>(cols + r * (9LL * C) + (int64_t)tap * C + 8 * c) = v;
  }
}

// F.interpolate(mode="bilinear", align_corners=True) on NHWC fp16: source coordinate = dst * (in - 1) / (out - 1)
__global__ void __launch_bounds__(256) bilinear_nhwc_kernel(const __half* __restrict__ x, __half* __restrict__ out, int N,
                                                            int Hi, int Wi, int Ho, int Wo, int C) {
  pdl_wait();
  pdl_trigger();
  const int c8 = C >> 3;
  const int64_t total = (int64_t)N * Ho * Wo * c8;
  const float sy = Ho > 1 ? (float)(Hi - 1) / (float)(Ho - 1) : 0.f;
  const float sx = Wo > 1 ? (float)(Wi - 1) / (float)(Wo - 1) : 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % c8);
    int64_t r = i / c8;
    const int xo = (int)(r % Wo);
    const int yo = (int)((r / Wo) % Ho);
    const int n = (int)(r / ((int64_t)Wo * Ho));
    const float fy = yo * sy, fx = xo * sx;
    const int y0 = min((int)fy, Hi - 1), x0 = min((int)fx, Wi - 1);
    const int y1 = min(y0 + 1, Hi - 1), x1 = min(x0 + 1, Wi - 1);
    const float wy = fy - (float)y0, wx = fx - (float)x0;
    const __half* base = x + (int64_t)n * Hi * Wi * C + 8 * c;
    const uint4 v00 = *reinterpret_cast<const uint4*>(base + ((int64_t)y0 * Wi + x0) * C);
    const uint4 v01 = *reinterpret_cast<const uint4*>(base + ((int64_t)y0 * Wi + x1) * C);
    const uint4 v10 = *reinterpret_cast<const uint4*>(base + ((int64_t)y1 * Wi + x0) * C);
    const uint4 v11 = *reinterpret_cast<const uint4*>(base + ((int64_t)y1 * Wi + x1) * C);
    const __half2 *a = reinterpret_cast<const __half2*>(&v00), *b = reinterpret_cast<const __half2*>(&v01);
    const __half2 *cc = reinterpret_cast<const __half2*>(&v10), *d = reinterpret_cast<const __half2*>(&v11);
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __half22float2(a[k]), fb = __half22float2(b[k]), fc = __half22float2(cc[k]), fd = __half22float2(d[k]);
      const float t0 = fa.x + wx * (fb.x - fa.x), t1 = fc.x + wx * (fd.x - fc.x);
      const float u0 = fa.y + wx * (fb.y - fa.y), u1 = fc.y + wx * (fd.y - fc.y);
      oh[k] = __floats2half2_rn(t0 + wy * (t1 - t0), u0 + wy * (u1 - u0));
    }
    *reinterpret_cast<uint4*>(out + r * C + 8 * c) = o;
  }
}

}  // namespace

extern "C" int r3g_im2col3x3(r3g_ctx* ctx, const void* x, void* cols, int N, int H, int W, int C, int stride, int relu_in,
                             void* stream) {
  R3G_ENTRY(ctx, "im2col3x3");
  if (!x || !cols || N < 1 || H < 1 || W < 1 || C < 8 || C % 8 || (stride != 1 && stride != 2) || !r3g_aligned16(x) ||
      !r3g_aligned16(cols))
    return r3g_fail(ctx, R3G_E_INVALID, "im2col3x3: C %% 8 == 0, stride 1 or 2, 16-byte aligned buffers required");
  const int Ho = (H + 2 - 3) / stride + 1, Wo = (W + 2 - 3) / stride + 1;
  const int64_t total = (int64_t)N * Ho * Wo * 9 * (C / 8);
  const unsigned grid = (unsigned)min((total + 255) / 256, (int64_t)ctx->num_sms * 16);
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, im2col3x3_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const __half*)x,
                                   (__half*)cols, N, H, W, C, Ho, Wo, stride, relu_in));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_bilinear_nhwc(r3g_ctx* ctx, const void* x, void* out, int N, int Hi, int Wi, int Ho, int Wo, int C,
                                 void* stream) {
  R3G_ENTRY(ctx, "bilinear_nhwc");
  if (!x || !out || N < 1 || Hi < 1 || Wi < 1 || Ho < 1 || Wo < 1 || C < 8 || C % 8 || !r3g_aligned16(x) ||
      !r3g_aligned16(out))
    return r3g_fail(ctx, R3G_E_INVALID, "bilinear_nhwc: C %% 8 == 0 and 16-byte aligned buffers required");
  const int64_t total = (int64_t)N * Ho * Wo * (C / 8);
  const unsigned grid = (unsigned)min((total + 255) / 256, (int64_t)ctx->num_sms * 16);
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, bilinear_nhwc_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const __half*)x,
                                   (__half*)out, N, Hi, Wi, Ho, Wo, C));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}
