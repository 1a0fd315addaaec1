// Float32-activation operators of VGGT's camera head (vggt/vggt/heads/camera_head.py:73-141): the reference runs the
// head outside autocast, on S pose tokens (S = number of frames: 2 in 3D-RE-GEN's stage 4), four refinement iterations of a
// 4-block trunk at width 2048 with 16 heads of 128.  Every linear is therefore a GEMV over a large weight matrix
// (216 M parameters per iteration): HBM-bound.  Weights are held in fp16 (half the bytes), activations, accumulation and
// the residual stream stay float32.
#include <cuda_fp16.h>
#include <math.h>

#include "r3g_internal.h"
#include "r3g_ptx.cuh"

namespace {

using namespace r3g;

constexpr int kRowsPerWarp = 4;
constexpr int kMaxB = 8;

// out[b, n] = epi( W[n, :] . act(vec[b, :]) + bias[n] ),  epi(v) = res[b, n] + gamma[n] * g(v)  (res / gamma optional)
// act: 0 none, 1 silu.  g: 0 none, 1 exact (erf) GELU.
template <int BT>
__global__ void __launch_bounds__(256) gemv_f32_kernel(const __half* __restrict__ w, const float* __restrict__ bias,
                                                       const float* __restrict__ vec, int64_t vec_ld,
                                                       float* __restrict__ out, int64_t out_ld,
                                                       const float* __restrict__ res, const float* __restrict__ gamma,
                                                       int B, int N, int K, int act_in, int act_out) {
  extern __shared__ float sx[];   // [BT][K]
  pdl_wait();
  pdl_trigger();
  for (int i = threadIdx.x; i < BT * K; i += blockDim.x) {
    const int b = i / K, k = i - b * K;
    float xv = 0.f;
    if (b < B) {
      xv = vec[(int64_t)b * vec_ld + k];
      if (act_in == 1) xv = xv / (1.f + expf(-xv));
    }
    sx[i] = xv;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * kRowsPerWarp;
  if (n0 >= N) return;
  float acc[kRowsPerWarp][BT];
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r)
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[r][b] = 0.f;
  const int nch = K >> 3;
  for (int c = lane; c < nch; c += 32) {
    uint4 wv[kRowsPerWarp];
#pragma unroll
    for (int r = 0; r < kRowsPerWarp; ++r) {
      const int n = min(n0 + r, N - 1);
      wv[r] = __ldg(reinterpret_cast<const uint4*>(w + (int64_t)n * K) + c);
    }
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      const float4 lo = reinterpret_cast<const float4*>(sx + b * K)[2 * c];
      const float4 hi = reinterpret_cast<const float4*>(sx + b * K)[2 * c + 1];
      const float xf[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
#pragma unroll
      for (int r = 0; r < kRowsPerWarp; ++r) {
        const __half2* h = reinterpret_cast<const __half2*>(&wv[r]);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 t = __half22float2(h[i]);
          acc[r][b] = fmaf(t.x, xf[2 * i], acc[r][b]);
          acc[r][b] = fmaf(t.y, xf[2 * i + 1], acc[r][b]);
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < kRowsPerWarp; ++r) {
    const int n = n0 + r;
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      float v = warp_sum(acc[r][b]);
      if (lane == 0 && n < N && b < B) {
        if (bias) v += bias[n];
        if (act_out == 1) v = 0.5f * v * (1.f + erff(v * 0.7071067811865476f));
        if (res) v = res[(int64_t)b * out_ld + n] + (gamma ? gamma[n] : 1.f) * v;
        out[(int64_t)b * out_ld + n] = v;
      }
    }
  }
}

// y[r, :] = LN(x[r, :]; eps) (* w + b if given); with modulation: y = gate * (y * (1 + scale) + shift) + x
// (camera_head.py:118-120: gate_msa * modulate(adaln_norm(pose_tokens), shift_msa, scale_msa) + pose_tokens).
__global__ void __launch_bounds__(256) layernorm_f32_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ y,
                                                            int64_t ldy, int width, float eps, const float* __restrict__ w,
                                                            const float* __restrict__ b, const float* __restrict__ shift,
                                                            const float* __restrict__ scale, const float* __restrict__ gate,
                                                            int64_t mod_ld) {
  pdl_wait();
  pdl_trigger();
  __shared__ float red[8], stat[2];
  const int r = blockIdx.x;
  const float* xr = x + (int64_t)r * ldx;
  float s = 0.f;
  for (int i = threadIdx.x; i < width; i += blockDim.x) s += xr[i];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    stat[0] = t / width;
  }
  __syncthreads();
  const float mean = stat[0];
  float q = 0.f;
  for (int i = threadIdx.x; i < width; i += blockDim.x) {
    const float d = xr[i] - mean;
    q += d * d;
  }
  q = warp_sum(q);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = q;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += red[i];
    stat[1] = rsqrtf(t / width + eps);
  }
  __syncthreads();
  const float rstd = stat[1];
  for (int i = threadIdx.x; i < width; i += blockDim.x) {
    float v = (xr[i] - mean) * rstd;
    if (w) v = v * w[i] + (b ? b[i] : 0.f);
    if (gate) v = gate[(int64_t)r * mod_ld + i] * (v * (1.f + scale[(int64_t)r * mod_ld + i]) + shift[(int64_t)r * mod_ld + i]) + xr[i];
    y[(int64_t)r * ldy + i] = v;
  }
}

// Attention over a handful of tokens: qkv float32 [B*S, 3*H*D] laid out (3, H, D) (vggt/layers/attention.py:52-56), one
// warp per (batch, head, query); S <= 64, D a multiple of 32 up to 256.
template <int DPL>   // D / 32
__global__ void __launch_bounds__(128) small_attention_f32_kernel(const float* __restrict__ qkv, float* __restrict__ out, int B,
                                                                  int S, int H, float scale) {
  pdl_wait();
  pdl_trigger();
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B * H * S) return;
  const int i = warp % S, h = (warp / S) % H, bb = warp / (S * H);
  constexpr int D = DPL * 32;
  const int64_t ld = 3LL * H * D;
  const float* q = qkv + (int64_t)(bb * S + i) * ld + (int64_t)h * D;
  float qv[DPL];
#pragma unroll
  for (int d = 0; d < DPL; ++d) qv[d] = q[lane + 32 * d];
  float m = -INFINITY, l = 0.f, acc[DPL];
#pragma unroll
  for (int d = 0; d < DPL; ++d) acc[d] = 0.f;
  for (int j = 0; j < S; ++j) {
    const float* k = qkv + (int64_t)(bb * S + j) * ld + (int64_t)(H + h) * D;
    const float* v = qkv + (int64_t)(bb * S + j) * ld + (int64_t)(2 * H + h) * D;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DPL; ++d) s = fmaf(qv[d], k[lane + 32 * d], s);
    s = warp_sum(s) * scale;
    const float mn = fmaxf(m, s), a = expf(m - mn), p = expf(s - mn);
    l = l * a + p;
#pragma unroll
    for (int d = 0; d < DPL; ++d) acc[d] = acc[d] * a + p * v[lane + 32 * d];
    m = mn;
  }
  float* o = out + (int64_t)(bb * S + i) * (H * D) + (int64_t)h * D;
#pragma unroll
  for (int d = 0; d < DPL; ++d) o[lane + 32 * d] = acc[d] / l;
}

}  // namespace

extern "C" int r3g_gemv_f32(r3g_ctx* ctx, const void* w_f16, const float* bias, const float* vec, int64_t vec_ld, float* out,
                            int64_t out_ld, const float* residual, const float* gamma, int B, int N, int K, int act_in,
                            int act_out, void* stream) {
  R3G_ENTRY(ctx, "gemv_f32");
  if (!w_f16 || !vec || !out || B < 1 || B > kMaxB || K % 8 || vec_ld % 4 || !r3g_aligned16(w_f16) ||
      !r3g_aligned16(vec))
    return r3g_fail(ctx, R3G_E_INVALID, "gemv_f32: B in [1,%d], K %% 8 == 0, 16-byte aligned w / vec required", kMaxB);
  const int bt = B <= 1 ? 1 : B <= 2 ? 2 : B <= 4 ? 4 : 8;
  const size_t smem = (size_t)bt * K * sizeof(float);
  if (smem > 200 * 1024) return r3g_fail(ctx, R3G_E_INVALID, "gemv_f32: B_pad * K * 4 bytes must fit 200 KB of shared memory");
  if (!(ctx->attr_done & R3G_ATTR_MISC0)) {
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(gemv_f32_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(gemv_f32_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(gemv_f32_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(gemv_f32_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    ctx->attr_done |= R3G_ATTR_MISC0;
  }
  const unsigned grid = (unsigned)((N + 8 * kRowsPerWarp - 1) / (8 * kRowsPerWarp));
  auto go = [&](auto kern) {
    return r3g_launch_pdl(ctx, kern, dim3(grid), dim3(256), smem, (cudaStream_t)stream, (const __half*)w_f16, bias, vec, vec_ld,
                          out, out_ld, residual, gamma, B, N, K, act_in, act_out);
  };
  R3G_CUDA_OK(ctx, bt == 1 ? go(gemv_f32_kernel<1>) : bt == 2 ? go(gemv_f32_kernel<2>) : bt == 4 ? go(gemv_f32_kernel<4>)
                                                                                              : go(gemv_f32_kernel<8>));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_layernorm_f32(r3g_ctx* ctx, const float* x, int64_t ldx, float* y, int64_t ldy, int rows, int width,
                                 float eps, const float* w, const float* b, const float* shift, const float* scale,
                                 const float* gate, int64_t mod_ld, void* stream) {
  R3G_ENTRY(ctx, "layernorm_f32");
  if (!x || !y || width < 1 || ((shift == nullptr) != (scale == nullptr)) || ((gate == nullptr) != (scale == nullptr)))
    return r3g_fail(ctx, R3G_E_INVALID, "layernorm_f32: bad arguments (shift / scale / gate come together)");
  if (rows <= 0) return R3G_OK;
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, layernorm_f32_kernel, dim3((unsigned)rows), dim3(256), 0, (cudaStream_t)stream, x, ldx, y,
                                   ldy, width, eps, w, b, shift, scale, gate, mod_ld));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_small_attention_f32(r3g_ctx* ctx, const float* qkv, float* out, int B, int S, int H, int D, float scale,
                                       void* stream) {
  R3G_ENTRY(ctx, "small_attention_f32");
  if (!qkv || !out || B < 1 || S < 1 || S > 64 || H < 1 || D % 32 || D < 32 || D > 256)
    return r3g_fail(ctx, R3G_E_INVALID, "small_attention_f32: S <= 64 and D in {32, 64, ..., 256} required");
  const int warps = B * H * S;
  const unsigned grid = (unsigned)((warps + 3) / 4);
  auto go = [&](auto kern) {
    return r3g_launch_pdl(ctx, kern, dim3(grid), dim3(128), 0, (cudaStream_t)stream, qkv, out, B, S, H, scale);
  };
  cudaError_t e;
  switch (D / 32) {
    case 1: e = go(small_attention_f32_kernel<1>); break;
    case 2: e = go(small_attention_f32_kernel<2>); break;
    case 4: e = go(small_attention_f32_kernel<4>); break;
    case 8: e = go(small_attention_f32_kernel<8>); break;
    default: return r3g_fail(ctx, R3G_E_INVALID, "small_attention_f32: head_dim %d not built (32, 64, 128, 256)", D);
  }
  R3G_CUDA_OK(ctx, e);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}
