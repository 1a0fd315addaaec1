// Row-wise / element-wise operators around the tensor-core kernels: LayerNorm(+adaLN modulation), per-head
// q/k normalisation, tiny-M GEMV, timestep embedding, CFG + Euler step, grid Fourier features,
// ln_post + output projection, depth back-projection.  All are HBM-bound: 128-bit accesses, one pass.
#include <cuda_fp16.h>
#include <math.h>

#include <type_traits>

#include "r3g_internal.h"
#include "r3g_ptx.cuh"

using namespace r3g;

namespace {
// Every fp16 row / vector these kernels touch moves as 16-byte accesses: pointers must be 16-byte aligned (leading
// dimensions and column offsets are already required to be multiples of 8 halfs).

// ------------------------------------------------------------------------------------------- LayerNorm
// One warp per row; the row (<= 2048 halfs) lives in registers between the statistics and the write.
constexpr int kLnMaxChunks = 8;  // 8 chunks * 32 lanes * 8 halfs = 2048

// Rows are walked by persistent warps; the NEXT row's 16-byte loads are issued (into packed registers) before the
// current row is reduced, so every warp always has a full row in flight.  NCH = chunks of 8 halfs per lane
// (4: width <= 1024, 8: width <= 2048).  The arithmetic works on fp32 pairs (f2_*, r3g_ptx.cuh) and the affine
// weights sit in shared memory as fp32, which keeps the per-element instruction count low enough for an HBM-bound
// fp16 LayerNorm.
template <int NCH>
__device__ __forceinline__ void load_row(Half8 (&d)[NCH], const Half8* xr, int lane, int nchunks) {
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunks) d[j] = xr[c];
  }
}

// widen a packed row to fp32 pairs; returns the lane's partial sum.  Chunks beyond nchunks are never touched.
template <int NCH>
__device__ __forceinline__ float widen_row(const Half8 (&raw)[NCH], uint64_t (&d)[NCH][4], int lane, int nchunks) {
  uint64_t s2 = f2_pack(0.f, 0.f);
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    if (lane + 32 * j < nchunks) {
      const uint32_t* hw = reinterpret_cast<const uint32_t*>(&raw[j]);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        d[j][k] = h2_to_f2(hw[k]);
        s2 = f2_add(s2, d[j][k]);
      }
    }
  }
  float s0, s1;
  f2_unpack(s2, s0, s1);
  return s0 + s1;
}
// d <- d - mean; returns rstd
template <int NCH>
__device__ __forceinline__ float center_row(uint64_t (&d)[NCH][4], float lane_sum, int lane, int nchunks, int width,
                                            float eps) {
  const float mean = warp_sum(lane_sum) / (float)width;
  const uint64_t nmean = f2_pack(-mean, -mean);
  uint64_t q2 = f2_pack(0.f, 0.f);
#pragma unroll
  for (int j = 0; j < NCH; ++j) {
    if (lane + 32 * j < nchunks) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        d[j][k] = f2_add(d[j][k], nmean);
        q2 = f2_fma(d[j][k], d[j][k], q2);
      }
    }
  }
  float q0, q1;
  f2_unpack(q2, q0, q1);
  return rsqrtf(warp_sum(q0 + q1) / (float)width + eps);
}

template <int NCH>
__global__ void __launch_bounds__(256, NCH == 4 ? 3 : 2) layernorm_kernel(const __half* __restrict__ x, int64_t ldx,
                                                        __half* __restrict__ y, int64_t ldy, int rows, int width,
                                                        float eps, const __half* __restrict__ w,
                                                        const __half* __restrict__ b,
                                                        const __half* __restrict__ scale,
                                                        const __half* __restrict__ shift, int64_t mod_ld,
                                                        int rows_per_batch, int seg_len, int64_t x_seg_stride,
                                                        int64_t y_seg_stride) {
  extern __shared__ __align__(16) float ln_wb[];   // [width] weight (1 if absent), [width] bias (0 if absent)
  if (w || b) {
    for (int i = threadIdx.x; i < width; i += blockDim.x) {
      ln_wb[i] = w ? h2f(w[i]) : 1.f;
      ln_wb[width + i] = b ? h2f(b[i]) : 0.f;
    }
    __syncthreads();
  }
  pdl_wait();      // the affine weights above are constants; x (and the modulation vectors) come from earlier kernels
  pdl_trigger();
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nchunks = width >> 3;
  auto x_row = [&](int r) {
    int64_t xr = r;
    if (seg_len > 0) xr = (int64_t)(r / seg_len) * x_seg_stride + (r % seg_len);
    return reinterpret_cast<const Half8*>(x + xr * ldx);
  };
  Half8 nxt[NCH];
  load_row<NCH>(nxt, x_row(row), lane, nchunks);
  for (; row < rows; row += nwarps) {
    uint64_t d[NCH][4];
    const float lane_sum = widen_row<NCH>(nxt, d, lane, nchunks);
    if (row + nwarps < rows) load_row<NCH>(nxt, x_row(row + nwarps), lane, nchunks);   // in flight under the math
    const float rstd = center_row<NCH>(d, lane_sum, lane, nchunks, width, eps);
    const uint64_t rstd2 = f2_pack(rstd, rstd);
    int64_t yrow = row;
    if (seg_len > 0) yrow = (int64_t)(row / seg_len) * y_seg_stride + (row % seg_len);
    const int bi = rows_per_batch > 0 ? row / rows_per_batch : 0;
    Half8* yr = reinterpret_cast<Half8*>(y + yrow * ldy);
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunks) {
        uint32_t o[4];
        if (w || b) {
          const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(ln_wb + 8 * c);
          const ulonglong2* bp = reinterpret_cast<const ulonglong2*>(ln_wb + width + 8 * c);
          const ulonglong2 w01 = wp[0], w23 = wp[1], b01 = bp[0], b23 = bp[1];
          o[0] = f2_to_h2(f2_fma(f2_mul(d[j][0], rstd2), w01.x, b01.x));
          o[1] = f2_to_h2(f2_fma(f2_mul(d[j][1], rstd2), w01.y, b01.y));
          o[2] = f2_to_h2(f2_fma(f2_mul(d[j][2], rstd2), w23.x, b23.x));
          o[3] = f2_to_h2(f2_fma(f2_mul(d[j][3], rstd2), w23.y, b23.y));
        } else {
#pragma unroll
          for (int k = 0; k < 4; ++k) o[k] = f2_to_h2(f2_mul(d[j][k], rstd2));
        }
        if (scale) {
          // reference: (1 + scale) * LN(x) + shift, every op rounded to fp16 (hunyuan3ddit.py:193).  The operands
          // are halfs, so each fp32-then-round step equals the IEEE half operation: done as three half2 instructions.
          const Half8 sc = reinterpret_cast<const Half8*>(scale + (int64_t)bi * mod_ld)[c];
          const Half8 sh = reinterpret_cast<const Half8*>(shift + (int64_t)bi * mod_ld)[c];
          const __half2* sc2 = reinterpret_cast<const __half2*>(&sc);
          const __half2* sh2 = reinterpret_cast<const __half2*>(&sh);
          const __half2 one = __floats2half2_rn(1.f, 1.f);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const __half2 t = __hadd2(__hmul2(__hadd2(one, sc2[k]), *reinterpret_cast<const __half2*>(&o[k])), sh2[k]);
            o[k] = *reinterpret_cast<const uint32_t*>(&t);
          }
        }
        yr[c] = *reinterpret_cast<const Half8*>(o);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------- q/k norm
// 8 lanes per 64-wide head, 4 (row, head, q|k) groups per warp.
__device__ __forceinline__ float head_sum(float s) {   // over the 8 lanes of a head
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
  s += __shfl_xor_sync(0xffffffffu, s, 4);
  return s;
}

// Normalises in place the 8 features f this lane (sub = lane & 7) holds of a 64-wide head:
//   rms:  f = fp16(f * rrms) * w            ((x*rrms).to(fp16) * scale)
//   else: f = (f - mean) * rstd * w + b     (LayerNorm, b optional)
//   mode 2 (torch's nn.RMSNorm, one rounding): f = f * rrms * w
__device__ __forceinline__ void norm_head8(float (&f)[8], int mode, float eps, const __half* w, const __half* b,
                                           int sub) {
  float wf[8];
  unpack8(reinterpret_cast<const Half8*>(w)[sub], wf);
  if (mode != 1) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[i] * f[i];
    const float rrms = rsqrtf(head_sum(s) * (1.f / 64.f) + eps);
    if (mode == 0) {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = rnd_h(f[i] * rrms) * wf[i];
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[i] = f[i] * rrms * wf[i];
    }
    return;
  }
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += f[i];
  const float mean = head_sum(s) * (1.f / 64.f);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float d = f[i] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(head_sum(q) * (1.f / 64.f) + eps);
  float bf[8];
  if (b) unpack8(reinterpret_cast<const Half8*>(b)[sub], bf);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = (f[i] - mean) * rstd * wf[i] + (b ? bf[i] : 0.f);
}

__global__ void __launch_bounds__(256) qk_norm_kernel(__half* __restrict__ buf, int64_t ld, int64_t ngroups,
                                                      int heads, int64_t q_off, int64_t k_off, int64_t head_stride,
                                                      int mode, float eps, const __half* __restrict__ q_w,
                                                      const __half* __restrict__ q_b, const __half* __restrict__ k_w,
                                                      const __half* __restrict__ k_b, int nsel, int seg_len,
                                                      int64_t seg_stride) {
  const int64_t grp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const bool active = grp < ngroups;
  const int64_t g = active ? grp : 0;
  const int sel = (int)(g % nsel);
  const int64_t rh = g / nsel;
  const int h = (int)(rh % heads);
  int64_t row = rh / heads;
  if (seg_len > 0) row = (row / seg_len) * seg_stride + (row % seg_len);
  __half* p = buf + row * ld + (sel ? k_off : q_off) + (int64_t)h * head_stride + sub * 8;
  float f[8];
  unpack8(*reinterpret_cast<const Half8*>(p), f);
  norm_head8(f, mode, eps, sel ? k_w : q_w, sel ? k_b : q_b, sub);
  if (active) *reinterpret_cast<Half8*>(p) = pack8(f);
}

// ------------------------------------------------------------------------------------------- LayerNorm, fp32 input
__global__ void __launch_bounds__(256) layernorm_f32in_kernel(const float* __restrict__ x, int64_t ldx,
                                                              __half* __restrict__ y, int64_t ldy, int rows,
                                                              int width, float eps, const __half* __restrict__ w,
                                                              const __half* __restrict__ b) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nchunks = width >> 3;
  float v[kLnMaxChunks][8];
  float s = 0.f;
  const float4* xr = reinterpret_cast<const float4*>(x + (int64_t)row * ldx);
#pragma unroll
  for (int j = 0; j < kLnMaxChunks; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunks) {
      const float4 a = xr[2 * c], bb = xr[2 * c + 1];
      v[j][0] = a.x; v[j][1] = a.y; v[j][2] = a.z; v[j][3] = a.w;
      v[j][4] = bb.x; v[j][5] = bb.y; v[j][6] = bb.z; v[j][7] = bb.w;
#pragma unroll
      for (int i = 0; i < 8; ++i) s += v[j][i];
    }
  }
  const float mean = warp_sum(s) / (float)width;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < kLnMaxChunks; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunks) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float d = v[j][i] - mean;
        q += d * d;
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)width + eps);
  Half8* yr = reinterpret_cast<Half8*>(y + (int64_t)row * ldy);
#pragma unroll
  for (int j = 0; j < kLnMaxChunks; ++j) {
    const int c = lane + 32 * j;
    if (c < nchunks) {
      float o[8], wf[8], bf[8];
      if (w) unpack8(reinterpret_cast<const Half8*>(w)[c], wf);
      if (b) unpack8(reinterpret_cast<const Half8*>(b)[c], bf);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        float t = (v[j][i] - mean) * rstd;
        if (w) t *= wf[i];
        if (b) t += bf[i];
        o[i] = t;
      }
      yr[c] = pack8(o);
    }
  }
}

// ------------------------------------------------------------------------------------------- q/k LayerNorm + 2-D RoPE
// 8 lanes per (row, head, q|k) group of 64 features; lanes 0-3 hold the "vertical" half, 4-7 the "horizontal" one;
// inside a half the rotation partner of feature i is i +- 16, i.e. the lane 2 apart.
__global__ void __launch_bounds__(256) qk_norm_rope_kernel(__half* __restrict__ qkv, int64_t ld, int64_t ngroups,
                                                           int heads, float eps, const __half* __restrict__ q_w,
                                                           const __half* __restrict__ q_b,
                                                           const __half* __restrict__ k_w,
                                                           const __half* __restrict__ k_b, float rope_freq,
                                                           int tokens_per_frame, int n_special, int patches_w) {
  const int64_t grp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  const int sub = threadIdx.x & 7;
  const bool active = grp < ngroups;
  const int64_t g = active ? grp : 0;
  const int sel = (int)(g & 1);
  const int64_t rh = g >> 1;
  const int h = (int)(rh % heads);
  const int64_t row = rh / heads;
  __half* p = qkv + row * ld + (int64_t)sel * heads * 64 + (int64_t)h * 64 + sub * 8;
  float f[8];
  unpack8(*reinterpret_cast<const Half8*>(p), f);
  const __half* wv = sel ? k_w : q_w;
  if (wv) norm_head8(f, 1, eps, wv, sel ? k_b : q_b, sub);
  float partner[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) partner[i] = __shfl_xor_sync(0xffffffffu, f[i], 2);
  if (rope_freq > 0.f) {
    const int tok = (int)(row % tokens_per_frame);
    int py = 0, px = 0;
    if (tok >= n_special) {
      const int pidx = tok - n_special;
      py = pidx / patches_w + 1;
      px = pidx % patches_w + 1;
    }
    const float pos = (float)((sub < 4) ? py : px);
    const int within = (sub & 3) * 8;      // feature index inside the 32-wide half
    const bool upper = within >= 16;       // second 16: rotate_features gives +x1, first 16: -x2
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int j = (within + i) & 15;     // frequency index
      const float inv_freq = 1.f / powf(rope_freq, (float)(2 * j) / 32.f);
      const float ang = pos * inv_freq;
      float sn, cs;
      sincosf(ang, &sn, &cs);
      const float rot = upper ? partner[i] : -partner[i];
      f[i] = f[i] * cs + rot * sn;
    }
  }
  if (active) *reinterpret_cast<Half8*>(p) = pack8(f);
}

// ------------------------------------------------------------------------------------------- patchify
__global__ void __launch_bounds__(256) patchify_kernel(const float* __restrict__ img, __half* __restrict__ out,
                                                       int64_t out_ld, int N, int H, int W, int ps, float m0, float m1,
                                                       float m2, float s0, float s1, float s2) {
  const int hp = H / ps, wp = W / ps, kk = 3 * ps * ps;
  const int64_t row = blockIdx.x;   // one block per patch
  const int n = (int)(row / (hp * wp)), pr = (int)(row % (hp * wp));
  const int y0 = (pr / wp) * ps, x0 = (pr % wp) * ps;
  for (int col = threadIdx.x; col < out_ld; col += blockDim.x) {
    float v = 0.f;
    if (col < kk) {
      const int c = col / (ps * ps), r = col % (ps * ps);
      const float px = img[(((int64_t)n * 3 + c) * H + y0 + r / ps) * W + x0 + r % ps];
      const float mean = c == 0 ? m0 : (c == 1 ? m1 : m2), sd = c == 0 ? s0 : (c == 1 ? s1 : s2);
      v = (px - mean) / sd;
    }
    out[row * out_ld + col] = __float2half_rn(v);
  }
}

// ------------------------------------------------------------------------------------------- GEMV (M <= 8)
constexpr int kGemvMaxB = 8;
constexpr int kGemvRows = 4;   // output rows per warp, their weight loads issued together (bytes in flight)
// The activated input vectors are staged once per block in shared memory, so silu() -- an expf and a divide -- is
// evaluated once per input element instead of once per output row.
template <int BT>
__global__ void __launch_bounds__(256) gemv_kernel(const __half* __restrict__ w, const __half* __restrict__ bias,
                                                   const __half* __restrict__ vec, int64_t vec_ld,
                                                   __half* out, int64_t out_ld, const __half* residual, int B, int N,
                                                   int K, int silu_in, int silu_out) {
  extern __shared__ float gemv_x[];   // [BT][K]
  pdl_wait();      // vec is the previous kernel's output
  pdl_trigger();
  for (int i = threadIdx.x; i < BT * K; i += blockDim.x) {
    const int b = i / K, k = i - b * K;
    float xv = 0.f;
    if (b < B) {
      xv = h2f(vec[(int64_t)b * vec_ld + k]);
      if (silu_in) xv = rnd_h(xv / (1.f + expf(-xv)));
    }
    gemv_x[i] = xv;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * kGemvRows;
  if (n0 >= N) return;
  float acc[kGemvRows][BT];
#pragma unroll
  for (int r = 0; r < kGemvRows; ++r)
#pragma unroll
    for (int b = 0; b < BT; ++b) acc[r][b] = 0.f;
  const int nch = K >> 3;
  for (int c = lane; c < nch; c += 32) {
    Half8 wv[kGemvRows];
#pragma unroll
    for (int r = 0; r < kGemvRows; ++r) {
      const int n = min(n0 + r, N - 1);
      wv[r] = reinterpret_cast<const Half8*>(w + (int64_t)n * K)[c];
    }
    float xf[BT][8];
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      const float4 lo = reinterpret_cast<const float4*>(gemv_x + b * K)[2 * c];
      const float4 hi = reinterpret_cast<const float4*>(gemv_x + b * K)[2 * c + 1];
      xf[b][0] = lo.x; xf[b][1] = lo.y; xf[b][2] = lo.z; xf[b][3] = lo.w;
      xf[b][4] = hi.x; xf[b][5] = hi.y; xf[b][6] = hi.z; xf[b][7] = hi.w;
    }
#pragma unroll
    for (int r = 0; r < kGemvRows; ++r) {
      float wf[8];
      unpack8(wv[r], wf);
#pragma unroll
      for (int b = 0; b < BT; ++b)
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[r][b] += wf[i] * xf[b][i];
    }
  }
#pragma unroll
  for (int r = 0; r < kGemvRows; ++r) {
    const int n = n0 + r;
#pragma unroll
    for (int b = 0; b < BT; ++b) {
      float v = warp_sum(acc[r][b]);
      if (lane == 0 && n < N && b < B) {
        if (bias) v += h2f(bias[n]);
        if (silu_out) {
          v = rnd_h(v);
          v = v / (1.f + expf(-v));
        }
        // residual may alias out: this lane reads the element before it writes it
        if (residual) v = rnd_h(v) + h2f(residual[(int64_t)b * out_ld + n]);
        out[(int64_t)b * out_ld + n] = __float2half_rn(v);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------- timestep embedding
__global__ void timestep_embedding_kernel(const __half* __restrict__ t, __half* __restrict__ out, int B, int dim,
                                          float time_factor, float max_period) {
  const int half_dim = dim / 2;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * half_dim) return;
  const int b = i / half_dim, k = i % half_dim;
  const float ts = rnd_h(time_factor * h2f(t[b]));  // `time_factor * t` is evaluated in t's dtype (fp16)
  const float freq = expf(-logf(max_period) * (float)k / (float)half_dim);
  const float arg = ts * freq;
  out[(int64_t)b * dim + k] = __float2half_rn(cosf(arg));
  out[(int64_t)b * dim + half_dim + k] = __float2half_rn(sinf(arg));
  if ((dim & 1) && k == 0) out[(int64_t)b * dim + dim - 1] = __float2half_rn(0.f);
}

// ------------------------------------------------------------------------------------------- CFG + Euler
// nb = 2: v = cat(cond, uncond), mixed with the guidance scale first.  nb = 1: v is the prediction itself (a model run
// without CFG), guidance is not read.
__global__ void cfg_euler_kernel(__half* __restrict__ x, const __half* __restrict__ v, __half* __restrict__ x_dup,
                                 int64_t n, int nb, float guidance, float dsigma) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float mix = h2f(v[i]);
  if (nb == 2) {
    const float vc = mix, vu = h2f(v[n + i]);
    // noise_pred_uncond + g * (cond - uncond), each op rounded to fp16 (pipelines.py:753)
    mix = rnd_h(vu + rnd_h(guidance * rnd_h(vc - vu)));
  }
  // (sigma_next - sigma) is a 0-dim fp32 tensor: the product takes the fp16 dtype of model_output,
  // the sum is fp32 (schedulers.py:300-309, :462-469)
  const float step = rnd_h(dsigma * mix);
  const __half r = __float2half_rn(h2f(x[i]) + step);
  x[i] = r;
  if (x_dup) {
    x_dup[i] = r;
    if (nb == 2) x_dup[n + i] = r;
  }
}

// ------------------------------------------------------------------------------------------- grid Fourier features
struct GridParams {
  double lo[3], step[3], hi[3];
  int R;
  int num_freqs;
  int include_pi;
};

// kF32 = false: the queries are an fp16 tensor, the products x * f are fp16 arithmetic (the dense-grid path,
// volume_decoders.py:168); kF32 = true: float32 queries (FlashVDM's refinement levels, volume_decoders.py:395-396): the
// embedding is computed in float32 and only the result is cast to the latents' dtype (attention_blocks.py:486).
template <bool kF32 = false>
__device__ __forceinline__ void fourier_row(__half* o, int64_t out_ld, const float* xh, int F, int include_pi);

__global__ void __launch_bounds__(256) grid_fourier_kernel(__half* __restrict__ out, int64_t out_ld, int64_t start,
                                                           int64_t count, GridParams gp) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int64_t p = start + i;
  const int n = gp.R + 1;
  int idx[3];
  idx[2] = (int)(p % n);
  idx[1] = (int)((p / n) % n);
  idx[0] = (int)(p / ((int64_t)n * n));
  __half* o = out + i * out_ld;
  float xh[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    // np.linspace(lo, hi, R+1, dtype=float32): float64 arange*step+lo, endpoint forced, then float32, then fp16
    double c = (idx[d] == gp.R) ? gp.hi[d] : __dadd_rn(__dmul_rn((double)idx[d], gp.step[d]), gp.lo[d]);
    xh[d] = rnd_h((float)c);
  }
  fourier_row(o, out_ld, xh, gp.num_freqs, gp.include_pi);
}

// T = __half or float queries
template <typename T>
__global__ void __launch_bounds__(256) points_fourier_kernel(const T* __restrict__ q, __half* __restrict__ out,
                                                             int64_t out_ld, int64_t n, int F, int include_pi) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float xh[3] = {(float)q[3 * i], (float)q[3 * i + 1], (float)q[3 * i + 2]};
  fourier_row<std::is_same<T, float>::value>(out + i * out_ld, out_ld, xh, F, include_pi);
}

template <bool kF32>
__device__ __forceinline__ void fourier_row(__half* o, int64_t out_ld, const float* xh, int F, int include_pi) {
  if (F == 8 && out_ld == 64 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
    // the geo-decoder's shape: the 51 features + 13 zeros of a row are built in registers and leave as eight
    // 16-byte stores (a thread owns 128 contiguous bytes) instead of 64 strided 2-byte ones.
    // sinf / cosf (not the fast intrinsics) because torch.sin on an fp16 tensor is sinf of the widened value; their
    // Payne-Hanek branch for |x| > 105615 is where this kernel's 32 bytes of stack come from -- unreachable for an
    // fp16 argument (|e| <= 65504), so the local memory is never touched at run time.
    __half r[64];
#pragma unroll
    for (int c = 0; c < 64; ++c) r[c] = __float2half_rn(0.f);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      r[d] = __float2half_rn(xh[d]);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        float f = (float)(1 << k);
        if (include_pi) f = rnd_h(f * 3.14159265358979323846f);
        const float e = kF32 ? xh[d] * f : rnd_h(xh[d] * f);
        r[3 + d * 8 + k] = __float2half_rn(sinf(e));
        r[3 + 24 + d * 8 + k] = __float2half_rn(cosf(e));
      }
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) reinterpret_cast<uint4*>(o)[c] = reinterpret_cast<const uint4*>(r)[c];
    return;
  }
#pragma unroll
  for (int d = 0; d < 3; ++d) o[d] = __float2half_rn(xh[d]);
  for (int d = 0; d < 3; ++d)
    for (int k = 0; k < F; ++k) {
      float f = (float)(1 << k);
      if (include_pi) f = rnd_h(f * 3.14159265358979323846f);
      const float e = kF32 ? xh[d] * f : rnd_h(xh[d] * f);  // fp16 product (frequencies buffer is cast to fp16 with the module)
      o[3 + d * F + k] = __float2half_rn(sinf(e));
      o[3 + 3 * F + d * F + k] = __float2half_rn(cosf(e));
    }
  for (int c = 3 + 6 * F; c < out_ld; ++c) o[c] = __float2half_rn(0.f);
}

// ------------------------------------------------------------------------------------------- SwiGLU gate
// out[r, j] = fp16( fp16(silu(x[r, j])) * x[r, F + j] ): Dinov2SwiGLUFFN (transformers modeling_dinov2.py: hidden =
// silu(x1) * x2 after weights_in(...).chunk(2)), the MLP of the DINOv2-giant conditioner (conditioner.py:125-131).
__global__ void __launch_bounds__(256) swiglu_kernel(const __half* __restrict__ x, int64_t ldx, __half* __restrict__ out,
                                                     int64_t ldo, int64_t rows, int F) {
  pdl_wait();
  pdl_trigger();
  const int chunks = F >> 3;
  const int64_t total = rows * chunks;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / chunks;
    const int c = (int)(i - r * chunks);
    const Half8 a = *reinterpret_cast<const Half8*>(x + r * ldx + 8 * c);
    const Half8 b = *reinterpret_cast<const Half8*>(x + r * ldx + F + 8 * c);
    float fa[8], fb[8], o[8];
    unpack8(a, fa);
    unpack8(b, fb);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = rnd_h(fa[k] / (1.f + __expf(-fa[k]))) * fb[k];
    *reinterpret_cast<Half8*>(out + r * ldo + 8 * c) = pack8(o);
  }
}

// ------------------------------------------------------------------------------------------- ln_post + output_proj
template <int NCH>
__global__ void __launch_bounds__(256, NCH == 4 ? 3 : 2) lnpost_dot_kernel(const __half* __restrict__ x, int64_t ldx, int rows,
                                                         int width, float eps, const __half* __restrict__ ln_w,
                                                         const __half* __restrict__ ln_b,
                                                         const __half* __restrict__ w_out,
                                                         const __half* __restrict__ b_out, float* __restrict__ out) {
  extern __shared__ __align__(16) float lp_c[];   // [width] ln weight, [width] ln bias, [width] output_proj weight
  for (int i = threadIdx.x; i < width; i += blockDim.x) {
    lp_c[i] = h2f(ln_w[i]);
    lp_c[width + i] = h2f(ln_b[i]);
    lp_c[2 * width + i] = h2f(w_out[i]);
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nchunks = width >> 3;
  Half8 nxt[NCH];
  load_row<NCH>(nxt, reinterpret_cast<const Half8*>(x + (int64_t)row * ldx), lane, nchunks);
  for (; row < rows; row += nwarps) {
    uint64_t d[NCH][4];
    const float lane_sum = widen_row<NCH>(nxt, d, lane, nchunks);
    if (row + nwarps < rows)
      load_row<NCH>(nxt, reinterpret_cast<const Half8*>(x + (int64_t)(row + nwarps) * ldx), lane, nchunks);
    const float rstd = center_row<NCH>(d, lane_sum, lane, nchunks, width, eps);
    const uint64_t rstd2 = f2_pack(rstd, rstd);
    uint64_t acc2 = f2_pack(0.f, 0.f);
#pragma unroll
    for (int j = 0; j < NCH; ++j) {
      const int c = lane + 32 * j;
      if (c < nchunks) {
        const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(lp_c + 8 * c);
        const ulonglong2* bp = reinterpret_cast<const ulonglong2*>(lp_c + width + 8 * c);
        const ulonglong2* op = reinterpret_cast<const ulonglong2*>(lp_c + 2 * width + 8 * c);
        const ulonglong2 w01 = wp[0], w23 = wp[1], b01 = bp[0], b23 = bp[1], o01 = op[0], o23 = op[1];
        // ln_post output is an fp16 tensor (rounded), the 1024 -> 1 projection accumulates in fp32
        acc2 = f2_fma(h2_to_f2(f2_to_h2(f2_fma(f2_mul(d[j][0], rstd2), w01.x, b01.x))), o01.x, acc2);
        acc2 = f2_fma(h2_to_f2(f2_to_h2(f2_fma(f2_mul(d[j][1], rstd2), w01.y, b01.y))), o01.y, acc2);
        acc2 = f2_fma(h2_to_f2(f2_to_h2(f2_fma(f2_mul(d[j][2], rstd2), w23.x, b23.x))), o23.x, acc2);
        acc2 = f2_fma(h2_to_f2(f2_to_h2(f2_fma(f2_mul(d[j][3], rstd2), w23.y, b23.y))), o23.y, acc2);
      }
    }
    float a0, a1;
    f2_unpack(acc2, a0, a1);
    const float acc = warp_sum(a0 + a1);
    if (lane == 0) out[row] = rnd_h(acc + (b_out ? h2f(b_out[0]) : 0.f));
  }
}

// ------------------------------------------------------------------------------------------- back-projection
struct UnprojectFrame {
  double r[9];  // cam-to-world rotation, row-major
  double t[3];
  float fu, fv, cu, cv;
};
constexpr int kMaxFrames = 32;  // 32 * 112 B of kernel parameters
struct UnprojectParams {
  UnprojectFrame f[kMaxFrames];
};

template <bool kF64>
__global__ void __launch_bounds__(256) unproject_kernel(const float* __restrict__ depth, void* __restrict__ out,
                                                        int H, int W, int frame0,
                                                        const __grid_constant__ UnprojectParams prm) {
  // one thread = 2 horizontally adjacent pixels: 8-byte load, 3 x 16-byte (f64) stores
  const int s = blockIdx.z;
  const UnprojectFrame& fr = prm.f[s];
  const int64_t pairs_per_frame = ((int64_t)H * W + 1) / 2;
  const int64_t pi = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (pi >= pairs_per_frame) return;
  const int64_t frame_off = (int64_t)(frame0 + s) * H * W;
  const int64_t p0 = 2 * pi;
  float d[2];
  const bool two = p0 + 1 < (int64_t)H * W;
  const bool vec = two && (((frame_off + p0) & 1) == 0);  // 8/16-byte alignment of the pair
  if (vec) {
    float2 t = *reinterpret_cast<const float2*>(depth + frame_off + p0);
    d[0] = t.x; d[1] = t.y;
  } else {
    d[0] = depth[frame_off + p0];
    d[1] = two ? depth[frame_off + p0 + 1] : 0.f;
  }
  double wx[2], wy[2], wz[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int64_t p = p0 + k;
    const int u = (int)(p % W), v = (int)(p / W);
    // (u - cu) * depth / fu in float64, stored float32 (geometry.py:107-114)
    const float xc = (float)(__ddiv_rn(__dmul_rn((double)u - (double)fr.cu, (double)d[k]), (double)fr.fu));
    const float yc = (float)(__ddiv_rn(__dmul_rn((double)v - (double)fr.cv, (double)d[k]), (double)fr.fv));
    const float zc = d[k];
    // np.dot(cam, R^T) + t in float64 (geometry.py:80)
    wx[k] = fma((double)zc, fr.r[2], fma((double)yc, fr.r[1], (double)xc * fr.r[0])) + fr.t[0];
    wy[k] = fma((double)zc, fr.r[5], fma((double)yc, fr.r[4], (double)xc * fr.r[3])) + fr.t[1];
    wz[k] = fma((double)zc, fr.r[8], fma((double)yc, fr.r[7], (double)xc * fr.r[6])) + fr.t[2];
  }
  if (kF64) {
    double* o = reinterpret_cast<double*>(out) + 3 * (frame_off + p0);
    if (vec) {
      reinterpret_cast<double2*>(o)[0] = make_double2(wx[0], wy[0]);
      reinterpret_cast<double2*>(o)[1] = make_double2(wz[0], wx[1]);
      reinterpret_cast<double2*>(o)[2] = make_double2(wy[1], wz[1]);
    } else {
      o[0] = wx[0]; o[1] = wy[0]; o[2] = wz[0];
      if (two) { o[3] = wx[1]; o[4] = wy[1]; o[5] = wz[1]; }
    }
  } else {
    float* o = reinterpret_cast<float*>(out) + 3 * (frame_off + p0);
    if (vec) {
      reinterpret_cast<float2*>(o)[0] = make_float2((float)wx[0], (float)wy[0]);
      reinterpret_cast<float2*>(o)[1] = make_float2((float)wz[0], (float)wx[1]);
      reinterpret_cast<float2*>(o)[2] = make_float2((float)wy[1], (float)wz[1]);
    } else {
      o[0] = (float)wx[0]; o[1] = (float)wy[0]; o[2] = (float)wz[0];
      if (two) { o[3] = (float)wx[1]; o[4] = (float)wy[1]; o[5] = (float)wz[1]; }
    }
  }
}

}  // namespace

extern "C" int r3g_layernorm(r3g_ctx* ctx, const void* x, int64_t ldx, void* y, int64_t ldy, int rows, int width,
                             float eps, const void* w, const void* b, const void* scale, const void* shift,
                             int64_t mod_ld, int rows_per_batch, int seg_len, int64_t x_seg_stride,
                             int64_t y_seg_stride, void* stream) {
  R3G_ENTRY(ctx, "layernorm");
  if (width % 8 || width > kLnMaxChunks * 256 || ldx % 8 || ldy % 8 || (scale && (mod_ld % 8)))
    return r3g_fail(ctx, R3G_E_INVALID, "layernorm: width %d must be a multiple of 8 and <= %d", width,
                    kLnMaxChunks * 256);
  if ((scale == nullptr) != (shift == nullptr)) return r3g_fail(ctx, R3G_E_INVALID, "layernorm: scale/shift pair");
  if (!r3g_aligned16(x) || !r3g_aligned16(y) || !r3g_aligned16(w) || !r3g_aligned16(b) || !r3g_aligned16(scale) ||
      !r3g_aligned16(shift))
    return r3g_fail(ctx, R3G_E_INVALID, "layernorm: pointers must be 16-byte aligned");
  if (rows <= 0) return R3G_OK;
  // persistent beyond one resident wave (3 blocks per SM at width <= 1024, 2 above)
  const unsigned grid = (unsigned)min((rows + 7) / 8, ctx->num_sms * (width <= 1024 ? 3 : 2));
  const size_t smem = (w || b) ? (size_t)2 * width * sizeof(float) : 0;
  auto go = [&](auto kern) {
    return r3g_launch_pdl(ctx, kern, dim3(grid), dim3(256), smem, (cudaStream_t)stream, (const __half*)x, ldx, (__half*)y,
                          ldy, rows, width, eps, (const __half*)w, (const __half*)b, (const __half*)scale,
                          (const __half*)shift, mod_ld, rows_per_batch, seg_len, x_seg_stride, y_seg_stride);
  };
  R3G_CUDA_OK(ctx, width <= 1024 ? go(layernorm_kernel<4>) : go(layernorm_kernel<8>));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_layernorm_f32in(r3g_ctx* ctx, const float* x, int64_t ldx, void* y, int64_t ldy, int rows,
                                   int width, float eps, const void* w, const void* b, void* stream) {
  R3G_ENTRY(ctx, "layernorm_f32in");
  if (width % 8 || width > kLnMaxChunks * 256 || ldx % 4 || ldy % 8)
    return r3g_fail(ctx, R3G_E_INVALID, "layernorm_f32in: width %d must be a multiple of 8 and <= %d", width,
                    kLnMaxChunks * 256);
  if (!r3g_aligned16(x) || !r3g_aligned16(y) || !r3g_aligned16(w) || !r3g_aligned16(b))
    return r3g_fail(ctx, R3G_E_INVALID, "layernorm_f32in: pointers must be 16-byte aligned");
  if (rows <= 0) return R3G_OK;
  layernorm_f32in_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, ldx, (__half*)y, ldy, rows, width, eps,
                                                                             (const __half*)w, (const __half*)b);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_qk_norm_rope(r3g_ctx* ctx, void* qkv, int64_t ld, int64_t rows, int heads, float eps,
                                const void* q_w, const void* q_b, const void* k_w, const void* k_b, float rope_freq,
                                int tokens_per_frame, int n_special, int patches_w, void* stream) {
  R3G_ENTRY(ctx, "qk_norm_rope");
  if (ld % 8 || (q_w == nullptr) != (k_w == nullptr) || tokens_per_frame < 1 || patches_w < 1)
    return r3g_fail(ctx, R3G_E_INVALID, "qk_norm_rope: bad arguments");
  if (!r3g_aligned16(qkv) || !r3g_aligned16(q_w) || !r3g_aligned16(q_b) || !r3g_aligned16(k_w) || !r3g_aligned16(k_b))
    return r3g_fail(ctx, R3G_E_INVALID, "qk_norm_rope: pointers must be 16-byte aligned");
  const int64_t ngroups = rows * heads * 2;
  if (ngroups <= 0) return R3G_OK;
  qk_norm_rope_kernel<<<(unsigned)((ngroups * 8 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (__half*)qkv, ld, ngroups, heads, eps, (const __half*)q_w, (const __half*)q_b, (const __half*)k_w,
      (const __half*)k_b, rope_freq, tokens_per_frame, n_special, patches_w);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_patchify(r3g_ctx* ctx, const float* images, void* out, int64_t out_ld, int N, int H, int W,
                            int patch, const float* mean3_host, const float* std3_host, void* stream) {
  R3G_ENTRY(ctx, "patchify");
  if (!images || !out || patch < 1 || H % patch || W % patch || out_ld < 3 * patch * patch)
    return r3g_fail(ctx, R3G_E_INVALID, "patchify: bad arguments");
  const float m[3] = {mean3_host ? mean3_host[0] : 0.f, mean3_host ? mean3_host[1] : 0.f, mean3_host ? mean3_host[2] : 0.f};
  const float sd[3] = {std3_host ? std3_host[0] : 1.f, std3_host ? std3_host[1] : 1.f, std3_host ? std3_host[2] : 1.f};
  const int64_t rows = (int64_t)N * (H / patch) * (W / patch);
  if (rows <= 0) return R3G_OK;
  patchify_kernel<<<(unsigned)rows, 256, 0, (cudaStream_t)stream>>>(images, (__half*)out, out_ld, N, H, W, patch, m[0],
                                                                     m[1], m[2], sd[0], sd[1], sd[2]);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_qk_norm(r3g_ctx* ctx, void* buf, int64_t ld, int rows, int heads, int64_t q_off, int64_t k_off,
                           int64_t head_stride, int mode, float eps, const void* q_w, const void* q_b,
                           const void* k_w, const void* k_b, int seg_len, int64_t seg_stride, void* stream) {
  R3G_ENTRY(ctx, "qk_norm");
  if (ld % 8 || q_off % 8 || k_off % 8 || head_stride % 8 || !q_w)
    return r3g_fail(ctx, R3G_E_INVALID, "qk_norm: offsets/strides must be multiples of 8 halfs");
  if (mode < 0 || mode > 2) return r3g_fail(ctx, R3G_E_INVALID, "qk_norm: mode must be 0, 1 or 2, got %d", mode);
  if (!r3g_aligned16(buf) || !r3g_aligned16(q_w) || !r3g_aligned16(q_b) || !r3g_aligned16(k_w) || !r3g_aligned16(k_b))
    return r3g_fail(ctx, R3G_E_INVALID, "qk_norm: pointers must be 16-byte aligned");
  const int nsel = k_w ? 2 : 1;
  const int64_t ngroups = (int64_t)rows * heads * nsel;
  if (ngroups <= 0) return R3G_OK;
  const int64_t threads = ngroups * 8;
  qk_norm_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (__half*)buf, ld, ngroups, heads, q_off, k_off, head_stride, mode, eps, (const __half*)q_w,
      (const __half*)q_b, (const __half*)k_w, (const __half*)k_b, nsel, seg_len, seg_stride);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_gemv(r3g_ctx* ctx, const void* w, const void* bias, const void* vec, int64_t vec_ld, void* out,
                        int64_t out_ld, const void* residual, int B, int N, int K, int silu_in, int silu_out,
                        void* stream) {
  R3G_ENTRY(ctx, "gemv");
  if (B < 1 || B > kGemvMaxB || K % 8 || vec_ld % 8)
    return r3g_fail(ctx, R3G_E_INVALID, "gemv: B in [1,%d], K %% 8 == 0 required", kGemvMaxB);
  if (!r3g_aligned16(w)) return r3g_fail(ctx, R3G_E_INVALID, "gemv: the weight matrix must be 16-byte aligned");
  const int bt = B <= 1 ? 1 : B <= 2 ? 2 : B <= 4 ? 4 : 8;
  const size_t smem = (size_t)bt * K * sizeof(float);
  if (smem > 48 * 1024) return r3g_fail(ctx, R3G_E_INVALID, "gemv: B_pad * K * 4 bytes must fit 48 KB of shared memory");
  const unsigned grid = (unsigned)((N + 8 * kGemvRows - 1) / (8 * kGemvRows));
  auto args = [&](auto kern) {
    return r3g_launch_pdl(ctx, kern, dim3(grid), dim3(256), smem, (cudaStream_t)stream, (const __half*)w,
                          (const __half*)bias, (const __half*)vec, vec_ld, (__half*)out, out_ld, (const __half*)residual, B, N, K, silu_in,
                          silu_out);
  };
  R3G_CUDA_OK(ctx, bt == 1 ? args(gemv_kernel<1>) : bt == 2 ? args(gemv_kernel<2>) : bt == 4 ? args(gemv_kernel<4>)
                                                                                              : args(gemv_kernel<8>));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_timestep_embedding(r3g_ctx* ctx, const void* t_f16, void* out, int B, int dim, float time_factor,
                                      float max_period, void* stream) {
  R3G_ENTRY(ctx, "timestep_embedding");
  const int n = B * (dim / 2);
  timestep_embedding_kernel<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>((const __half*)t_f16, (__half*)out, B,
                                                                                 dim, time_factor, max_period);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_cfg_euler_step(r3g_ctx* ctx, void* x, const void* v, void* x_dup, int64_t n, int nb,
                                  float guidance, float dsigma, void* stream) {
  R3G_ENTRY(ctx, "cfg_euler_step");
  if (nb != 1 && nb != 2) return r3g_fail(ctx, R3G_E_INVALID, "cfg_euler_step: nb must be 1 or 2, got %d", nb);
  cfg_euler_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>((__half*)x, (const __half*)v,
                                                                                    (__half*)x_dup, n, nb, guidance,
                                                                                    dsigma);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_grid_fourier(r3g_ctx* ctx, void* out, int64_t out_ld, int64_t start, int64_t count, int R,
                                const float* bounds6_host, int num_freqs, int include_pi, void* stream) {
  R3G_ENTRY(ctx, "grid_fourier");
  if (!bounds6_host || R < 1 || out_ld < 3 + 6 * num_freqs)
    return r3g_fail(ctx, R3G_E_INVALID, "grid_fourier: bad arguments");
  GridParams gp;
  for (int d = 0; d < 3; ++d) {
    // bounds reach numpy as float64 (np.array of python floats, volume_decoders.py:159); the header
    // passes them as the float32 the caller holds, widened here.
    gp.lo[d] = (double)bounds6_host[d];
    gp.hi[d] = (double)bounds6_host[3 + d];
    gp.step[d] = (gp.hi[d] - gp.lo[d]) / (double)R;
  }
  gp.R = R;
  gp.num_freqs = num_freqs;
  gp.include_pi = include_pi;
  if (count <= 0) return R3G_OK;
  grid_fourier_kernel<<<(unsigned)((count + 255) / 256), 256, 0, (cudaStream_t)stream>>>((__half*)out, out_ld, start,
                                                                                           count, gp);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_points_fourier(r3g_ctx* ctx, const void* queries, void* out, int64_t out_ld, int64_t n,
                                  int num_freqs, int include_pi, void* stream) {
  R3G_ENTRY(ctx, "points_fourier");
  if (!queries || !out || out_ld < 3 + 6 * num_freqs) return r3g_fail(ctx, R3G_E_INVALID, "points_fourier: bad arguments");
  if (n <= 0) return R3G_OK;
  points_fourier_kernel<__half><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      (const __half*)queries, (__half*)out, out_ld, n, num_freqs, include_pi);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_swiglu(r3g_ctx* ctx, const void* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int F,
                          void* stream) {
  R3G_ENTRY(ctx, "swiglu");
  if (!x || !out || F < 8 || F % 8 || ldx % 8 || ldo % 8 || ldx < 2 * (int64_t)F || ldo < F || !r3g_aligned16(x) ||
      !r3g_aligned16(out))
    return r3g_fail(ctx, R3G_E_INVALID, "swiglu: F %% 8 == 0, ldx >= 2F, 16-byte aligned rows required");
  if (rows <= 0) return R3G_OK;
  const int64_t total = rows * (F / 8);
  const unsigned grid = (unsigned)min((total + 255) / 256, (int64_t)ctx->num_sms * 8);
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, swiglu_kernel, dim3(grid), dim3(256), 0, (cudaStream_t)stream, (const __half*)x, ldx,
                                   (__half*)out, ldo, rows, F));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_points_fourier_f32(r3g_ctx* ctx, const float* queries, void* out, int64_t out_ld, int64_t n,
                                      int num_freqs, int include_pi, void* stream) {
  R3G_ENTRY(ctx, "points_fourier_f32");
  if (!queries || !out || out_ld < 3 + 6 * num_freqs) return r3g_fail(ctx, R3G_E_INVALID, "points_fourier_f32: bad arguments");
  if (n <= 0) return R3G_OK;
  points_fourier_kernel<float><<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      queries, (__half*)out, out_ld, n, num_freqs, include_pi);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_lnpost_dot(r3g_ctx* ctx, const void* x, int64_t ldx, int rows, int width, float eps,
                              const void* ln_w, const void* ln_b, const void* w_out, const void* b_out, float* out,
                              void* stream) {
  R3G_ENTRY(ctx, "lnpost_dot");
  if (width % 8 || width > kLnMaxChunks * 256 || ldx % 8) return r3g_fail(ctx, R3G_E_INVALID, "lnpost_dot: width");
  if (!r3g_aligned16(x)) return r3g_fail(ctx, R3G_E_INVALID, "lnpost_dot: x must be 16-byte aligned");
  if (rows <= 0) return R3G_OK;
  const unsigned grid = (unsigned)min((rows + 7) / 8, ctx->num_sms * (width <= 1024 ? 3 : 2));
  auto go = [&](auto kern) {
    return r3g_launch_pdl(ctx, kern, dim3(grid), dim3(256), (size_t)3 * width * sizeof(float), (cudaStream_t)stream,
                          (const __half*)x, ldx, rows, width, eps, (const __half*)ln_w, (const __half*)ln_b,
                          (const __half*)w_out, (const __half*)b_out, out);
  };
  R3G_CUDA_OK(ctx, width <= 1024 ? go(lnpost_dot_kernel<4>) : go(lnpost_dot_kernel<8>));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

extern "C" int r3g_unproject(r3g_ctx* ctx, const float* depth, const double* cam_to_world_host,
                             const float* intrinsic_host, void* out, int S, int H, int W, int out_f64, void* stream) {
  R3G_ENTRY(ctx, "unproject");
  if (!depth || !cam_to_world_host || !intrinsic_host || !out || S < 1 || H < 1 || W < 1)
    return r3g_fail(ctx, R3G_E_INVALID, "unproject: bad arguments");
  const int64_t pairs = ((int64_t)H * W + 1) / 2;
  for (int s0 = 0; s0 < S; s0 += kMaxFrames) {
    const int ns = (S - s0) < kMaxFrames ? (S - s0) : kMaxFrames;
    UnprojectParams prm;
    for (int s = 0; s < ns; ++s) {
      const double* e = cam_to_world_host + 12 * (s0 + s);
      const float* k = intrinsic_host + 9 * (s0 + s);
      if (k[1] != 0.f || k[3] != 0.f) return r3g_fail(ctx, R3G_E_INVALID, "Intrinsic matrix must have zero skew");
      for (int i = 0; i < 3; ++i) {
        for (int j = 0; j < 3; ++j) prm.f[s].r[3 * i + j] = e[4 * i + j];
        prm.f[s].t[i] = e[4 * i + 3];
      }
      prm.f[s].fu = k[0]; prm.f[s].fv = k[4]; prm.f[s].cu = k[2]; prm.f[s].cv = k[5];
    }
    dim3 grid((unsigned)((pairs + 255) / 256), 1, ns);
    if (out_f64)
      unproject_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(depth, out, H, W, s0, prm);
    else
      unproject_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(depth, out, H, W, s0, prm);
    R3G_LAUNCH_OK(ctx);
  }
  return R3G_OK;
}
