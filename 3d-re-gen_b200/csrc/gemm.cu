// r3g_linear: Y = epilogue(X . W^T + bias) on the Hopper tensor cores (wgmma).
//
// Warp-specialised sm_90a kernel, one 128 x BN output tile per CTA:
//   warp 8      TMA producer   (cp.async.bulk.tensor, 128B-swizzled K-major tiles of X and W into a smem ring)
//   warps 0..7  two consumer warpgroups (wgmma.mma_async m64nBNk16, fp16 in, fp32 accumulators in registers; warpgroup
//               g computes rows [64 g, 64 g + 64) of the tile).  After the main loop the accumulators are staged as an
//               fp32 tile in the (then idle) operand ring and each of the 256 threads runs the epilogue for one row and
//               half of the columns: bias, GELU, gate*y+residual, fp16/fp32 conversion, 16-byte global stores.
// Covers every nn.Linear on the hot path: DiT qkv/proj/mlp/linear1/linear2 (hunyuan3ddit.py:196-216,259-267),
// ShapeVAE c_qkv/c_proj/c_fc (attention_blocks.py:166-182,345-363), geo-decoder query_proj/c_q/c_kv/c_proj/mlp
// (attention_blocks.py:250-261,484-494).
#include <cuda_fp16.h>
#include <string.h>

#include "r3g_internal.h"
#include "r3g_ptx.cuh"

namespace {

using namespace r3g;

constexpr int BM = 128;
constexpr int BK = 64;  // 64 halfs = one 128-byte swizzle row
constexpr int kNumEpilogueWarps = 8;   // the two consumer warpgroups; two warps per 32-row group, one per column half
constexpr int kNumThreads = 32 * kNumEpilogueWarps + 32;

struct LinearParams {
  int M, N, K;
  const __half* bias;
  void* y;
  int64_t ldy;
  int seg_len;            // rows per segment (== M when unsegmented)
  int64_t y_seg_stride;   // output rows between segment starts
  int tiles_per_seg;
  int act, act_col0, act_col1;
  const __half* gate;
  int64_t gate_ld;
  int gate_rows;
  const __half* residual;
  const float* residual_f32;  // fp32 residual stream (VGGT blocks): y_f32 = res_f32 + ls_gamma[n] * fp16(acc + bias)
  const float* ls_gamma;
  int out_f32;
  int tiles_m, tiles_n;
  // fused per-head q/k normalisation (0 off, 1 RMS, 2 LayerNorm) of the 64-column heads in two column ranges
  int qkn_mode, qkn_q_col0, qkn_k_col0, qkn_cols;
  float qkn_eps;
  const __half *qkn_q_w, *qkn_q_b, *qkn_k_w, *qkn_k_b;
};

__device__ __forceinline__ float rcpf(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// tanh-GELU: 0.5 x (1 + tanh(u)) == x * sigmoid(2u), u = sqrt(2/pi) (x + 0.044715 x^3).
// 5 FMA-pipe ops + 2 MUFU per element, accurate to ~1e-6 relative (well inside the fp16 output rounding).
__device__ __forceinline__ float gelu_tanh_f(float x) {
  constexpr float a = -2.f * 0.7978845608028654f * 1.4426950408889634f;  // -2 sqrt(2/pi) log2(e)
  constexpr float b = a * 0.044715f;
  const float t = x * x;
  const float z = x * fmaf(b, t, a);          // -2u log2(e)
  return x * rcpf(1.f + ex2_approx(z));
}
// erf-GELU: 0.5 x (1 + erf(x / sqrt 2)), erf by Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7).
__device__ __forceinline__ float gelu_erf_f(float x) {
  const float az = fabsf(x) * 0.7071067811865476f;
  const float t = rcpf(fmaf(0.3275911f, az, 1.f));
  float pl = fmaf(1.061405429f, t, -1.453152027f);
  pl = fmaf(pl, t, 1.421413741f);
  pl = fmaf(pl, t, -0.284496736f);
  pl = fmaf(pl, t, 0.254829592f);
  pl *= t;
  const float e = ex2_approx(az * az * -1.4426950408889634f);
  const float erf_abs = fmaf(-pl, e, 1.f);
  return 0.5f * x + 0.5f * fabsf(x) * erf_abs;   // x>0: 0.5x(1+erf), x<0: 0.5x(1-erf|.|)
}

// Epilogue operands.  An L2 round trip per 32-column chunk would stall the epilogue, so each epilogue warp stages its
// (at most 128-column) slice of the bias row and of the (at most two) gate rows its 32 rows can belong to in its own
// 768 bytes of shared memory before the main loop, and the fp16 residual -- the only per-thread operand -- is fetched
// one chunk ahead of its use.
constexpr int kEpiSmemPerWarp = 768;   // uint4 [0,16) bias, [16,32) gate row of lane 0's batch, [32,48) of lane 31's
template <int BN>
struct Cfg {
  static constexpr int kStageBytesA = BM * BK * 2;
  static constexpr int kStageBytesB = BN * BK * 2;
  static constexpr int kStageBytes = kStageBytesA + kStageBytesB;
  // 128-column tiles keep a 3-deep ring (96 KB) so that two CTAs share an SM and one's epilogue overlaps the other's
  // main loop; 256-column tiles (one CTA per SM) take a 4-deep ring.
  static constexpr int kStages = BN == 256 ? 4 : 3;
  static constexpr int kMinBlocks = BN == 256 ? 1 : 2;
  static constexpr int kLdStage = BN + 4;   // floats per row of the staged accumulator tile (16 B skew per row)
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/ +
                                    kNumEpilogueWarps * kEpiSmemPerWarp /*epilogue operand slices*/;
  static_assert(BM * kLdStage * 4 <= kStages * kStageBytes, "the staged accumulator tile must fit in the ring");
};

struct ChunkOperands {
  uint4 res[4];
};
__device__ __forceinline__ void prefetch_residual(const LinearParams& p, int64_t out_row, int n0, ChunkOperands& o) {
  if (p.residual) {
    const uint4* rp = reinterpret_cast<const uint4*>(p.residual + out_row * p.ldy + n0);
#pragma unroll
    for (int q = 0; q < 4; ++q) o.res[q] = rp[q];
  }
}
// stage this warp's bias / gate slices for the tile (columns [ncol0, ncol0 + ncols)); returns this lane's gate slice
// selector (0 / 1) or -1 when gates are read from global memory (gate_rows < 64: more than two batches per warp)
__device__ __forceinline__ int stage_tile_operands(const LinearParams& p, uint4* wsm, int lane, int ncol0, int ncols,
                                                   int r_lane0, int r_lane31, int r_mine) {
  __syncwarp();   // the previous tile's readers are done
  const bool in = lane < ncols / 8 && ncol0 + lane * 8 < p.N;
  int sel = -1;
  if (p.bias && in) wsm[lane] = __ldg(reinterpret_cast<const uint4*>(p.bias + ncol0) + lane);
  if (p.gate && p.gate_rows >= 64) {
    const int b_lo = r_lane0 / p.gate_rows, b_hi = r_lane31 / p.gate_rows;
    if (in) {
      wsm[16 + lane] = __ldg(reinterpret_cast<const uint4*>(p.gate + (int64_t)b_lo * p.gate_ld + ncol0) + lane);
      wsm[32 + lane] = __ldg(reinterpret_cast<const uint4*>(p.gate + (int64_t)b_hi * p.gate_ld + ncol0) + lane);
    }
    sel = r_mine / p.gate_rows - b_lo;
  }
  __syncwarp();
  return sel;
}

// One 32-column chunk of one accumulator row: v = fp32 accumulators of columns [n0, n0+32) of logical row r.
// sbias / sgate: this chunk's 4 uint4 of the staged slices (sgate NULL: gate from global memory or no gate);
// `pre` holds this chunk's residual and is refilled for chunk next_n0 (>= 0) as soon as it has been consumed.
__device__ __forceinline__ void epilogue_chunk(const LinearParams& p, const uint32_t* v, int r, int64_t out_row,
                                               int n0, const uint4* sbias, const uint4* sgate, const __half* gate_row,
                                               ChunkOperands& pre, int next_n0) {
    float f[32];
#pragma unroll
    for (int j = 0; j < 32; ++j) f[j] = __uint_as_float(v[j]);
    if (p.bias) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 b4 = sbias[q];
        const __half2* h = reinterpret_cast<const __half2*>(&b4);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 t = __half22float2(h[j]);
          f[q * 8 + 2 * j] += t.x;
          f[q * 8 + 2 * j + 1] += t.y;
        }
      }
    }
    // act_col0 / act_col1 are multiples of 32 (checked at the API), so a 32-column chunk is activated as a whole:
    // one warp-uniform branch, then 32 independent element chains (per-element range checks serialise the MUFU chains)
    if (p.act && n0 >= p.act_col0 && n0 < p.act_col1) {
      if (p.act == 1) {
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] = gelu_tanh_f(__half2float(__float2half_rn(f[j])));  // Linear output is fp16
      } else if (p.act == 3) {   // ReLU (the DPT head's convolutions, dpt_head.py:344-392)
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] = fmaxf(f[j], 0.f);
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) f[j] = gelu_erf_f(__half2float(__float2half_rn(f[j])));
      }
    }
    if (p.residual) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const uint4 r4 = pre.res[q];
        const __half2* h = reinterpret_cast<const __half2*>(&r4);
        uint4 g4 = make_uint4(0, 0, 0, 0);
        if (sgate) g4 = sgate[q];
        else if (gate_row) g4 = __ldg(reinterpret_cast<const uint4*>(gate_row + n0) + q);
        const __half2* gh = reinterpret_cast<const __half2*>(&g4);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float2 rr = __half22float2(h[j]);
          float y0 = __half2float(__float2half_rn(f[q * 8 + 2 * j]));
          float y1 = __half2float(__float2half_rn(f[q * 8 + 2 * j + 1]));
          if (gate_row) {
            float2 gg = __half22float2(gh[j]);
            y0 = __half2float(__float2half_rn(gg.x * y0));
            y1 = __half2float(__float2half_rn(gg.y * y1));
          }
          f[q * 8 + 2 * j] = rr.x + y0;
          f[q * 8 + 2 * j + 1] = rr.y + y1;
        }
      }
      if (next_n0 >= 0) prefetch_residual(p, out_row, next_n0, pre);
    }
    if (p.residual_f32) {
      const float4* rp = reinterpret_cast<const float4*>(p.residual_f32 + out_row * p.ldy + n0);
      const float4* gp = reinterpret_cast<const float4*>(p.ls_gamma + n0);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const float4 r4 = rp[q];
        float4 g4 = make_float4(1.f, 1.f, 1.f, 1.f);
        if (p.ls_gamma) g4 = __ldg(gp + q);
        f[4 * q + 0] = r4.x + g4.x * __half2float(__float2half_rn(f[4 * q + 0]));
        f[4 * q + 1] = r4.y + g4.y * __half2float(__float2half_rn(f[4 * q + 1]));
        f[4 * q + 2] = r4.z + g4.z * __half2float(__float2half_rn(f[4 * q + 2]));
        f[4 * q + 3] = r4.w + g4.w * __half2float(__float2half_rn(f[4 * q + 3]));
      }
    }
    if (p.out_f32) {
      float4* op = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.y) + out_row * p.ldy + n0);
#pragma unroll
      for (int q = 0; q < 8; ++q) op[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
    } else {
      uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.y) + out_row * p.ldy + n0);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        uint4 o;
        o.x = pack_half2(f[8 * q + 0], f[8 * q + 1]);
        o.y = pack_half2(f[8 * q + 2], f[8 * q + 3]);
        o.z = pack_half2(f[8 * q + 4], f[8 * q + 5]);
        o.w = pack_half2(f[8 * q + 6], f[8 * q + 7]);
        op[q] = o;
      }
    }

}

// One 64-column head of one accumulator row with the q/k normalisation fused (qkn_mode): v0 / v1 = the two 32-column
// accumulator chunks of columns [n0, n0+64).  Same arithmetic as qk_norm_kernel (rowops.cu): the Linear output is an
// fp16 tensor, the statistics are fp32, RMS: (x * rrms).to(fp16) * scale; LayerNorm: (x - mean) * rstd * w + b.
__device__ __forceinline__ void epilogue_qknorm(const LinearParams& p, const uint32_t* v0, const uint32_t* v1,
                                                int64_t out_row, int n0, const __half* nw, const __half* nb,
                                                const uint4* sbias8) {
  float f[64];
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    f[j] = __uint_as_float(v0[j]);
    f[32 + j] = __uint_as_float(v1[j]);
  }
  if (p.bias) {
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 b4 = sbias8[q];
      const __half2* h = reinterpret_cast<const __half2*>(&b4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 t = __half22float2(h[j]);
        f[q * 8 + 2 * j] += t.x;
        f[q * 8 + 2 * j + 1] += t.y;
      }
    }
  }
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
  for (int j = 0; j < 64; j += 4) {
    f[j] = __half2float(__float2half_rn(f[j]));
    f[j + 1] = __half2float(__float2half_rn(f[j + 1]));
    f[j + 2] = __half2float(__float2half_rn(f[j + 2]));
    f[j + 3] = __half2float(__float2half_rn(f[j + 3]));
    if (p.qkn_mode == 1) {
      s0 = fmaf(f[j], f[j], s0); s1 = fmaf(f[j + 1], f[j + 1], s1);
      s2 = fmaf(f[j + 2], f[j + 2], s2); s3 = fmaf(f[j + 3], f[j + 3], s3);
    } else {
      s0 += f[j]; s1 += f[j + 1]; s2 += f[j + 2]; s3 += f[j + 3];
    }
  }
  if (p.qkn_mode == 1) {
    const float rrms = rsqrtf(((s0 + s1) + (s2 + s3)) * (1.f / 64.f) + p.qkn_eps);
    const uint4* wp = reinterpret_cast<const uint4*>(nw);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 w4 = __ldg(wp + q);
      const __half2* h = reinterpret_cast<const __half2*>(&w4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 t = __half22float2(h[j]);
        f[q * 8 + 2 * j] = __half2float(__float2half_rn(f[q * 8 + 2 * j] * rrms)) * t.x;
        f[q * 8 + 2 * j + 1] = __half2float(__float2half_rn(f[q * 8 + 2 * j + 1] * rrms)) * t.y;
      }
    }
  } else {
    const float mean = ((s0 + s1) + (s2 + s3)) * (1.f / 64.f);
    float q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
#pragma unroll
    for (int j = 0; j < 64; j += 4) {
      f[j] -= mean; f[j + 1] -= mean; f[j + 2] -= mean; f[j + 3] -= mean;
      q0 = fmaf(f[j], f[j], q0); q1 = fmaf(f[j + 1], f[j + 1], q1);
      q2 = fmaf(f[j + 2], f[j + 2], q2); q3 = fmaf(f[j + 3], f[j + 3], q3);
    }
    const float rstd = rsqrtf(((q0 + q1) + (q2 + q3)) * (1.f / 64.f) + p.qkn_eps);
    const uint4* wp = reinterpret_cast<const uint4*>(nw);
    const uint4* bp = reinterpret_cast<const uint4*>(nb);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint4 w4 = __ldg(wp + q);
      uint4 b4 = make_uint4(0, 0, 0, 0);
      if (nb) b4 = __ldg(bp + q);
      const __half2* hw = reinterpret_cast<const __half2*>(&w4);
      const __half2* hb = reinterpret_cast<const __half2*>(&b4);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 tw = __half22float2(hw[j]), tb = __half22float2(hb[j]);
        f[q * 8 + 2 * j] = f[q * 8 + 2 * j] * rstd * tw.x + tb.x;
        f[q * 8 + 2 * j + 1] = f[q * 8 + 2 * j + 1] * rstd * tw.y + tb.y;
      }
    }
  }
  uint4* op = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.y) + out_row * p.ldy + n0);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    uint4 o;
    o.x = pack_half2(f[8 * q + 0], f[8 * q + 1]);
    o.y = pack_half2(f[8 * q + 2], f[8 * q + 3]);
    o.z = pack_half2(f[8 * q + 4], f[8 * q + 5]);
    o.w = pack_half2(f[8 * q + 6], f[8 * q + 7]);
    op[q] = o;
  }
}

// which normalisation range (0 = q, 1 = k, -1 = none) the 64-column group starting at n0 belongs to
__device__ __forceinline__ int qkn_range(const LinearParams& p, int n0) {
  if (!p.qkn_mode) return -1;
  if (n0 >= p.qkn_q_col0 && n0 < p.qkn_q_col0 + p.qkn_cols) return 0;
  if (p.qkn_k_col0 >= 0 && n0 >= p.qkn_k_col0 && n0 < p.qkn_k_col0 + p.qkn_cols) return 1;
  return -1;
}

template <int BN>
__device__ __forceinline__ void wgmma_tile(float* acc, uint64_t da, uint64_t db) {
  if constexpr (BN == 256) wgmma_m64n256k16_ss(acc, da, db, 1u);
  else wgmma_m64n128k16_ss(acc, da, db, 1u);
}

template <int BN>
__global__ void __launch_bounds__(kNumThreads, Cfg<BN>::kMinBlocks)
linear_kernel(const __grid_constant__ CUtensorMap tmap_x0, const __grid_constant__ CUtensorMap tmap_w0,
              const __grid_constant__ CUtensorMap tmap_x1, const __grid_constant__ CUtensorMap tmap_w1,
              const __grid_constant__ LinearParams p0, const __grid_constant__ LinearParams p1) {
  // Two problems may share one launch (r3g_linear_args.group_next: the img and txt streams of a DoubleStreamBlock):
  // tiles [0, tiles0) belong to p0, the rest to p1 (p1.tiles_m == 0: no second problem).
  using C = Cfg<BN>;
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment is required by the 128B swizzle atoms
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::kStages * C::kStageBytes);
  uint64_t* empty_bar = full_bar + C::kStages;
  uint8_t* epi_smem = smem + C::kStages * C::kStageBytes + 256;   // per-epilogue-warp operand slices
  float* acc_smem = reinterpret_cast<float*>(smem);               // the staged accumulator tile (after the main loop)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles0 = p0.tiles_m * p0.tiles_n;
  const int tile = blockIdx.x;
  const bool second = tile >= tiles0;
  const LinearParams& p = second ? p1 : p0;
  const int lt = second ? tile - tiles0 : tile;
  const int tm = lt / p.tiles_n, tn = lt % p.tiles_n;
  const int sg = tm / p.tiles_per_seg;
  const int num_k_blocks = (p.K + BK - 1) / BK;

  if (warp == kNumEpilogueWarps && lane == 0) {
    tma_prefetch_desc(second ? &tmap_x1 : &tmap_x0);
    tma_prefetch_desc(second ? &tmap_w1 : &tmap_w0);
    for (int s = 0; s < C::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 32 * kNumEpilogueWarps);   // every consumer thread releases the slot
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // everything above overlapped the previous kernel's tail; its results are visible from here on

  if (warp == kNumEpilogueWarps) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      const CUtensorMap* tmap_x = second ? &tmap_x1 : &tmap_x0;
      const CUtensorMap* tmap_w = second ? &tmap_w1 : &tmap_w0;
      const int l0 = (tm % p.tiles_per_seg) * BM;
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        uint8_t* sa = smem + stage * C::kStageBytes;
        uint8_t* sb = sa + C::kStageBytesA;
        mbar_expect_tx(&full_bar[stage], C::kStageBytes);
        tma_load_3d(sa, tmap_x, &full_bar[stage], kb * BK, l0, sg, kEvictFirst);
        tma_load_2d(sb, tmap_w, &full_bar[stage], kb * BK, tn * BN, kEvictLast);
        if (++stage == C::kStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers (warps 0..7)
  const int wg = warp >> 2;                     // warpgroup: MMA rows [64 wg, 64 wg + 64)
  uint4* wsm = reinterpret_cast<uint4*>(epi_smem + warp * kEpiSmemPerWarp);
  // stage the warp's bias / gate slices before the main loop: the loads land while the tensor cores work.  The
  // row-derived epilogue values are recomputed after the loop instead of being held in registers across it.
  int gsel = -1;
  {
    const int row_in_tile = threadIdx.x & (BM - 1), col_half = threadIdx.x >> 7;
    const int l = (tm % p.tiles_per_seg) * BM + row_in_tile;
    const int l0 = l - lane, l31 = min(l0 + 31, p.seg_len - 1);
    if (l0 < p.seg_len)
      gsel = stage_tile_operands(p, wsm, lane, tn * BN + col_half * (BN / 2), BN / 2, sg * p.seg_len + l0,
                                 sg * p.seg_len + l31, l < p.seg_len ? sg * p.seg_len + l : sg * p.seg_len + l31);
  }

  {
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int kb = 0; kb < num_k_blocks; ++kb) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * C::kStageBytes) + wg * 64 * 128;
      const uint32_t sb = smem_u32(smem + stage * C::kStageBytes + C::kStageBytesA);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k)
        wgmma_tile<BN>(acc, gmma_desc_sw128(sa + k * 32, 1024, 16), gmma_desc_sw128(sb + k * 32, 1024, 16));
      wgmma_commit();
      wgmma_wait<1>();   // the previous k-block's MMAs have retired: its slot goes back to the producer
      if (kb > 0) mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == C::kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_reg_fence<BN / 2>(acc);
    named_bar_sync(1, 32 * kNumEpilogueWarps);   // both warpgroups are done reading the ring
    const int w4 = warp & 3;
#pragma unroll
    for (int i = 0; i < BN / 2; i += 2) {
      const int row = wg * 64 + w4 * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
      const int col = 8 * (i >> 2) + 2 * (lane & 3);
      *reinterpret_cast<float2*>(acc_smem + row * C::kLdStage + col) = make_float2(acc[i], acc[i + 1]);
    }
    named_bar_sync(1, 32 * kNumEpilogueWarps);
  }

  // -------------------------------------------------------------------- epilogue: one row, half of the columns
  const int row_in_tile = threadIdx.x & (BM - 1);   // epilogue row
  const int col_half = threadIdx.x >> 7;        // which half of the tile's columns this thread's epilogue owns
  const int l = (tm % p.tiles_per_seg) * BM + row_in_tile;  // row inside the segment
  const bool row_ok = l < p.seg_len;
  const int r = sg * p.seg_len + l;                          // logical row
  const int64_t out_row = (int64_t)sg * p.y_seg_stride + l;
  const __half* gate_row = p.gate ? p.gate + (int64_t)(row_ok ? r / p.gate_rows : 0) * p.gate_ld : nullptr;
  const float* srow = acc_smem + row_in_tile * C::kLdStage;
  ChunkOperands pre;
  bool have_pre = false;
#pragma unroll 1
  for (int c0 = col_half * (BN / 2); c0 < (col_half + 1) * (BN / 2); c0 += 32) {
    const int n0 = tn * BN + c0;
    if (n0 >= p.N) break;  // warp-uniform
    const uint4* sbias = wsm + ((c0 - col_half * (BN / 2)) >> 3);
    const uint32_t* v = reinterpret_cast<const uint32_t*>(srow + c0);
    const int nr = ((c0 & 32) == 0) ? qkn_range(p, n0) : -1;   // warp-uniform
    if (nr >= 0) {
      if (row_ok)
        epilogue_qknorm(p, v, v + 32, out_row, n0, nr ? p.qkn_k_w : p.qkn_q_w, nr ? p.qkn_k_b : p.qkn_q_b, sbias);
      c0 += 32;
      have_pre = false;
      continue;
    }
    if (!have_pre && row_ok) prefetch_residual(p, out_row, n0, pre);
    const int c1 = c0 + 32;   // the next chunk of this thread's column half, if it is an ordinary one
    const bool more = c1 < (col_half + 1) * (BN / 2) && tn * BN + c1 < p.N &&
                      !((c1 & 32) == 0 && qkn_range(p, tn * BN + c1) >= 0);
    if (row_ok)
      epilogue_chunk(p, v, r, out_row, n0, sbias, gsel >= 0 ? sbias + 16 + 16 * gsel : nullptr, gate_row, pre,
                     more ? tn * BN + c1 : -1);
    have_pre = more;
  }
}

// One problem of a launch: tensor maps + kernel parameters.  tile_m = rows per tile, box_n = rows of W one CTA fetches
// per k-block, bn = output columns per tile.
struct Problem {
  LinearParams p;
  CUtensorMap tx, tw;
};

int make_problem(r3g_ctx* ctx, const r3g_linear_args* a, int tile_m, int box_n, int bn, Problem& out) {
  LinearParams& p = out.p;
  memset(&p, 0, sizeof(p));
  if (!a) return R3G_OK;   // no second problem: tiles_m = 0
  const int seg_len = a->seg_len > 0 ? a->seg_len : a->M;
  const int nseg = a->M / seg_len;
  {
    const uint64_t dims[3] = {(uint64_t)a->K, (uint64_t)seg_len, (uint64_t)nseg};
    const uint64_t strides[3] = {2, (uint64_t)a->ldx * 2, (uint64_t)(nseg > 1 ? a->x_seg_stride : seg_len) * a->ldx * 2};
    const uint32_t box[3] = {BK, BM, 1};
    int rc = r3g_make_tmap_f16(ctx, &out.tx, a->x, 3, dims, strides, box);
    if (rc) return rc;
  }
  {
    const uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N};
    const uint64_t strides[2] = {2, (uint64_t)a->K * 2};
    const uint32_t box[2] = {BK, (uint32_t)box_n};
    int rc = r3g_make_tmap_f16(ctx, &out.tw, a->w, 2, dims, strides, box);
    if (rc) return rc;
  }
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.bias = (const __half*)a->bias;
  p.y = a->y; p.ldy = a->ldy;
  p.seg_len = seg_len;
  p.y_seg_stride = nseg > 1 ? a->y_seg_stride : seg_len;
  p.tiles_per_seg = (seg_len + tile_m - 1) / tile_m;
  p.act = a->act; p.act_col0 = a->act_col0; p.act_col1 = a->act_col1;
  p.gate = (const __half*)a->gate; p.gate_ld = a->gate_ld; p.gate_rows = a->gate_rows > 0 ? a->gate_rows : 1;
  p.residual = a->residual_f32 ? nullptr : (const __half*)a->residual;
  p.residual_f32 = a->residual_f32 ? (const float*)a->residual : nullptr;
  p.ls_gamma = (const float*)a->ls_gamma;
  p.out_f32 = a->out_f32;
  p.qkn_mode = a->qkn_mode; p.qkn_q_col0 = a->qkn_q_col0; p.qkn_k_col0 = a->qkn_k_col0; p.qkn_cols = a->qkn_cols;
  p.qkn_eps = a->qkn_eps;
  p.qkn_q_w = (const __half*)a->qkn_q_w; p.qkn_q_b = (const __half*)a->qkn_q_b;
  p.qkn_k_w = (const __half*)a->qkn_k_w; p.qkn_k_b = (const __half*)a->qkn_k_b;
  p.tiles_m = nseg * p.tiles_per_seg;
  p.tiles_n = (a->N + bn - 1) / bn;
  return R3G_OK;
}

template <int BN>
int launch_linear(r3g_ctx* ctx, const r3g_linear_args* a, const r3g_linear_args* b, cudaStream_t s) {
  using C = Cfg<BN>;
  Problem pa, pb;
  int rc = make_problem(ctx, a, BM, BN, BN, pa);
  if (rc) return rc;
  rc = make_problem(ctx, b, BM, BN, BN, pb);
  if (rc) return rc;
  if (!b) { pb.tx = pa.tx; pb.tw = pa.tw; }
  constexpr unsigned kAttrBit = BN == 256 ? R3G_ATTR_LINEAR256 : R3G_ATTR_LINEAR128;
  if (!(ctx->attr_done & kAttrBit)) {
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(linear_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          C::kSmemBytes));
    ctx->attr_done |= kAttrBit;
  }
  const int tiles = pa.p.tiles_m * pa.p.tiles_n + pb.p.tiles_m * pb.p.tiles_n;
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, linear_kernel<BN>, dim3(tiles), dim3(kNumThreads), C::kSmemBytes, s, pa.tx, pa.tw,
                                   pb.tx, pb.tw, pa.p, pb.p));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

int validate_linear(r3g_ctx* ctx, const r3g_linear_args* a) {
  if (!a->x || !a->w || !a->y) return r3g_fail(ctx, R3G_E_INVALID, "linear: null argument");
  if (a->N % 32 || a->K % 8 || a->ldx % 8 || a->ldy % 8)
    return r3g_fail(ctx, R3G_E_INVALID, "linear: need N %% 32 == 0, K %% 8 == 0, ldx/ldy %% 8 == 0 (N=%d K=%d)", a->N,
                    a->K);
  if (a->seg_len > 0 && a->M % a->seg_len) return r3g_fail(ctx, R3G_E_INVALID, "linear: M must be a multiple of seg_len");
  if (a->residual && (a->out_f32 != 0) != (a->residual_f32 != 0))
    return r3g_fail(ctx, R3G_E_INVALID, "linear: an fp32 output takes an fp32 residual (residual_f32=1) and vice versa");
  if (a->ls_gamma && !a->residual_f32) return r3g_fail(ctx, R3G_E_INVALID, "linear: ls_gamma needs the fp32 residual form");
  if (a->gate && (!a->residual || a->gate_ld % 8)) return r3g_fail(ctx, R3G_E_INVALID, "linear: gate needs residual");
  if (a->act && (a->act_col0 % 32 || a->act_col1 % 32))
    return r3g_fail(ctx, R3G_E_INVALID, "linear: activation column range must be aligned to 32 columns");
  if (a->qkn_mode) {
    const bool k_on = a->qkn_k_col0 >= 0;
    if (a->qkn_mode < 0 || a->qkn_mode > 2 || a->N < 128 || a->qkn_cols <= 0 || a->qkn_cols % 64 || a->qkn_q_col0 % 64 ||
        (k_on && a->qkn_k_col0 % 64) || a->qkn_q_col0 < 0 || a->qkn_q_col0 + a->qkn_cols > a->N ||
        (k_on && a->qkn_k_col0 + a->qkn_cols > a->N) || !a->qkn_q_w || (k_on && !a->qkn_k_w))
      return r3g_fail(ctx, R3G_E_INVALID, "linear: qkn ranges must be 64-column aligned inside [0, N), N >= 128, weights set");
    if (a->residual || a->out_f32)
      return r3g_fail(ctx, R3G_E_INVALID, "linear: the fused q/k normalisation takes a plain fp16 output (no residual)");
    auto overlaps = [&](int c0) { return a->act && c0 < a->act_col1 && c0 + a->qkn_cols > a->act_col0; };
    if (overlaps(a->qkn_q_col0) || (k_on && overlaps(a->qkn_k_col0)))
      return r3g_fail(ctx, R3G_E_INVALID, "linear: normalised columns must lie outside the activation range");
  }
  return R3G_OK;
}

}  // namespace

extern "C" int r3g_linear(r3g_ctx* ctx, const r3g_linear_args* a, void* stream) {
  R3G_ENTRY(ctx, "linear");
  if (!a) return r3g_fail(ctx, R3G_E_INVALID, "linear: null argument");
  const r3g_linear_args* b = (const r3g_linear_args*)a->group_next;
  if (b && b->group_next) return r3g_fail(ctx, R3G_E_INVALID, "linear: at most two problems per launch");
  if (a->M <= 0) { a = b; b = nullptr; }
  if (b && b->M <= 0) b = nullptr;
  if (!a) return R3G_OK;
  int rc = validate_linear(ctx, a);
  if (rc) return rc;
  if (b && (rc = validate_linear(ctx, b))) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  // Tile choice: wave efficiency (tiles / (waves * resident CTAs)) over the tiles of BOTH problems of a grouped launch.
  // A 128 x 256 tile reads half the operand bytes per FLOP of a 128 x 128 one but runs one CTA per SM instead of
  // two; it is taken unless it leaves more of the last wave idle.
  const int sms = ctx->num_sms;
  auto eff = [&](int64_t tiles, int units) {
    if (tiles <= 0) return 0.0;
    const int64_t waves = (tiles + units - 1) / units;
    return (double)tiles / (double)(waves * units);
  };
  auto tiles_of = [&](const r3g_linear_args* q, int tm, int tn) -> int64_t {
    if (!q) return 0;
    const int seg = q->seg_len > 0 ? q->seg_len : q->M;
    return (int64_t)(q->M / seg) * ((seg + tm - 1) / tm) * ((q->N + tn - 1) / tn);
  };
  const int n_min = b ? (a->N < b->N ? a->N : b->N) : a->N;
  const double e256 = n_min >= 256 ? eff(tiles_of(a, BM, 256) + tiles_of(b, BM, 256), sms) : 0.0;
  const double e128 = eff(tiles_of(a, BM, 128) + tiles_of(b, BM, 128), 2 * sms);
  if (e256 > 0.0 && e256 >= e128) return launch_linear<256>(ctx, a, b, s);
  return launch_linear<128>(ctx, a, b, s);
}
