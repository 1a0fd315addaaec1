// r3g_linear: Y = epilogue(X . W^T + bias) on the Hopper tensor cores (wgmma).
//
// Warp-specialised sm_90a kernel, one 128 x BN output tile per CTA:
//   warp 8      TMA producer   (cp.async.bulk.tensor, 128B-swizzled K-major tiles of X and W into a smem ring)
//   warps 0..7  two consumer warpgroups (wgmma.mma_async m64nBNk16, fp16 in, fp32 accumulators in registers; warpgroup
//               g computes rows [64 g, 64 g + 64) of the tile).  After the main loop the accumulators are staged as an
//               fp32 tile in the (then idle) operand ring and each of the 256 threads runs the epilogue for one row and
//               half of the columns: bias, GELU, gate*y+residual, fp16/fp32 conversion, written back over its staged
//               row; each warp then stores its 32 rows x BN/2 columns as coalesced 16-byte accesses.
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
// The result overwrites the chunk's own staged accumulators (fp16: the first 64 of its 128 bytes, fp32: all of them);
// store_rows() moves it to global memory.
__device__ __forceinline__ void epilogue_chunk(const LinearParams& p, const uint32_t* v, int r, int64_t out_row,
                                               int n0, const uint4* sbias, const uint4* sgate, const __half* gate_row,
                                               ChunkOperands& pre, int next_n0, uint4* sout) {
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
      float4* op = reinterpret_cast<float4*>(sout);
#pragma unroll
      for (int q = 0; q < 8; ++q) op[q] = make_float4(f[4 * q], f[4 * q + 1], f[4 * q + 2], f[4 * q + 3]);
    } else {
      uint4* op = sout;
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
// The result overwrites the staged accumulators like epilogue_chunk's: each 32-column half at the start of its chunk
// (sout: the first chunk's 128 bytes, the second's follow).
__device__ __forceinline__ void epilogue_qknorm(const LinearParams& p, const uint32_t* v0, const uint32_t* v1,
                                                const __half* nw, const __half* nb, const uint4* sbias8, uint4* sout) {
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
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    uint4 o;
    o.x = pack_half2(f[8 * q + 0], f[8 * q + 1]);
    o.y = pack_half2(f[8 * q + 2], f[8 * q + 3]);
    o.z = pack_half2(f[8 * q + 4], f[8 * q + 5]);
    o.w = pack_half2(f[8 * q + 6], f[8 * q + 7]);
    sout[q + (q & 4)] = o;
  }
}

// Global stores of one epilogue warp's region: the 32 rows of the tile starting at segment row l0 (rows at or past
// seg_len are skipped), columns [n_start, n_start + ncols) (ncols <= 128, a multiple of 32).  srow0 points at the first
// row's staged results: each 32-column chunk's fp16 output in the first 64 of its 128 bytes, fp32 output filling them.
// A thread's epilogue owns a row, so a direct store would touch 32 rows per instruction; here 16 (fp16) or 32 (fp32)
// lanes write 256 or 512 contiguous bytes of one row.
template <int LD>
__device__ __forceinline__ void store_rows(const LinearParams& p, const float* srow0, int lane, int l0, int sg,
                                           int n_start, int ncols) {
  __syncwarp();   // every lane's results are in shared memory
  const int64_t row0 = (int64_t)sg * p.y_seg_stride + l0;
  if (p.out_f32) {
#pragma unroll 4
    for (int i = 0; i < 32; ++i) {
      if (l0 + i < p.seg_len && lane * 4 < ncols)
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.y) + (row0 + i) * p.ldy + n_start + lane * 4) =
            *reinterpret_cast<const float4*>(srow0 + i * LD + lane * 4);
    }
  } else {
    const int j = lane & 15;   // 16-byte piece of the row: chunk j / 4, bytes 16 (j % 4) of its fp16 output
#pragma unroll 4
    for (int i = lane >> 4; i < 32; i += 2) {
      if (l0 + i < p.seg_len && j * 8 < ncols)
        *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(p.y) + (row0 + i) * p.ldy + n_start + j * 8) =
            *reinterpret_cast<const uint4*>(srow0 + i * LD + 32 * (j >> 2) + 4 * (j & 3));
    }
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

// The operand ring, shared by linear_kernel and moe_gemm_kernel so that a row's accumulators are the same in both:
// Cfg<BN>::kStages slots of one BM x BK tile of X and one BN x BK tile of W at the 1024-aligned smem, followed by the
// slots' full / empty barriers.  ring_init (one thread) runs before the __syncthreads that publishes the barriers.
template <int BN>
__device__ __forceinline__ void ring_init(const CUtensorMap* tmap_x, const CUtensorMap* tmap_w, uint64_t* full_bar,
                                          uint64_t* empty_bar) {
  tma_prefetch_desc(tmap_x);
  tma_prefetch_desc(tmap_w);
  for (int s = 0; s < Cfg<BN>::kStages; ++s) {
    mbar_init(&full_bar[s], 1);
    mbar_init(&empty_bar[s], 32 * kNumEpilogueWarps);   // every consumer thread releases the slot
  }
  fence_barrier_init();
}

// TMA producer (one thread): every k-block of the tile's X rows [x_row, x_row + BM) of segment x_seg and W rows
// [w_row, w_row + BN), each into the next free slot
template <int BN>
__device__ __forceinline__ void ring_produce(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             const CUtensorMap* tmap_x, const CUtensorMap* tmap_w, int x_row,
                                             int x_seg, int w_row, int num_k_blocks) {
  using C = Cfg<BN>;
  int stage = 0;
  uint32_t phase = 0;
  for (int kb = 0; kb < num_k_blocks; ++kb) {
    mbar_wait(&empty_bar[stage], phase ^ 1);
    uint8_t* sa = smem + stage * C::kStageBytes;
    uint8_t* sb = sa + C::kStageBytesA;
    mbar_expect_tx(&full_bar[stage], C::kStageBytes);
    tma_load_3d(sa, tmap_x, &full_bar[stage], kb * BK, x_row, x_seg, kEvictFirst);
    tma_load_2d(sb, tmap_w, &full_bar[stage], kb * BK, w_row, kEvictLast);
    if (++stage == C::kStages) { stage = 0; phase ^= 1; }
  }
}

// Consumers (warps 0..7, warpgroup g: MMA rows [64 g, 64 g + 64)): the main loop over the ring, then the fp32
// accumulator tile staged row-major (Cfg<BN>::kLdStage floats per row) over the ring, visible to all 256 threads
template <int BN>
__device__ __forceinline__ void ring_consume(uint8_t* smem, uint64_t* full_bar, uint64_t* empty_bar,
                                             int num_k_blocks, int warp, int lane) {
  using C = Cfg<BN>;
  const int wg = warp >> 2;
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
  float* acc_smem = reinterpret_cast<float*>(smem);
  const int w4 = warp & 3;
#pragma unroll
  for (int i = 0; i < BN / 2; i += 2) {
    const int row = wg * 64 + w4 * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);
    const int col = 8 * (i >> 2) + 2 * (lane & 3);
    *reinterpret_cast<float2*>(acc_smem + row * C::kLdStage + col) = make_float2(acc[i], acc[i + 1]);
  }
  named_bar_sync(1, 32 * kNumEpilogueWarps);
}

template <int BN>
__global__ void __launch_bounds__(kNumThreads, Cfg<BN>::kMinBlocks)
linear_kernel(const __grid_constant__ CUtensorMap tmap_x0, const __grid_constant__ CUtensorMap tmap_w0,
              const __grid_constant__ CUtensorMap tmap_x1, const __grid_constant__ CUtensorMap tmap_w1,
              const __grid_constant__ CUtensorMap tmap_x2, const __grid_constant__ CUtensorMap tmap_w2,
              const __grid_constant__ LinearParams p0, const __grid_constant__ LinearParams p1,
              const __grid_constant__ LinearParams p2) {
  // Up to three problems share one launch (r3g_linear_args.group_next: the img and txt streams of a DoubleStreamBlock,
  // the txt stream possibly split by batch): tiles [0, tiles0) belong to p0, [tiles0, tiles01) to p1, the rest to p2
  // (tiles_m == 0: no such problem).
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
  const int tiles01 = tiles0 + p1.tiles_m * p1.tiles_n;
  const int tile = blockIdx.x;
  const int which = tile >= tiles01 ? 2 : tile >= tiles0 ? 1 : 0;
  const LinearParams& p = which == 2 ? p2 : which == 1 ? p1 : p0;
  const int lt = tile - (which == 2 ? tiles01 : which == 1 ? tiles0 : 0);
  const int tm = lt / p.tiles_n, tn = lt % p.tiles_n;
  const int sg = tm / p.tiles_per_seg;
  const int num_k_blocks = (p.K + BK - 1) / BK;
  const CUtensorMap* tmap_x = which == 2 ? &tmap_x2 : which == 1 ? &tmap_x1 : &tmap_x0;
  const CUtensorMap* tmap_w = which == 2 ? &tmap_w2 : which == 1 ? &tmap_w1 : &tmap_w0;

  if (warp == kNumEpilogueWarps && lane == 0) ring_init<BN>(tmap_x, tmap_w, full_bar, empty_bar);
  __syncthreads();
  pdl_wait();   // everything above overlapped the previous kernel's tail; its results are visible from here on

  if (warp == kNumEpilogueWarps) {
    if (lane == 0)
      ring_produce<BN>(smem, full_bar, empty_bar, tmap_x, tmap_w, (tm % p.tiles_per_seg) * BM, sg, tn * BN,
                       num_k_blocks);
    return;
  }

  // -------------------------------------------------------------------- consumers (warps 0..7)
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

  ring_consume<BN>(smem, full_bar, empty_bar, num_k_blocks, warp, lane);

  // -------------------------------------------------------------------- epilogue: one row, half of the columns
  const int row_in_tile = threadIdx.x & (BM - 1);   // epilogue row
  const int col_half = threadIdx.x >> 7;        // which half of the tile's columns this thread's epilogue owns
  const int l = (tm % p.tiles_per_seg) * BM + row_in_tile;  // row inside the segment
  const bool row_ok = l < p.seg_len;
  const int r = sg * p.seg_len + l;                          // logical row
  const int64_t out_row = (int64_t)sg * p.y_seg_stride + l;
  const __half* gate_row = p.gate ? p.gate + (int64_t)(row_ok ? r / p.gate_rows : 0) * p.gate_ld : nullptr;
  float* srow = acc_smem + row_in_tile * C::kLdStage;
  ChunkOperands pre;
  bool have_pre = false;
#pragma unroll 1
  for (int c0 = col_half * (BN / 2); c0 < (col_half + 1) * (BN / 2); c0 += 32) {
    const int n0 = tn * BN + c0;
    if (n0 >= p.N) break;  // warp-uniform
    const uint4* sbias = wsm + ((c0 - col_half * (BN / 2)) >> 3);
    const uint32_t* v = reinterpret_cast<const uint32_t*>(srow + c0);
    uint4* sout = reinterpret_cast<uint4*>(srow + c0);
    const int nr = ((c0 & 32) == 0) ? qkn_range(p, n0) : -1;   // warp-uniform
    if (nr >= 0) {
      if (row_ok)
        epilogue_qknorm(p, v, v + 32, nr ? p.qkn_k_w : p.qkn_q_w, nr ? p.qkn_k_b : p.qkn_q_b, sbias, sout);
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
                     more ? tn * BN + c1 : -1, sout);
    have_pre = more;
  }
  // the warp's 32 rows x (at most) BN / 2 columns, now in the staged rows, go out as coalesced 16-byte stores
  const int n_start = tn * BN + col_half * (BN / 2);
  store_rows<C::kLdStage>(p, acc_smem + (row_in_tile - lane) * C::kLdStage + col_half * (BN / 2), lane, l - lane, sg,
                          n_start, min(BN / 2, p.N - n_start));
}

// One problem of a launch: tensor maps + kernel parameters.  tile_m = rows per tile, box_n = rows of W one CTA fetches
// per k-block, bn = output columns per tile.
struct Problem {
  LinearParams p;
  CUtensorMap tx, tw;
};

// The ring's operand maps (ring_produce): X as nseg segments of seg_len rows of K halfs (row stride ldx, segment stride
// seg_stride rows), read as BM x BK boxes; W as w_rows rows of K halfs, read as box_n x BK boxes.
int make_operand_maps(r3g_ctx* ctx, const void* x, int64_t ldx, int64_t seg_len, int nseg, int64_t seg_stride,
                      const void* w, int64_t w_rows, int K, int box_n, CUtensorMap& tx, CUtensorMap& tw) {
  {
    const uint64_t dims[3] = {(uint64_t)K, (uint64_t)seg_len, (uint64_t)nseg};
    const uint64_t strides[3] = {2, (uint64_t)ldx * 2, (uint64_t)seg_stride * ldx * 2};
    const uint32_t box[3] = {BK, BM, 1};
    int rc = r3g_make_tmap_f16(ctx, &tx, x, 3, dims, strides, box);
    if (rc) return rc;
  }
  const uint64_t dims[2] = {(uint64_t)K, (uint64_t)w_rows};
  const uint64_t strides[2] = {2, (uint64_t)K * 2};
  const uint32_t box[2] = {BK, (uint32_t)box_n};
  return r3g_make_tmap_f16(ctx, &tw, w, 2, dims, strides, box);
}

int make_problem(r3g_ctx* ctx, const r3g_linear_args* a, int tile_m, int box_n, int bn, Problem& out) {
  LinearParams& p = out.p;
  memset(&p, 0, sizeof(p));
  if (!a) return R3G_OK;   // no such problem: tiles_m = 0
  const int seg_len = a->seg_len > 0 ? a->seg_len : a->M;
  const int nseg = a->M / seg_len;
  int rc = make_operand_maps(ctx, a->x, a->ldx, seg_len, nseg, nseg > 1 ? a->x_seg_stride : seg_len, a->w, a->N, a->K,
                             box_n, out.tx, out.tw);
  if (rc) return rc;
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

constexpr int kMaxGroup = 3;   // problems per launch

// probs[0..n): the non-empty problems of one call, n >= 1
template <int BN>
int launch_linear(r3g_ctx* ctx, const r3g_linear_args* const* probs, int n, cudaStream_t s) {
  using C = Cfg<BN>;
  Problem pr[kMaxGroup];
  int tiles = 0;
  for (int i = 0; i < kMaxGroup; ++i) {
    int rc = make_problem(ctx, i < n ? probs[i] : nullptr, BM, BN, BN, pr[i]);
    if (rc) return rc;
    if (i >= n) { pr[i].tx = pr[0].tx; pr[i].tw = pr[0].tw; }
    tiles += pr[i].p.tiles_m * pr[i].p.tiles_n;
  }
  constexpr unsigned kAttrBit = BN == 256 ? R3G_ATTR_LINEAR256 : R3G_ATTR_LINEAR128;
  if (!(ctx->attr_done & kAttrBit)) {
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(linear_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                          C::kSmemBytes));
    ctx->attr_done |= kAttrBit;
  }
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, linear_kernel<BN>, dim3(tiles), dim3(kNumThreads), C::kSmemBytes, s, pr[0].tx,
                                   pr[0].tw, pr[1].tx, pr[1].tw, pr[2].tx, pr[2].tw, pr[0].p, pr[1].p, pr[2].p));
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
  if (a->gate && a->residual_f32)
    return r3g_fail(ctx, R3G_E_INVALID, "linear: gate takes the fp16 residual form, not residual_f32 (use ls_gamma)");
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

// ------------------------------------------------------------------------------------------ mixture of experts
// (r3g_linear moe_mode; include/r3g.h).  MoEGate with N <= 64 experts is a GEMV-sized problem per row: one warp per row
// computes the logits, the softmax, the top-k and the slot assignment, and copies the row into each chosen slot.
constexpr int kRouteWarps = 8;
constexpr int kMaxExperts = 64;

// Does score a of expert ea rank before score b of expert eb?  Higher first, NaN above every number (torch.topk's
// order), equal scores and two NaNs to the lower expert.  A strict total order whatever the scores are, so the
// butterfly below agrees on one winner in every lane, and -1 (no expert, or taken) never beats a valid score or a NaN.
__device__ __forceinline__ bool route_before(float a, int ea, float b, int eb) {
  const bool na = a != a, nb = b != b;
  if (na != nb) return na;
  return na || a == b ? ea < eb : a > b;
}

__global__ void __launch_bounds__(32 * kRouteWarps)
moe_route_kernel(const __half* __restrict__ x, int64_t ldx, const __half* __restrict__ wg, __half* __restrict__ logits,
                 int64_t ldl, int M, int K, int E, int top_k, int cap, int32_t* __restrict__ counts,
                 int32_t* __restrict__ ids, __half* __restrict__ weights, int32_t* __restrict__ slots,
                 __half* __restrict__ slot_x, __half* __restrict__ slot_scale) {
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kRouteWarps + (threadIdx.x >> 5);
  if (r >= M) return;
  const __half* xr = x + (int64_t)r * ldx;
  // expert e's fp16 logit ends up in lane e % 32, register e / 32
  float lg[2] = {-INFINITY, -INFINITY};
  for (int e = 0; e < E; ++e) {
    const __half* we = wg + (int64_t)e * K;
    float acc = 0.f;
    for (int k = lane * 8; k < K; k += 256) {
      float a[8], b[8];
      unpack8(*reinterpret_cast<const Half8*>(xr + k), a);
      unpack8(*reinterpret_cast<const Half8*>(we + k), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(a[j], b[j], acc);
    }
    acc = rnd_h(warp_sum(acc));
    if (lane == (e & 31)) lg[e >> 5] = acc;
  }
  for (int h = 0; h < 2; ++h)
    if (h * 32 + lane < E) logits[(int64_t)r * ldl + h * 32 + lane] = __float2half_rn(lg[h]);
  // softmax over the fp16 logits in fp32, scores rounded to fp16 (torch's half softmax)
  float mx = fmaxf(lg[0], lg[1]);
#pragma unroll
  for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float ex[2];
  for (int h = 0; h < 2; ++h) ex[h] = h * 32 + lane < E ? expf(lg[h] - mx) : 0.f;
  const float inv = 1.f / warp_sum(ex[0] + ex[1]);
  float sc[2];
  for (int h = 0; h < 2; ++h) sc[h] = h * 32 + lane < E ? rnd_h(ex[h] * inv) : -1.f;
  for (int j = 0; j < top_k; ++j) {
    // the first expert in route_before's order; valid scores are >= 0 or NaN, so the winner is a valid, untaken one
    const bool hi = route_before(sc[1], 32 + lane, sc[0], lane);
    float bv = hi ? sc[1] : sc[0];
    int be = hi ? 32 + lane : lane;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      if (route_before(ov, oe, bv, be)) { bv = ov; be = oe; }
    }
    if (lane == (be & 31)) sc[be >> 5] = -1.f;   // taken
    int slot = 0;
    if (lane == 0) {
      slot = be * cap + atomicAdd(&counts[be], 1);
      const int64_t o = (int64_t)r * top_k + j;
      ids[o] = be;
      weights[o] = __float2half_rn(bv);
      slots[o] = slot;
      slot_scale[slot] = __float2half_rn(bv);
    }
    slot = __shfl_sync(0xffffffffu, slot, 0);
    __half* dst = slot_x + (int64_t)slot * K;
    for (int k = lane * 8; k < K; k += 256) *reinterpret_cast<uint4*>(dst + k) = *reinterpret_cast<const uint4*>(xr + k);
  }
}

// Grouped expert GEMM (moe_mode 2) and the shared expert's combine GEMM (moe_mode 3): the operand ring of
// linear_kernel<128> (ring_init / ring_produce / ring_consume; X as one segment of groups * M rows), so that a row's
// accumulators are those r3g_linear computes for it, with a per-row epilogue in which each thread writes its own row.
// No PDL: the row counts come from the route launch before it.
struct MoeParams {
  int M, N, K;               // M: rows per group (grouped) or rows (combine)
  int groups, experts, tiles_m, tiles_n;
  const int32_t* counts;
  const __half* bias;        // [groups, N]
  __half* y;
  int64_t ldy;
  int act;
  const __half* row_scale;   // [groups * M]
  const __half* residual;    // combine
  const __half* slot_y;      // combine: [*, N]
  const int32_t* slots;
  const int32_t* ids;
  int top_k;
};

__global__ void __launch_bounds__(kNumThreads, Cfg<128>::kMinBlocks)
moe_gemm_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                const __grid_constant__ MoeParams p) {
  using C = Cfg<128>;
  constexpr int BN = 128;
  const int per_group = p.tiles_m * p.tiles_n;
  const int g = blockIdx.x / per_group, lt = blockIdx.x % per_group;
  const int tm = lt / p.tiles_n, tn = lt % p.tiles_n;
  const int rows = g < p.experts ? p.counts[g] : p.M;
  if (tm * BM >= rows) return;   // surplus tile of the worst-case grid: the whole CTA leaves before any barrier
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::kStages * C::kStageBytes);
  uint64_t* empty_bar = full_bar + C::kStages;
  float* acc_smem = reinterpret_cast<float*>(smem);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_k_blocks = (p.K + BK - 1) / BK;
  const int row0 = g * p.M + tm * BM;   // first x / y row of the tile

  if (warp == kNumEpilogueWarps && lane == 0) ring_init<BN>(&tmap_x, &tmap_w, full_bar, empty_bar);
  __syncthreads();

  if (warp == kNumEpilogueWarps) {
    if (lane == 0)
      ring_produce<BN>(smem, full_bar, empty_bar, &tmap_x, &tmap_w, row0, 0, g * p.N + tn * BN, num_k_blocks);
    return;
  }

  ring_consume<BN>(smem, full_bar, empty_bar, num_k_blocks, warp, lane);

  // epilogue: one row, half of the tile's columns, 8 columns at a time
  const int row_in_tile = threadIdx.x & (BM - 1);
  const int col_half = threadIdx.x >> 7;
  if (tm * BM + row_in_tile >= rows) return;
  const int64_t yr = row0 + row_in_tile;
  const float* srow = acc_smem + row_in_tile * C::kLdStage;
  const float scale = p.row_scale ? __half2float(p.row_scale[yr]) : 1.f;
  int64_t src[4] = {0, 0, 0, 0};   // combine: the row's slots in increasing expert order
  if (p.slot_y) {
    int e[4];
    for (int j = 0; j < p.top_k; ++j) { e[j] = p.ids[yr * p.top_k + j]; src[j] = p.slots[yr * p.top_k + j]; }
    for (int i = 1; i < p.top_k; ++i)
      for (int j = i; j > 0 && e[j - 1] > e[j]; --j) {
        const int te = e[j]; e[j] = e[j - 1]; e[j - 1] = te;
        const int64_t ts = src[j]; src[j] = src[j - 1]; src[j - 1] = ts;
      }
  }
#pragma unroll 1
  for (int c = col_half * (BN / 2); c < (col_half + 1) * (BN / 2); c += 8) {
    const int n = tn * BN + c;
    if (n >= p.N) break;
    float f[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = srow[c + j];
    if (p.bias) {
      float b[8];
      unpack8(*reinterpret_cast<const Half8*>(p.bias + (int64_t)g * p.N + n), b);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] += b[j];
    }
    if (p.act == 2) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = gelu_erf_f(rnd_h(f[j]));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = rnd_h(f[j]);
    if (p.row_scale) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = rnd_h(f[j] * scale);
    }
    if (p.slot_y) {
      float s[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, t[8], res[8];
      for (int k = 0; k < p.top_k; ++k) {
        unpack8(*reinterpret_cast<const Half8*>(p.slot_y + src[k] * p.N + n), t);
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = rnd_h(s[j] + t[j]);
      }
      unpack8(*reinterpret_cast<const Half8*>(p.residual + yr * p.ldy + n), res);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = res[j] + rnd_h(s[j] + f[j]);
    }
    *reinterpret_cast<Half8*>(p.y + yr * p.ldy + n) = pack8(f);
  }
}

int launch_moe_route(r3g_ctx* ctx, const r3g_linear_args* a, cudaStream_t s) {
  const int E = a->moe_experts;
  if (a->N != E || E < 1 || E > kMaxExperts || a->moe_top_k < 1 || a->moe_top_k > 4 || a->moe_top_k > E ||
      a->moe_cap < a->M || a->K % 8 || a->ldx % 8 || a->bias || !a->moe_counts || !a->moe_ids || !a->moe_weights ||
      !a->moe_slots || !a->moe_slot_x || !a->moe_slot_scale)
    return r3g_fail(ctx, R3G_E_INVALID, "linear (moe route): need N == moe_experts <= %d, 1 <= moe_top_k <= min(4, N), "
                    "moe_cap >= M, K %% 8 == 0, no bias and every moe buffer (N=%d experts=%d top_k=%d)", kMaxExperts,
                    a->N, E, a->moe_top_k);
  R3G_CUDA_OK(ctx, cudaMemsetAsync(a->moe_counts, 0, sizeof(int32_t) * E, s));
  moe_route_kernel<<<(a->M + kRouteWarps - 1) / kRouteWarps, 32 * kRouteWarps, 0, s>>>(
      (const __half*)a->x, a->ldx, (const __half*)a->w, (__half*)a->y, a->ldy, a->M, a->K, E, a->moe_top_k, a->moe_cap,
      a->moe_counts, a->moe_ids, (__half*)a->moe_weights, a->moe_slots, (__half*)a->moe_slot_x,
      (__half*)a->moe_slot_scale);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

int launch_moe_gemm(r3g_ctx* ctx, const r3g_linear_args* a, cudaStream_t s) {
  const bool combine = a->moe_mode == R3G_MOE_COMBINE;
  const int groups = combine ? 1 : a->moe_groups;
  if (a->N % 8 || a->K % 8 || a->ldx % 8 || a->ldy % 8 || groups < 1)
    return r3g_fail(ctx, R3G_E_INVALID, "linear (moe): need N %% 8 == 0, K %% 8 == 0, ldx/ldy %% 8 == 0, moe_groups >= 1");
  if ((a->act != 0 && a->act != 2) || (combine && a->act))
    return r3g_fail(ctx, R3G_E_INVALID, "linear (moe): act must be 0, or 2 (erf-GELU) in grouped mode");
  if (combine ? (!a->residual || !a->moe_slot_y || !a->moe_slots || !a->moe_ids || a->moe_top_k < 1 ||
                 a->moe_top_k > 4 || a->moe_slot_scale)
              : (a->moe_experts < 0 || a->moe_experts > groups || a->moe_cap != a->M ||
                 (a->moe_experts && !a->moe_counts) || a->residual || a->moe_slot_y))
    return r3g_fail(ctx, R3G_E_INVALID, "linear (moe %s): inconsistent moe operands", combine ? "combine" : "grouped");
  CUtensorMap tx, tw;
  const int64_t rows = (int64_t)groups * a->M;
  int rc = make_operand_maps(ctx, a->x, a->ldx, rows, 1, rows, a->w, (int64_t)groups * a->N, a->K, 128, tx, tw);
  if (rc) return rc;
  MoeParams p;
  memset(&p, 0, sizeof(p));
  p.M = a->M; p.N = a->N; p.K = a->K;
  p.groups = groups;
  p.experts = combine ? 0 : a->moe_experts;
  p.tiles_m = (a->M + BM - 1) / BM;
  p.tiles_n = (a->N + 127) / 128;
  p.counts = a->moe_counts;
  p.bias = (const __half*)a->bias;
  p.y = (__half*)a->y; p.ldy = a->ldy;
  p.act = a->act;
  p.row_scale = (const __half*)a->moe_slot_scale;
  if (combine) {
    p.residual = (const __half*)a->residual;
    p.slot_y = (const __half*)a->moe_slot_y;
    p.slots = a->moe_slots;
    p.ids = a->moe_ids;
    p.top_k = a->moe_top_k;
  }
  using C = Cfg<128>;
  if (!(ctx->attr_done & R3G_ATTR_MOE_GEMM)) {
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(moe_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmemBytes));
    ctx->attr_done |= R3G_ATTR_MOE_GEMM;
  }
  moe_gemm_kernel<<<(unsigned)(groups * p.tiles_m * p.tiles_n), kNumThreads, C::kSmemBytes, s>>>(tx, tw, p);
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}

}  // namespace

extern "C" int r3g_linear(r3g_ctx* ctx, const r3g_linear_args* a, void* stream) {
  R3G_ENTRY(ctx, "linear");
  if (!a) return r3g_fail(ctx, R3G_E_INVALID, "linear: null argument");
  if (a->moe_mode) {
    if (a->moe_mode < R3G_MOE_ROUTE || a->moe_mode > R3G_MOE_COMBINE)
      return r3g_fail(ctx, R3G_E_INVALID, "linear: unknown moe_mode %d", a->moe_mode);
    if (!a->x || !a->w || !a->y || a->group_next || a->gate || a->out_f32 || a->residual_f32 || a->ls_gamma ||
        a->qkn_mode || a->seg_len || (a->moe_mode == R3G_MOE_ROUTE && a->act))
      return r3g_fail(ctx, R3G_E_INVALID, "linear (moe): no group_next, gate, fp32, qkn or segment operands");
    if (a->M <= 0) return R3G_OK;
    cudaStream_t s = (cudaStream_t)stream;
    return a->moe_mode == R3G_MOE_ROUTE ? launch_moe_route(ctx, a, s) : launch_moe_gemm(ctx, a, s);
  }
  // the non-empty problems of the group_next chain, in order
  const r3g_linear_args* probs[kMaxGroup];
  int n = 0, len = 0;
  for (const r3g_linear_args* q = a; q; q = (const r3g_linear_args*)q->group_next) {
    if (++len > kMaxGroup) return r3g_fail(ctx, R3G_E_INVALID, "linear: at most %d problems per launch", kMaxGroup);
    if (q->M <= 0) continue;
    int rc = validate_linear(ctx, q);
    if (rc) return rc;
    probs[n++] = q;
  }
  if (!n) return R3G_OK;
  cudaStream_t s = (cudaStream_t)stream;
  // Tile choice: wave efficiency (tiles / (waves * resident CTAs)) over the tiles of ALL problems of a grouped launch.
  // A 128 x 256 tile reads half the operand bytes per FLOP of a 128 x 128 one but runs one CTA per SM instead of
  // two; it is taken unless it leaves more of the last wave idle.
  const int sms = ctx->num_sms;
  auto eff = [&](int64_t tiles, int units) {
    if (tiles <= 0) return 0.0;
    const int64_t waves = (tiles + units - 1) / units;
    return (double)tiles / (double)(waves * units);
  };
  auto tiles_of = [&](const r3g_linear_args* q, int tm, int tn) -> int64_t {
    const int seg = q->seg_len > 0 ? q->seg_len : q->M;
    return (int64_t)(q->M / seg) * ((seg + tm - 1) / tm) * ((q->N + tn - 1) / tn);
  };
  int n_min = probs[0]->N;
  int64_t t256 = 0, t128 = 0;
  for (int i = 0; i < n; ++i) {
    n_min = probs[i]->N < n_min ? probs[i]->N : n_min;
    t256 += tiles_of(probs[i], BM, 256);
    t128 += tiles_of(probs[i], BM, 128);
  }
  const double e256 = n_min >= 256 ? eff(t256, sms) : 0.0;
  const double e128 = eff(t128, 2 * sms);
  if (e256 > 0.0 && e256 >= e128) return launch_linear<256>(ctx, probs, n, s);
  return launch_linear<128>(ctx, probs, n, s);
}
