// r3g_attention: O = softmax(Q K^T * scale) V for head_dim 64, no mask -- flash-attention forward on wgmma (sm_90a).
//
// One CTA = one 192-row query tile of one (batch, head):
//   warps 0..11  three consumer warpgroups, 64 query rows each.  Per 128-key tile: S = Q K^T (wgmma m64n128k16 x4,
//                both operands from shared memory, fp32 accumulators in registers); online softmax in registers (a
//                row lives in the 4 threads of a quad: two shuffles for its max); P is packed to fp16 in registers and
//                is directly the A operand of O += P V (wgmma m64n64k16 x8, V read MN-major from its row-major tile).
//   warp 12      TMA producer: Q once, then K and V tiles (128 x 64) through 3-deep rings.
// Three warpgroups per SM let one warpgroup's softmax overlap the others' MMAs.
// Call sites replaced: F.scaled_dot_product_attention in hunyuan3ddit.py:33-36 (L = 4442 joint txt+img tokens),
// attention_blocks.py:328 (ShapeVAE, L = 3072), attention_processors.py:29-32 (geo-decoder cross attention,
// Lk = 3072), vggt/layers/attention.py:61.
#include <cuda_fp16.h>
#include <math.h>

#include "r3g_internal.h"
#include "r3g_ptx.cuh"

namespace {

using namespace r3g;

constexpr int kD = 64;
constexpr int kWG = 3;                            // consumer warpgroups
constexpr int kBQ = 64 * kWG;                     // query rows per CTA
constexpr int kBKV = 128;
constexpr int kStg = 3;                           // K / V ring depth
constexpr int kQBytes = 64 * kD * 2;              // 8 KB per warpgroup
constexpr int kTileBytes = kBKV * kD * 2;         // 16 KB: K and V tiles
constexpr int kTilesBytes = kQBytes * kWG + 2 * kStg * kTileBytes;   // 120 KB
constexpr int kSmemBytes = kTilesBytes + 1024 + 256;   // + alignment slack + barriers
constexpr int kThreads = 128 * kWG + 32;

struct AttnParams {
  __half* o;
  int64_t o_sb, o_sh, o_sl;
  int Lq, Lk;
  float scale_log2;  // scale * log2(e)
  // query windows (r3g_attention_args.win_*): nwin = 0, or one window per batch with the batches' query tiles
  // concatenated along grid.x (window 1 from tile tiles0 on)
  int nwin, tiles0;
  int row0[2], len[2];
};

// The key/value fill of a windowed call: rows [dst0[b], dst0[b] + rows[b]) of k and v of batch b become copies of row
// src[b] (r3g_attention_args.win_k0_count).
struct KvFill {
  __half *k, *v;
  int64_t k_sb, k_sh, k_sl, v_sb, v_sh, v_sl;
  int H;
  int src[2], dst0[2], rows[2];
};

__global__ void __launch_bounds__(256) kv_fill_kernel(const KvFill f) {
  pdl_wait();
  pdl_trigger();
  const int per_row = f.H * 2 * (kD / 8);           // 16-byte chunks of one row: heads x (k, v) x 8
  const int64_t n0 = (int64_t)f.rows[0] * per_row, total = n0 + (int64_t)f.rows[1] * per_row;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = i >= n0;
    int64_t r = b ? i - n0 : i;
    const int c = (int)(r % (kD / 8));
    r /= kD / 8;
    const int kv = (int)(r & 1);
    r >>= 1;
    const int h = (int)(r % f.H);
    r /= f.H;
    __half* base = kv ? f.v : f.k;
    const int64_t sb = kv ? f.v_sb : f.k_sb, sh = kv ? f.v_sh : f.k_sh, sl = kv ? f.v_sl : f.k_sl;
    __half* head = base + b * sb + h * sh + 8 * c;
    *reinterpret_cast<uint4*>(head + ((b ? f.dst0[1] : f.dst0[0]) + r) * sl) =
        *reinterpret_cast<const uint4*>(head + (int64_t)(b ? f.src[1] : f.src[0]) * sl);
  }
}

__global__ void __launch_bounds__(kThreads, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmap_q, const __grid_constant__ CUtensorMap tmap_k,
                 const __grid_constant__ CUtensorMap tmap_v, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + kWG * kQBytes;
  uint8_t* sV = sK + kStg * kTileBytes;
  uint64_t* q_full = reinterpret_cast<uint64_t*>(smem + kTilesBytes);
  uint64_t* k_full = q_full + 1;
  uint64_t* v_full = k_full + kStg;
  uint64_t* k_empty = v_full + kStg;
  uint64_t* v_empty = k_empty + kStg;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int h = blockIdx.y;
  int b = blockIdx.z, q0 = blockIdx.x * kBQ, row_base = 0, Lq = p.Lq;
  if (p.nwin) {
    const int w = blockIdx.x >= p.tiles0;
    b = w;
    q0 = (blockIdx.x - (w ? p.tiles0 : 0)) * kBQ;
    row_base = w ? p.row0[1] : p.row0[0];
    Lq = w ? p.len[1] : p.len[0];
  }
  const int n_kv = (p.Lk + kBKV - 1) / kBKV;

  if (warp == 4 * kWG && lane == 0) {
    tma_prefetch_desc(&tmap_q);
    tma_prefetch_desc(&tmap_k);
    tma_prefetch_desc(&tmap_v);
    mbar_init(q_full, 1);
    for (int s = 0; s < kStg; ++s) {
      mbar_init(&k_full[s], 1);
      mbar_init(&v_full[s], 1);
      mbar_init(&k_empty[s], 128 * kWG);
      mbar_init(&v_empty[s], 128 * kWG);
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();      // q / k / v come from the projection kernel before us (no trigger here: a multi-wave grid must not
                   // let the next kernel's CTAs take SM slots from its own later waves; the implicit one at exit is used)

  if (warp == 4 * kWG) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      // a warpgroup whose 64 rows all lie past Lq gets no Q (it computes on stale data and stores nothing)
      const int groups = min(kWG, (Lq - q0 + 63) / 64);
      mbar_expect_tx(q_full, groups * kQBytes);
      for (int g = 0; g < groups; ++g)
        tma_load_4d(sQ + g * kQBytes, &tmap_q, q_full, 0, row_base + q0 + 64 * g, h, b, kEvictFirst);
      for (int j = 0; j < n_kv; ++j) {
        const int st = j % kStg;
        const uint32_t ph = (j / kStg) & 1;
        mbar_wait(&k_empty[st], ph ^ 1);
        mbar_expect_tx(&k_full[st], kTileBytes);
        tma_load_4d(sK + st * kTileBytes, &tmap_k, &k_full[st], 0, j * kBKV, h, b, kEvictLast);
        mbar_wait(&v_empty[st], ph ^ 1);
        mbar_expect_tx(&v_full[st], kTileBytes);
        tma_load_4d(sV + st * kTileBytes, &tmap_v, &v_full[st], 0, j * kBKV, h, b, kEvictLast);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers
  // accumulator layout (r3g_ptx.cuh): element i of a thread is row r0 + 8 ((i / 2) % 2), column 8 (i / 4) + c0 + i % 2
  const int wg = warp >> 2;
  const int r0 = (warp & 3) * 16 + (lane >> 2);
  const int c0 = 2 * (lane & 3);
  const uint32_t aq = smem_u32(sQ + wg * kQBytes);
  float o[kD / 2];
#pragma unroll
  for (int i = 0; i < kD / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int st = j % kStg;
    const uint32_t ph = (j / kStg) & 1;
    float s[kBKV / 2];
    mbar_wait(&k_full[st], ph);
    const uint32_t ak = smem_u32(sK + st * kTileBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kD / 16; ++k)
      wgmma_m64n128k16_ss(s, gmma_desc_sw128(aq + k * 32, 1024, 16), gmma_desc_sw128(ak + k * 32, 1024, 16),
                          k ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<kBKV / 2>(s);
    mbar_arrive(&k_empty[st]);

    const int valid = min(kBKV, p.Lk - j * kBKV);
    if (valid < kBKV) {
#pragma unroll
      for (int i = 0; i < kBKV / 2; ++i)
        if (8 * (i >> 2) + c0 + (i & 1) >= valid) s[i] = -INFINITY;
    }
    // row maxima (rows r0 and r0 + 8) over the quad, in log2 units
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < kBKV / 2; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
    float alpha[2];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 1));
      mx[rr] = fmaxf(mx[rr], __shfl_xor_sync(0xffffffffu, mx[rr], 2));
      const float m_new = fmaxf(m_run[rr], mx[rr] * p.scale_log2);
      alpha[rr] = ex2_approx(m_run[rr] - m_new);   // 0 on the first tile (m_run = -inf)
      m_run[rr] = m_new;
      l_run[rr] *= alpha[rr];
    }
#pragma unroll
    for (int i = 0; i < kD / 2; ++i) o[i] *= alpha[(i >> 1) & 1];
    // probabilities, packed to fp16 in the A-operand layout of the P V MMA (16 keys per k-step)
    uint32_t pk[kBKV / 16][4];
#pragma unroll
    for (int i = 0; i < kBKV / 2; i += 2) {
      const int rr = (i >> 1) & 1;
      const float e0 = ex2_approx(fmaf(s[i], p.scale_log2, -m_run[rr]));
      const float e1 = ex2_approx(fmaf(s[i + 1], p.scale_log2, -m_run[rr]));
      l_run[rr] += e0 + e1;
      pk[i >> 3][(i >> 1) & 3] = pack_half2(e0, e1);
    }
    mbar_wait(&v_full[st], ph);
    const uint32_t av = smem_u32(sV + st * kTileBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kBKV / 16; ++k) wgmma_m64n64k16_rs_tb(o, pk[k], gmma_desc_sw128(av + k * 2048, 1024, 1024), 1u);
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence<kD / 2>(o);
    mbar_arrive(&v_empty[st]);
  }

  float inv_l[2];
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    float l = l_run[rr];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    inv_l[rr] = 1.f / l;
  }
#pragma unroll
  for (int rr = 0; rr < 2; ++rr) {
    const int qrow = q0 + wg * 64 + r0 + 8 * rr;
    if (qrow >= Lq) continue;
    __half* op = p.o + (int64_t)b * p.o_sb + (int64_t)h * p.o_sh + (int64_t)(row_base + qrow) * p.o_sl;
#pragma unroll
    for (int i = 2 * rr; i < kD / 2; i += 4)
      *reinterpret_cast<uint32_t*>(op + 8 * (i >> 2) + c0) = pack_half2(o[i] * inv_l[rr], o[i + 1] * inv_l[rr]);
  }
}

int make_qkv_map(r3g_ctx* ctx, CUtensorMap* m, const void* base, int64_t sb, int64_t sh, int64_t sl, int B, int H,
                 int L, int box_rows) {
  const uint64_t dims[4] = {(uint64_t)kD, (uint64_t)L, (uint64_t)H, (uint64_t)B};
  const uint64_t strides[4] = {2, (uint64_t)sl * 2, (uint64_t)sh * 2, (uint64_t)sb * 2};
  const uint32_t box[4] = {(uint32_t)kD, (uint32_t)box_rows, 1, 1};
  return r3g_make_tmap_f16(ctx, m, base, 4, dims, strides, box);
}

}  // namespace

extern "C" int r3g_attention(r3g_ctx* ctx, const r3g_attention_args* a, void* stream) {
  R3G_ENTRY(ctx, "attention");
  if (!a || !a->q || !a->k || !a->v || !a->o) return r3g_fail(ctx, R3G_E_INVALID, "attention: null argument");
  if (a->B < 1 || a->H < 1 || a->Lq < 1 || a->Lk < 1) return r3g_fail(ctx, R3G_E_INVALID, "attention: empty shape");
  if (a->o_sl % 8 || a->o_sh % 8 || a->o_sb % 8 || !r3g_aligned16(a->o))
    return r3g_fail(ctx, R3G_E_INVALID, "attention: output strides must be multiples of 8 halfs");
  CUtensorMap mq, mk, mv;
  int rc;
  if ((rc = make_qkv_map(ctx, &mq, a->q, a->q_sb, a->q_sh, a->q_sl, a->B, a->H, a->Lq, 64))) return rc;
  if ((rc = make_qkv_map(ctx, &mk, a->k, a->k_sb, a->k_sh, a->k_sl, a->B, a->H, a->Lk, kBKV))) return rc;
  if ((rc = make_qkv_map(ctx, &mv, a->v, a->v_sb, a->v_sh, a->v_sl, a->B, a->H, a->Lk, kBKV))) return rc;
  AttnParams p = {};
  p.o = (__half*)a->o;
  p.o_sb = a->o_sb; p.o_sh = a->o_sh; p.o_sl = a->o_sl;
  p.Lq = a->Lq; p.Lk = a->Lk;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  int tiles = (a->Lq + kBQ - 1) / kBQ, grid_z = a->B;
  KvFill f = {};
  if (a->win_len[0] > 0) {
    if (a->Lq != a->Lk || a->B > R3G_ATTN_MAX_WINDOWS)
      return r3g_fail(ctx, R3G_E_INVALID, "attention: windows need Lq == Lk and B <= %d", R3G_ATTN_MAX_WINDOWS);
    tiles = 0;
    for (int w = 0; w < a->B; ++w) {
      const int r0 = a->win_row0[w], n = a->win_len[w], cnt = a->win_k0_count[w] > 1 ? a->win_k0_count[w] : 1;
      if (r0 < 0 || n < 1 || r0 + n > a->Lq || r0 - (cnt - 1) < 0)
        return r3g_fail(ctx, R3G_E_INVALID, "attention: window %d [%d, %d + %d) with %d copies of its first key outside "
                        "[0, %d)", w, r0, r0, n, cnt, a->Lq);
      p.row0[w] = r0;
      p.len[w] = n;
      tiles += (n + kBQ - 1) / kBQ;
      if (w == 0) p.tiles0 = tiles;
      f.src[w] = r0;
      f.dst0[w] = r0 - (cnt - 1);
      f.rows[w] = cnt - 1;
    }
    p.nwin = a->B;
    grid_z = 1;
  }
  if (f.rows[0] > 0 || f.rows[1] > 0) {
    if (a->k_sb % 8 || a->k_sh % 8 || a->k_sl % 8 || a->v_sb % 8 || a->v_sh % 8 || a->v_sl % 8 || !r3g_aligned16(a->k) ||
        !r3g_aligned16(a->v))
      return r3g_fail(ctx, R3G_E_INVALID, "attention: copied keys need k / v strides that are multiples of 8 halfs");
    f.k = (__half*)a->k; f.v = (__half*)a->v;
    f.k_sb = a->k_sb; f.k_sh = a->k_sh; f.k_sl = a->k_sl;
    f.v_sb = a->v_sb; f.v_sh = a->v_sh; f.v_sl = a->v_sl;
    f.H = a->H;
    const int64_t chunks = ((int64_t)f.rows[0] + f.rows[1]) * a->H * 2 * (kD / 8);
    const unsigned fgrid = (unsigned)min((chunks + 255) / 256, (int64_t)ctx->num_sms * 8);
    R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, kv_fill_kernel, dim3(fgrid), dim3(256), 0, (cudaStream_t)stream, f));
    R3G_LAUNCH_OK(ctx);
  }
  if (!(ctx->attr_done & R3G_ATTR_ATTENTION)) {   // function attributes are per device: one flag per context
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    R3G_CUDA_OK(ctx, cudaFuncSetAttribute(attention_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
    ctx->attr_done |= R3G_ATTR_ATTENTION;
  }
  dim3 grid(tiles, a->H, grid_z);
  R3G_CUDA_OK(ctx, r3g_launch_pdl(ctx, attention_kernel, grid, dim3(kThreads), kSmemBytes, (cudaStream_t)stream, mq, mk, mv, p));
  R3G_LAUNCH_OK(ctx);
  return R3G_OK;
}
