/* r3g -- C ABI of the H100-native hot path of 3D-RE-GEN (stage 3: Hunyuan3D-2 shape generation,
 * stage 4: VGGT back-projection).  The reference has no FFI of its own: its operator interface is the
 * set of Python plug points listed in SURVEY.md section 8(b).  Every entry point below names the reference
 * interface (file:line under /root/reference) it sits underneath; the Python mirror of those
 * interfaces lives in 3d-re-gen_b200/r3g/ and calls this library through ctypes (INTEGRATION.md).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch types.
 *   - All pointers are DEVICE pointers on the context's device unless the name ends in _host.
 *   - Every call is asynchronous on `stream` (a cudaStream_t passed as void*) unless stated otherwise.
 *   - Return value: 0 = OK, negative = error (R3G_E_*); r3g_last_error(ctx) gives the message.
 *   - A context is bound to one device and is not thread-safe; distinct contexts are independent.
 *   - There is no CPU fallback: without a CUDA device every compute call returns R3G_E_CUDA.
 */
#ifndef R3G_H
#define R3G_H
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct r3g_ctx r3g_ctx;

enum {
  R3G_OK = 0,
  R3G_E_INVALID = -1,    /* bad argument / unsupported shape */
  R3G_E_CUDA = -2,       /* CUDA runtime / driver error (message has the string) */
  R3G_E_WORKSPACE = -3,  /* workspace too small */
  R3G_E_LEVEL = -4,      /* mc: level outside [min,max] of the volume  (skimage ValueError) */
  R3G_E_NOSURFACE = -5   /* mc: no vertices                              (skimage RuntimeError) */
};

int r3g_version(void);
int r3g_create(int device, r3g_ctx** out);
void r3g_destroy(r3g_ctx* ctx);
const char* r3g_last_error(r3g_ctx* ctx);
/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
int64_t r3g_launch_count(r3g_ctx* ctx);

/* ------------------------------------------------------------------------------------------------
 * Marching cubes.  Replaces MCSurfaceExtractor.run -> skimage.measure.marching_cubes(grid.cpu().numpy(),
 * mc_level, method="lewiner") and the bbox rescale
 *   (Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/surface_extractors.py:67-76, :50-64).
 * grid: float32 [n0][n1][n2] (C order; the reference's grid_logits[i] with n = octree_resolution+1).
 * Two phases so the caller can allocate exact outputs:
 *   r3g_mc_count   : classify + count; SYNCHRONISES `stream`; writes *nv_host, *nf_host.
 *                    Returns R3G_E_LEVEL / R3G_E_NOSURFACE like skimage raises.
 *   r3g_mc_extract : emits verts float32 [nv][3] in array-axis order and faces int32 [nf][3] in skimage's
 *                    default (gradient_direction='descent') winding, i.e. BEFORE export_to_trimesh's flip
 *                    (Hunyuan3D-2/hy3dgen/shapegen/pipelines.py:102).  If bounds_host != NULL (6 doubles:
 *                    min xyz, max xyz) vertices are rescaled v / n_axis * (max-min) + min in float64 and
 *                    stored float32, as surface_extractors.py:74-75,55 do.
 * workspace: r3g_mc_workspace_bytes(n0,n1,n2) bytes of device memory (about 23 bytes per grid point: 0.39 GB at
 *            257^3, 3.0 GB at 513^3; sized for the worst case of every cell crossed), contents need not be
 *            initialised; the same workspace must be passed to count and extract.
 * Limits: (n0-1)*(n1-1)*ceil((n2-1)/32) < 2^27 (about 1600^3), else R3G_E_INVALID.
 */
size_t r3g_mc_workspace_bytes(int n0, int n1, int n2);
int r3g_mc_count(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level, void* workspace,
                 size_t workspace_bytes, int64_t* nv_host, int64_t* nf_host, void* stream);
int r3g_mc_extract(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level,
                   const double* bounds_host, void* workspace, size_t workspace_bytes, float* verts,
                   int32_t* faces, void* stream);
/* Per-cell base case 0..14 (Lewiner's `cases[cubeindex][0]`), uint8 [(n0-1)*(n1-1)*(n2-1)]; parity probe. */
int r3g_mc_classify(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level,
                    unsigned char* case_out, void* stream);

/* Connected components of a triangle mesh (vertices joined by the faces): labels[v] = the smallest vertex index of v's
 * component.  The computation behind FloaterRemover (Hunyuan3D-2/hy3dgen/shapegen/postprocessors.py:58-63,118-129:
 * pymeshlab "select small disconnected components" with nbfaceratio 0.005 + delete), applied to every generated mesh
 * by src/2d_to_3d_models/run.py:93.  faces int32 [nf][3] with indices in [0, nv); labels int32 [nv].
 * SYNCHRONISES `stream` (it reports an out-of-range index as R3G_E_INVALID). */
int r3g_mesh_components(r3g_ctx* ctx, const int32_t* faces, int64_t nf, int64_t nv, int32_t* labels, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Dense-contraction building blocks (wgmma / TMA).  Used by the DiT, ShapeVAE and geo-decoder
 * mirrors; exported so that tests can check each against the oracle in isolation.
 *
 * r3g_linear:  Y = epilogue( X[M,K] . W[N,K]^T + bias )  -- nn.Linear semantics, fp16 in, fp32 accumulate.
 *   X row-major with leading dimension ldx (halfs), W row-major [N,K] contiguous, Y leading dimension ldy.
 *   Rows may be segmented: logical row r = s * seg_len + l (0 <= l < seg_len) is read from X row
 *   s * x_seg_stride + l and written to Y row s * y_seg_stride + l (seg_len = 0: one segment of M rows).
 *   This is how the txt / img streams of DoubleStreamBlock (one segment per batch element) live inside one
 *   joint [B, Ltxt+Limg, ...] buffer without any torch.cat (hunyuan3ddit.py:205-211,396); the caller offsets
 *   the x / y pointers to the first row of the stream.
 *   act: 0 none, 1 tanh-GELU (hunyuan3ddit.py:63-69), 2 erf-GELU (attention_blocks.py:178), 3 ReLU (the DPT head's
 *        convolutions, vggt/heads/dpt_head.py:344-392); applied to output columns [act_col0, act_col1) only.
 *   gate/residual: if residual != NULL,  Y = residual + gate[b, n] * (acc + bias)  with b = r / gate_rows
 *        (gate == NULL means gate 1; gate_ld is the stride between batches in halfs), covering the gated
 *        residuals of hunyuan3ddit.py:212-216,267 and the plain residuals of attention_blocks.py:296-299.
 *        residual uses Y's row mapping and may alias Y.
 *   out_f32: 0 -> Y is fp16, 1 -> Y is float32.
 *   residual_f32 / ls_gamma: the VGGT block form (vggt/layers/block.py:77-98 under autocast): the residual stream is
 *        float32, `residual` then points to float32 with Y's geometry (Y float32, may alias), and
 *        Y = residual + ls_gamma[n] * fp16(acc + bias)  with ls_gamma the float32 LayerScale vector (NULL = 1).
 *   qkn_*: the per-head q/k normalisation that follows a q/k/v projection, fused into the epilogue (the accumulator
 *        row of a 64-column head sits in one thread's registers): qkn_mode 1 = RMSNorm(64) with a learned scale
 *        (QKNorm, hunyuan3ddit.py:83-104,199,260), 2 = LayerNorm(64) with weight + bias (attention_blocks.py:315-316,
 *        250-258).  It is applied to the fp16-rounded Linear output of the 64-column heads in
 *        [qkn_q_col0, qkn_q_col0 + qkn_cols) with (qkn_q_w, qkn_q_b) and, if qkn_k_col0 >= 0, of
 *        [qkn_k_col0, qkn_k_col0 + qkn_cols) with (qkn_k_w, qkn_k_b); the weights are fp16 [64] (bias NULL in mode 1).
 *        Column offsets and qkn_cols are multiples of 64; these columns must carry no activation / gate / residual.
 *   group_next: a second, independent problem (its own x / w / y / epilogue operands and sizes; its group_next must be
 *        NULL) whose tiles share this call's persistent grid.  The img and txt streams of a DoubleStreamBlock apply
 *        different weights to 6144 and 2740 rows (hunyuan3ddit.py:196-216): separately their N = 1024 projections
 *        fill 1.3 and 0.65 waves of 256 x 256 tiles, together 1.95 of 2.  Results are those of two separate calls.
 */
typedef struct {
  const void* x; int64_t ldx;
  const void* w;
  const void* bias;          /* fp16 [N] or NULL */
  void* y; int64_t ldy;
  int M, N, K;
  int seg_len; int64_t x_seg_stride, y_seg_stride;
  int act, act_col0, act_col1;
  const void* gate; int64_t gate_ld; int gate_rows;
  const void* residual;      /* fp16 (or float32 if residual_f32), same geometry as y */
  int out_f32;
  int residual_f32;
  const void* ls_gamma;      /* float32 [N] or NULL */
  int qkn_mode, qkn_q_col0, qkn_k_col0, qkn_cols;
  float qkn_eps;
  const void* qkn_q_w; const void* qkn_q_b; const void* qkn_k_w; const void* qkn_k_b;
  const void* group_next;    /* NULL, or a second r3g_linear_args executed by the SAME launch */
} r3g_linear_args;
int r3g_linear(r3g_ctx* ctx, const r3g_linear_args* a, void* stream);

/* r3g_attention: O = softmax(Q K^T * scale) V, no mask (F.scaled_dot_product_attention call sites:
 * hunyuan3ddit.py:33-36, attention_blocks.py:328, attention_processors.py:29-32, vggt/layers/attention.py:61).
 * head_dim is 64.  Q/K/V/O are addressed by strides in halfs: element (b, h, l, d) at
 * base + b*stride_b + h*stride_h + l*stride_l + d.  O has the "B L (H D)" layout of hunyuan3ddit.py:35 when
 * o_stride_l = H*64, o_stride_h = 64.  O may alias Q (each CTA reads its Q tile before writing it). */
typedef struct {
  const void* q; int64_t q_sb, q_sh, q_sl;
  const void* k; int64_t k_sb, k_sh, k_sl;
  const void* v; int64_t v_sb, v_sh, v_sl;
  void* o; int64_t o_sb, o_sh, o_sl;
  int B, H, Lq, Lk;
  float scale;
} r3g_attention_args;
int r3g_attention(r3g_ctx* ctx, const r3g_attention_args* a, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Row-wise / element-wise operators of the DiT and VAE blocks (fp16 storage, fp32 math).
 */
/* y[r,:] = LN(x[r,:]) * (w or 1) + (b or 0), then  * (1 + scale[bi,:]) + shift[bi,:]  with bi = r / rows_per_batch
 * (scale/shift NULL -> skipped).  LayerNorm over `width` with eps; covers nn.LayerNorm(affine=False)+modulation
 * (hunyuan3ddit.py:192-193,257) and affine LayerNorm (attention_blocks.py:296-299,425-433).
 * Rows are segmented like r3g_linear's: r = s*seg_len + l lives at x row s*x_seg_stride + l, y row s*y_seg_stride + l. */
int r3g_layernorm(r3g_ctx* ctx, const void* x, int64_t ldx, void* y, int64_t ldy, int rows, int width, float eps,
                  const void* w, const void* b, const void* scale, const void* shift, int64_t mod_ld,
                  int rows_per_batch, int seg_len, int64_t x_seg_stride, int64_t y_seg_stride, void* stream);
/* Same with a float32 input (the VGGT residual stream, vggt/layers/block.py:79,82); y is fp16. */
int r3g_layernorm_f32in(r3g_ctx* ctx, const float* x, int64_t ldx, void* y, int64_t ldy, int rows, int width,
                        float eps, const void* w, const void* b, void* stream);
/* VGGT attention prologue, in place on a packed fp16 [rows, 3*H*64] projection laid out (3, H, D)
 * (vggt/layers/attention.py:52-59): LayerNorm(64, eps) with affine q_w/q_b, k_w/k_b on q and k (NULL weights skip
 * the norm), then 2-D rotary embedding (vggt/layers/rope.py:62-188, base `rope_freq`, first half of D by the y
 * position, second half by x) when rope_freq > 0.  Row r is token (r % tokens_per_frame); tokens below n_special
 * sit at position (0,0), patch p at (p / patches_w + 1, p % patches_w + 1) (aggregator.py:216-228). */
int r3g_qk_norm_rope(r3g_ctx* ctx, void* qkv, int64_t ld, int64_t rows, int heads, float eps, const void* q_w,
                     const void* q_b, const void* k_w, const void* k_b, float rope_freq, int tokens_per_frame,
                     int n_special, int patches_w, void* stream);
/* Patch extraction for the ViT patch embedding (vggt/layers/patch_embed.py:72-85 as a GEMM): images float32
 * [N,3,H,W]; each value is normalised (v - mean[c]) / std[c] first (aggregator.py:199-200; pass mean 0 / std 1 to
 * skip); out fp16 [N*(H/ps)*(W/ps), out_ld] with column c*ps*ps + py*ps + px (Conv2d weight order), zero padded. */
int r3g_patchify(r3g_ctx* ctx, const float* images, void* out, int64_t out_ld, int N, int H, int W, int patch,
                 const float* mean3_host, const float* std3_host, void* stream);
/* In-place per-head normalisation of q and k inside a packed projection output.
 * Element (r, h, d) of q lives at buf + r*ld + q_off + h*head_stride + d (same for k with k_off).
 * mode 0: RMSNorm over d with learned scale, computed in fp32, rounded to fp16, THEN multiplied by the fp16
 *         scale (hunyuan3ddit.py:83-104).  mode 1: LayerNorm(eps) with weight and bias (attention_blocks.py:315-316,
 *         vggt/layers/attention.py:44-45).  k_w == NULL skips k (geo-decoder query side). */
int r3g_qk_norm(r3g_ctx* ctx, void* buf, int64_t ld, int rows, int heads, int64_t q_off, int64_t k_off,
                int64_t head_stride, int mode, float eps, const void* q_w, const void* q_b, const void* k_w,
                const void* k_b, int seg_len, int64_t seg_stride, void* stream);
/* out[b, :] = W[N,K] . silu?(vec[b, :]) + bias   (tiny-M GEMV: Modulation.lin hunyuan3ddit.py:146-147,
 * MLPEmbedder hunyuan3ddit.py:79-80, LastLayer.adaLN_modulation :275).  fp16 in/out, fp32 accumulate. */
int r3g_gemv(r3g_ctx* ctx, const void* w, const void* bias, const void* vec, int64_t vec_ld, void* out,
             int64_t out_ld, int B, int N, int K, int silu_in, int silu_out, void* stream);
/* SwiGLU gate of the DINOv2-giant conditioner's MLP (Hunyuan3D-2/hy3dgen/shapegen/models/conditioner.py:125-131 runs
 * transformers' Dinov2Model; its Dinov2SwiGLUFFN computes weights_out(silu(x1) * x2) with x1, x2 = weights_in(h).chunk(2)):
 * out[r, j] = fp16(fp16(silu(x[r, j])) * x[r, F + j]) for j < F; x fp16 [rows, >= 2F] (ldx), out fp16 [rows, >= F] (ldo). */
int r3g_swiglu(r3g_ctx* ctx, const void* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int F, void* stream);
/* timestep_embedding(t, 256, time_factor=1000): cat(cos, sin), fp16 out [B,256] (hunyuan3ddit.py:39-60). */
int r3g_timestep_embedding(r3g_ctx* ctx, const void* t_f16, void* out, int B, int dim, float time_factor,
                           float max_period, void* stream);
/* Classifier-free-guidance mix + flow-matching Euler step (pipelines.py:751-756, schedulers.py:300-309):
 *   v = v_uncond + g*(v_cond - v_uncond)  (fp16 arithmetic like the reference), x <- fp16(fp32(x) + dsigma*v).
 * v holds [2*n] halfs (cond first, pipelines.py:752); x holds n halfs; x_dup (optional) receives x twice
 * (the next step's cat([latents]*2), pipelines.py:744). */
int r3g_cfg_euler_step(r3g_ctx* ctx, void* x, const void* v, void* x_dup, int64_t n, float guidance,
                       float dsigma, void* stream);

/* ------------------------------------------------------------------------------------------------
 * SDF decode helpers (VanillaVolumeDecoder + CrossAttentionDecoder, volume_decoders.py:141-182,
 * attention_blocks.py:484-494).
 */
/* Fourier features of the dense grid points [start, start+count) of the (R+1)^3 grid, x slowest / z fastest
 * (generate_dense_grid_points, volume_decoders.py:122-138): coordinates np.linspace(min,max,R+1) in float32,
 * cast to fp16 (volume_decoders.py:168), embedded as cat(x, sin(x*f), cos(x*f)) with f = 2^k (* pi)
 * (attention_blocks.py:113-131) in fp16 arithmetic, zero-padded to out_ld columns. */
int r3g_grid_fourier(r3g_ctx* ctx, void* out, int64_t out_ld, int64_t start, int64_t count, int R,
                     const float* bounds6_host, int num_freqs, int include_pi, void* stream);
/* Same embedding for explicit query points: queries fp16 [n,3] (the `queries=` argument of
 * CrossAttentionDecoder.forward, attention_blocks.py:484-486). */
int r3g_points_fourier(r3g_ctx* ctx, const void* queries, void* out, int64_t out_ld, int64_t n, int num_freqs,
                       int include_pi, void* stream);
/* The same for FLOAT32 query points [n,3]: FlashVDMVolumeDecoding builds its refinement-level queries in float32
 * (volume_decoders.py:395-396) and CrossAttentionDecoder.forward embeds them before casting to the latents' dtype
 * (attention_blocks.py:486), so x * f, sin and cos are float32 arithmetic and only the features are rounded to fp16. */
int r3g_points_fourier_f32(r3g_ctx* ctx, const float* queries, void* out, int64_t out_ld, int64_t n, int num_freqs,
                           int include_pi, void* stream);
/* logits[r] = float(fp16( LN(x[r,:]; w,b,eps) . w_out + b_out ))  -- ln_post + output_proj
 * (attention_blocks.py:491-493), written to the float32 grid at out[r]. */
int r3g_lnpost_dot(r3g_ctx* ctx, const void* x, int64_t ldx, int rows, int width, float eps, const void* ln_w,
                   const void* ln_b, const void* w_out, const void* b_out, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * VGGT DPT depth head (vggt/vggt/heads/dpt_head.py:172-291) on channels-last fp16 feature maps: 1x1 convolutions and the
 * kernel == stride transposed convolutions are r3g_linear on the [N*H*W, C] rows; a 3x3 convolution (padding 1) is
 *   r3g_im2col3x3: cols[(n,yo,xo), (ky*3+kx)*C + c] = relu?(x[n, yo*stride+ky-1, xo*stride+kx-1, c]) (0 outside) -> r3g_linear
 * with the weight permuted to [C_out, (ky, kx, C_in)]; Ho = (H - 1) / stride + 1.  r3g_bilinear_nhwc is
 * F.interpolate(mode="bilinear", align_corners=True) (custom_interpolate, dpt_head.py:459-484).  C % 8 == 0. */
int r3g_im2col3x3(r3g_ctx* ctx, const void* x, void* cols, int N, int H, int W, int C, int stride, int relu_in, void* stream);
int r3g_bilinear_nhwc(r3g_ctx* ctx, const void* x, void* out, int N, int Hi, int Wi, int Ho, int Wo, int C, void* stream);

/* ------------------------------------------------------------------------------------------------
 * VGGT camera head (vggt/vggt/heads/camera_head.py:73-141).  The reference runs it in float32 outside autocast on S pose
 * tokens (S = frames), so every nn.Linear is a GEMV over its weight matrix (HBM-bound): weights fp16, everything else
 * float32.
 *   r3g_gemv_f32:  out[b,n] = res[b,n] + gamma[n] * g( W[n,:] . a(vec[b,:]) + bias[n] )   (res, gamma, bias optional;
 *       a = SiLU if act_in == 1 (poseLN_modulation, :113), g = exact GELU if act_out == 1 (Mlp fc1, vggt/layers/mlp.py:22);
 *       res + gamma * y is Block's LayerScale residual, vggt/layers/block.py:77-98).  B <= 8 rows, K % 8 == 0.
 *   r3g_layernorm_f32:  y = LN(x; w, b, eps); with shift / scale / gate (float32 [rows, >= width], stride mod_ld):
 *       y = gate * (LN(x) * (1 + scale) + shift) + x   (camera_head.py:116-120).
 *   r3g_small_attention_f32:  softmax(q k^T * scale) v over S <= 64 tokens, qkv float32 [B*S, 3*H*D] laid out (3, H, D)
 *       (vggt/layers/attention.py:52-61), out float32 [B*S, H*D]; D in {32, 64, 128, 256} (the trunk has 16 heads of 128). */
int r3g_gemv_f32(r3g_ctx* ctx, const void* w_f16, const float* bias, const float* vec, int64_t vec_ld, float* out,
                 int64_t out_ld, const float* residual, const float* gamma, int B, int N, int K, int act_in, int act_out,
                 void* stream);
int r3g_layernorm_f32(r3g_ctx* ctx, const float* x, int64_t ldx, float* y, int64_t ldy, int rows, int width, float eps,
                      const float* w, const float* b, const float* shift, const float* scale, const float* gate,
                      int64_t mod_ld, void* stream);
int r3g_small_attention_f32(r3g_ctx* ctx, const float* qkv, float* out, int B, int S, int H, int D, float scale,
                            void* stream);

/* ------------------------------------------------------------------------------------------------
 * Back-projection.  Replaces the per-pixel work of unproject_depth_map_to_point_map
 * (vggt/vggt/utils/geometry.py:15-117): depth float32 [S,H,W] on the device (the reference squeezes a trailing 1).
 * cam_to_world_host: float64 [S,3,4] = rows 0..2 of closed_form_inverse_se3(extrinsic) (geometry.py:74-77) --
 * the 3x4 inverse is S tiny matrices computed by the host mirror with numpy exactly as the reference does (its
 * float32 matmul rounding is BLAS-dependent, so it is not re-derived here).  intrinsic_host float32 [S,3,3].
 * out [S,H,W,3] float64 (out_f64=1, the reference's result dtype) or float32. */
int r3g_unproject(r3g_ctx* ctx, const float* depth, const double* cam_to_world_host, const float* intrinsic_host,
                  void* out, int S, int H, int W, int out_f64, void* stream);

#ifdef __cplusplus
}
#endif
#endif
