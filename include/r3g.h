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
 *   - Programmatic dependent launch (PDL): r3g_linear, r3g_attention, r3g_layernorm, r3g_lnpost_dot, r3g_gemv,
 *     r3g_swiglu, r3g_gemv_f32, r3g_layernorm_f32, r3g_small_attention_f32, r3g_im2col3x3 and r3g_bilinear_nhwc launch
 *     their kernels with the programmatic-stream-serialization attribute, eagerly and under CUDA-graph capture, so a
 *     kernel's prologue may run under the tail of the kernel before it in the stream.  Each waits (griddepcontrol.wait)
 *     for that kernel to complete before it touches memory another kernel produces or still reads, with two
 *     exceptions: r3g_layernorm reads w and b, and r3g_lnpost_dot reads ln_w, ln_b and w_out, before the wait.  The
 *     launch immediately before either of them in the stream must therefore not write those buffers.  The r3g_linear
 *     and r3g_attention prologues touch only kernel parameters and shared memory.  The environment variable R3G_PDL,
 *     read once per context when it first launches such a kernel, controls this: unset or any value not starting with
 *     '0' enables PDL, "0" launches every kernel in plain stream order.  Results are the same bits either way.
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
 *
 * method: R3G_MC_LEWINER is the marching cubes above.  R3G_MC_DUAL is r3g's own dual marching cubes, the surface
 * extractor behind DMCSurfaceExtractor.run (surface_extractors.py:79-94, which calls diso.DiffDMC on -grid / R; diso's
 * vertex rule, quad split and output order are not reproduced).  Same count / extract protocol and workspace:
 *   - a point is above iff v > level (NaN is not), and each crossed cell takes the Lewiner tiling chosen above;
 *   - each connected component ("patch") of that tiling's triangles (joined through shared edge vertices and the
 *     centre vertex) gives one vertex: the mean of the crossings p_a + t (p_b - p_a), t = v_a / (v_a - v_b), on the
 *     patch's cube edges, summed in increasing edge order, divided by (n_axis - 1): float64 with explicit rounding,
 *     stored float32 in array-axis order, so the mesh lies in [0, 1]^3.  Vertices follow the crossed cells in
 *     traversal order, patches within a cell by their smallest cube edge;
 *   - each sign-changing grid edge whose four incident cells lie in the grid gives one quad over their four patch
 *     vertices, wound with its normal towards increasing values (the Lewiner method's winding), split along the
 *     shorter diagonal (squared float64 lengths; a tie takes vertices 0-2) into two consecutive triangles.  Quads follow
 *     their owner cell (the first of the four) in traversal order, then the edge's array axis 0, 1, 2.  Edges on the
 *     grid's outer faces give none, so a surface that reaches the boundary is open there.
 *   r3g_mc_count returns R3G_E_NOSURFACE when no cell is crossed and applies no level-range check; r3g_mc_extract
 *   requires bounds_host == NULL (R3G_E_INVALID otherwise).  Any other method is R3G_E_INVALID.
 */
enum { R3G_MC_LEWINER = 0, R3G_MC_DUAL = 1 };
size_t r3g_mc_workspace_bytes(int n0, int n1, int n2);
int r3g_mc_count(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level, int method, void* workspace,
                 size_t workspace_bytes, int64_t* nv_host, int64_t* nf_host, void* stream);
int r3g_mc_extract(r3g_ctx* ctx, const float* grid, int n0, int n1, int n2, float level, int method,
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

/* Decimation -- quadric edge-collapse mesh reduction on the device, the face reduction of stage 3
 * (src/2d_to_3d_models/run.py:95: FaceReducer, Hunyuan3D-2/hy3dgen/shapegen/postprocessors.py:37-51,118-128, pymeshlab
 * meshing_decimation_quadric_edge_collapse to 40 000 faces with qualitythr 1, preserveboundary, boundaryweight 3,
 * preservenormal, preservetopology, autoclean).  The algorithm below is r3g's own, not MeshLab's collapse order; it is
 * deterministic and pinned bit for bit by the numpy mirror oracle/decimate.py.
 *
 * Algorithm: rounds of independent edge collapses.
 *   Quadrics (float64, computed once from the input): every non-degenerate face adds u u^T / |n| with n = (p1-p0) x (p2-p0),
 *     u = (n, -n.p0) -- the plane quadric weighted by twice the face area; every boundary edge (one face) from corner j to
 *     j+1 adds 3 (e.e) m m^T / (m.m) with e = p_{j+1} - p_j, m = e x n, the plane (m, -m.p_j) through the edge
 *     perpendicular to its face.  A vertex sums the terms of its faces in ascending face order, each face's own plane
 *     before its boundary edges in corner order.  A collapse gives the kept vertex Q_a + Q_b.
 *   Placement: p minimises v^T Q v (v = (p, 1)) by the adjugate of Q's 3x3 block when |det| > 1e-6 trace^3; otherwise the
 *     cheapest of a, b and (a + b) / 2 (ties to the earlier).  err = max(v^T Q v, 0).
 *   Cost: (err + 1e-4 |a-b|^4) / clamp(min quality, 1e-3, 1), over the faces around a or b that survive with the endpoint
 *     moved to p; quality = 2 sqrt(3) |n| / (sum of squared edge lengths) (1 for an equilateral triangle).  Rounded up to
 *     float32; key = (float32 bits << 32) | edge index, edges numbered in ascending (min vertex, max vertex) order.
 *   Validity (an invalid edge waits for a later round): at most two faces on the edge and neither endpoint on an edge of
 *     more (frozen); not an interior edge between two boundary vertices; link condition (a and b have exactly as many
 *     common neighbours as the edge has faces); the component keeps at least 4 vertices; no surviving face around a or b
 *     with a non-zero normal flips (old normal . new normal <= 0 rejects; a zero-area face, such as marching cubes
 *     leaves where the field is 0 at a grid point, constrains nothing and so can be collapsed away).
 *   Selection: m(v) = min key of the valid edges at v, M(v) = min of m over v's closed 1-ring; an edge is collapsed iff
 *     key == M(a) == M(b).  Selected edges share no faces and no adjacent endpoints, so the tests above stay true while
 *     they are applied together, in any thread order.  A component that would fall under 4 vertices keeps only its
 *     cheapest selected edge.  When more than ceil((nf - target) / 2) edges remain selected, only that many of the
 *     cheapest are applied, so the face count ends at target or target - 1.
 *   Apply: the smaller endpoint index survives at p, the edge's faces die, the other faces keep their winding.
 *   The rounds stop when nf <= target or no edge is selectable (then the result is the smallest mesh the rules allow).
 *   Output: surviving vertices and faces compacted in their original relative order, positions rounded to float32; faces
 *     with a repeated index and unreferenced vertices are dropped.
 *
 * r3g_decimate_workspace_bytes: the device workspace r3g_mesh_decimate needs for a mesh of nv vertices and nf faces
 *   (pure arithmetic, no device): about 170 bytes per vertex and 310 per face (0.1 GB at 222 000 faces); 0 for sizes
 *   r3g_mesh_decimate refuses.
 * r3g_mesh_decimate: verts float32 [nv][3], faces int32 [nf][3] -> verts_out float32 [*nv_out_host][3], faces_out
 *   int32 [*nf_out_host][3] (capacities nv and nf); target >= 0.  *rounds_host (if not NULL) receives the number of
 *   collapse rounds.  SYNCHRONISES `stream` (the host loop reads the face count every round).  An index outside
 *   [0, nv), nv > 2^31 - 1 or 3 nf > 2^31 - 1 returns R3G_E_INVALID; a workspace under
 *   r3g_decimate_workspace_bytes(nv, nf), R3G_E_WORKSPACE. */
size_t r3g_decimate_workspace_bytes(int64_t nv, int64_t nf);
int r3g_mesh_decimate(r3g_ctx* ctx, const float* verts, int64_t nv, const int32_t* faces, int64_t nf, int64_t target,
                      void* workspace, size_t workspace_bytes, float* verts_out, int32_t* faces_out,
                      int64_t* nv_out_host, int64_t* nf_out_host, int64_t* rounds_host, void* stream);

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
 *        This form takes no gate: gate != NULL with residual_f32 is R3G_E_INVALID.
 *   qkn_*: the per-head q/k normalisation that follows a q/k/v projection, fused into the epilogue (the accumulator
 *        row of a 64-column head sits in one thread's registers): qkn_mode 1 = RMSNorm(64) with a learned scale
 *        (QKNorm, hunyuan3ddit.py:83-104,199,260), 2 = LayerNorm(64) with weight + bias (attention_blocks.py:315-316,
 *        250-258).  It is applied to the fp16-rounded Linear output of the 64-column heads in
 *        [qkn_q_col0, qkn_q_col0 + qkn_cols) with (qkn_q_w, qkn_q_b) and, if qkn_k_col0 >= 0, of
 *        [qkn_k_col0, qkn_k_col0 + qkn_cols) with (qkn_k_w, qkn_k_b); the weights are fp16 [64] (bias NULL in mode 1).
 *        Column offsets and qkn_cols are multiples of 64; these columns must carry no activation / gate / residual.
 *   group_next: a further, independent problem (its own x / w / y / epilogue operands and sizes) whose tiles share
 *        this call's grid; a chain holds at most three problems (the third's group_next must be NULL).  The img and txt
 *        streams of a DoubleStreamBlock apply different weights to 6144 and 2740 rows (hunyuan3ddit.py:196-216):
 *        separately their N = 1024 projections fill 1.45 and 0.67 waves of 128 x 256 tiles on 132 SMs, together 2.1
 *        of 3.  With the unconditional text collapsed to one row (r3g_attention windows) the txt stream is two
 *        problems, batch 0's 1370 rows and batch 1's single row: img + both fill 240 of the 264 tiles of 2 waves.
 *        Results are those of separate calls.
 *   moe_*: the mixture-of-experts FFN of HunYuanDiTPlain's last blocks (moe_layers.py:50-151) without a host sync, in
 *        three modes.  moe_mode 0 ignores every moe_* field.  Slot buffers hold one fixed-capacity segment of
 *        moe_cap rows per group: group g's rows are rows [g * moe_cap, g * moe_cap + count_g).  A mode-1 or mode-3 call
 *        takes no group_next, activation, gate, qkn or fp32 operands; its launches are plain stream-ordered (no PDL).
 *     1 route (MoEGate.forward, :50-68): x [M, K] the LayerNorm rows, w [N, K] the gate weight with N = moe_experts
 *        <= 64, y fp16 [M, N] receives the logits fp16(x . w^T) (bias must be NULL).  Per row, scores =
 *        fp16(softmax(logits)) in fp32, then the moe_top_k highest scores (equal scores: lower expert first; the weights
 *        are not renormalised).  For each of them, in decreasing score order j: moe_ids[r * top_k + j] = e,
 *        moe_weights[...] = the fp16 score, a position p in e's segment (from an atomic counter: the order of rows
 *        inside a segment varies between runs), moe_slots[...] = e * moe_cap + p, moe_slot_scale[e * moe_cap + p] =
 *        the score, and x's row is copied to row e * moe_cap + p of moe_slot_x (fp16, K columns, leading dimension
 *        K).  moe_counts (int32 [moe_experts]) is zeroed by the call and ends holding each expert's row count.
 *        moe_cap >= M (an expert takes a row at most once).  Rows whose logits are not all finite still get moe_top_k
 *        distinct experts in [0, moe_experts): a NaN score ranks above every number (torch.topk's order), NaNs among
 *        themselves lower expert first, and a NaN pick's weight is that NaN.  A NaN in x, or a logit that rounds to
 *        +inf, makes every score of the row NaN, so such a row takes experts 0 .. moe_top_k - 1 with NaN weights; a
 *        logit of -inf next to a finite one gives its expert score 0.
 *     2 grouped: moe_groups independent GEMMs in one launch, group g = x rows [g * moe_cap, ...) (ldx) against
 *        w[g] (w is [moe_groups, N, K]) plus bias[g] (bias [moe_groups, N] or NULL), written to the same rows of y
 *        (ldy), with act 0 or 2 (erf-GELU) over all columns.  Groups g < moe_experts have moe_counts[g] rows, read on
 *        the device; the others have M rows (the shared expert's identity rows); M = moe_cap.  The grid covers moe_cap
 *        rows of every group and the CTAs past a group's count exit.  moe_slot_scale (fp16 [moe_groups * moe_cap] or
 *        NULL) scales each row after the fp16 rounding: y = fp16(fp16(acc + bias) * scale[row]).
 *     3 combine: y = fp16(residual + fp16(fp16(routed) + fp16(acc + bias))) over M rows, where routed is the fp16
 *        sum, from 0 in increasing expert order, of rows moe_slots[r * top_k + j] of moe_slot_y (fp16 [*, N],
 *        leading dimension N), the weighted expert outputs of mode 2 (expert_cache + shared_experts(identity), then
 *        the block's residual, moe_layers.py:105-106, hunyuandit.py:351-352).  residual (ldy) may alias y.
 *        Every row's result is independent of the segment positions route chose, so repeated runs agree bit for bit.
 */
enum { R3G_MOE_ROUTE = 1, R3G_MOE_GROUPED = 2, R3G_MOE_COMBINE = 3 };
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
  int moe_mode, moe_groups, moe_experts, moe_top_k, moe_cap;
  int32_t* moe_counts;       /* int32 [moe_experts] */
  int32_t* moe_ids;          /* int32 [M, moe_top_k] */
  void* moe_weights;         /* fp16 [M, moe_top_k] */
  int32_t* moe_slots;        /* int32 [M, moe_top_k] */
  void* moe_slot_x;          /* fp16 [moe_experts * moe_cap, K] */
  void* moe_slot_scale;      /* fp16 [moe_groups * moe_cap] */
  const void* moe_slot_y;    /* fp16 [moe_experts * moe_cap, N] */
} r3g_linear_args;
int r3g_linear(r3g_ctx* ctx, const r3g_linear_args* a, void* stream);

/* r3g_attention: O = softmax(Q K^T * scale) V, no mask (F.scaled_dot_product_attention call sites:
 * hunyuan3ddit.py:33-36, attention_blocks.py:328, attention_processors.py:29-32, vggt/layers/attention.py:61).
 * head_dim is 64.  Q/K/V/O are addressed by strides in halfs: element (b, h, l, d) at
 * base + b*stride_b + h*stride_h + l*stride_l + d.  O has the "B L (H D)" layout of hunyuan3ddit.py:35 when
 * o_stride_l = H*64, o_stride_h = 64.  O may alias Q (each CTA reads its Q tile before writing it).
 * Windows (self-attention only, Lq == Lk, B <= R3G_ATTN_MAX_WINDOWS): if win_len[0] > 0, batch b computes and writes
 *   only the query rows [win_row0[b], win_row0[b] + win_len[b]) (the other rows of O are left as they are); every query
 *   still attends all Lk keys.  If win_k0_count[b] = n > 1, the window's first row stands for n equal rows: the call
 *   first overwrites rows [win_row0[b] - n + 1, win_row0[b]) of K and V with K and V of row win_row0[b] (in place, through
 *   the k / v pointers), so the result is attention over n copies of that key, bit for bit.  The DiT's unconditional
 *   CFG sample, whose Lt text rows are equal (hunyuan3ddit.py:33-36 with an all-equal text context), computes only its
 *   last text row and the latents this way.  All batches share one launch.  Zeroed windows: plain attention over
 *   [0, Lq). */
#define R3G_ATTN_MAX_WINDOWS 2
typedef struct {
  const void* q; int64_t q_sb, q_sh, q_sl;
  const void* k; int64_t k_sb, k_sh, k_sl;
  const void* v; int64_t v_sb, v_sh, v_sl;
  void* o; int64_t o_sb, o_sh, o_sl;
  int B, H, Lq, Lk;
  float scale;
  int win_row0[R3G_ATTN_MAX_WINDOWS], win_len[R3G_ATTN_MAX_WINDOWS], win_k0_count[R3G_ATTN_MAX_WINDOWS];
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
 *         vggt/layers/attention.py:44-45).  mode 2: torch's nn.RMSNorm(64, eps) (HunYuanDiTPlain's q/k norms,
 *         hunyuandit.py:153,256,491): fp16(x * rrms * w) with x * rrms * w in fp32, one rounding, where mode 0 rounds
 *         x * rrms before the scale.  Other modes are R3G_E_INVALID.  k_w == NULL skips k (geo-decoder query side). */
int r3g_qk_norm(r3g_ctx* ctx, void* buf, int64_t ld, int rows, int heads, int64_t q_off, int64_t k_off,
                int64_t head_stride, int mode, float eps, const void* q_w, const void* q_b, const void* k_w,
                const void* k_b, int seg_len, int64_t seg_stride, void* stream);
/* out[b, :] = W[N,K] . silu?(vec[b, :]) + bias   (tiny-M GEMV: Modulation.lin hunyuan3ddit.py:146-147,
 * MLPEmbedder hunyuan3ddit.py:79-80, LastLayer.adaLN_modulation :275).  fp16 in/out, fp32 accumulate.
 * residual (optional, fp16 [B, N] at out_ld; it may alias out): out = fp16(fp16(W . silu?(vec) + bias [, silu]) +
 * residual), the `vec = vec + guidance_in(...)` of a guidance-distilled model (hunyuan3ddit.py:392-396) in fp16.
 * residual == NULL writes the GEMV result alone.  out may alias neither vec nor w. */
int r3g_gemv(r3g_ctx* ctx, const void* w, const void* bias, const void* vec, int64_t vec_ld, void* out,
             int64_t out_ld, const void* residual, int B, int N, int K, int silu_in, int silu_out, void* stream);
/* SwiGLU gate of the DINOv2-giant conditioner's MLP (Hunyuan3D-2/hy3dgen/shapegen/models/conditioner.py:125-131 runs
 * transformers' Dinov2Model; its Dinov2SwiGLUFFN computes weights_out(silu(x1) * x2) with x1, x2 = weights_in(h).chunk(2)):
 * out[r, j] = fp16(fp16(silu(x[r, j])) * x[r, F + j]) for j < F; x fp16 [rows, >= 2F] (ldx), out fp16 [rows, >= F] (ldo). */
int r3g_swiglu(r3g_ctx* ctx, const void* x, int64_t ldx, void* out, int64_t ldo, int64_t rows, int F, void* stream);
/* timestep_embedding(t, 256, time_factor=1000): cat(cos, sin), fp16 out [B,256] (hunyuan3ddit.py:39-60). */
int r3g_timestep_embedding(r3g_ctx* ctx, const void* t_f16, void* out, int B, int dim, float time_factor,
                           float max_period, void* stream);
/* Classifier-free-guidance mix + flow-matching Euler step (pipelines.py:751-756, schedulers.py:300-309):
 *   v = v_uncond + g*(v_cond - v_uncond)  (fp16 arithmetic like the reference), x <- fp16(fp32(x) + fp16(dsigma*v)).
 * nb is the number of samples in v.  nb = 2: v holds [2*n] halfs (cond first, pipelines.py:752), mixed as above.
 * nb = 1: v holds n halfs, the prediction of a model run without CFG (pipelines.py:708-711, a guidance-distilled model
 * or guidance_scale < 0); guidance is ignored and the step is the plain Euler update of schedulers.py:300-309 /
 * ConsistencyFlowMatchEulerDiscreteScheduler's schedulers.py:462-469.  x holds n halfs; x_dup (optional) receives x nb
 * times (the next step's model input, cat([latents]*2) or latents, pipelines.py:742-745).  dsigma is the caller's
 * fp16-rounded sigma_next - sigma.  x, v and x_dup must not overlap. */
int r3g_cfg_euler_step(r3g_ctx* ctx, void* x, const void* v, void* x_dup, int64_t n, int nb, float guidance,
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
