"""Torch-tensor front end of the C ABI (include/r3g.h).  Torch is plumbing only: it owns device memory
and the stream; every computation below happens in libr3g.so.  No fallback paths."""
import ctypes as C
import math

import numpy as np
import torch

from . import _abi

ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_RELU = 0, 1, 2, 3


def _ptr(t, dev, op, arg):
    """The address of tensor `t` (None: NULL), which must live on CUDA device `dev`: the library cannot tell a host or
    foreign-device address from its own, so one would fault the kernel instead of raising here."""
    if t is None:
        return None
    if t.get_device() != dev:
        raise ValueError(f"{op}: argument {arg} must be a tensor on cuda:{dev}, got one on {t.device}")
    return t.data_ptr()


# the void* parameters of each entry point between the context and the stream (0-based).  Only they take a tensor:
# one in an integer slot reaches ctypes unconverted and is refused there, and _launch looks at a few arguments instead
# of all of them (the wrappers' host cost is on the timed path of the eager conditioner and ShapeVAE)
_PTR_ARGS = {name[len("r3g_"):]: [i for i, t in enumerate(argtypes[1:-1]) if t is C.c_void_p]
             for name, (_, argtypes) in _abi.SIGNATURES.items()}


def _launch(name, anchor, *args):
    """r3g_<name>(ctx, *args, stream) with the r3g context of the anchor tensor's device and torch's current stream OF
    THAT DEVICE (GraphCache captures on a side stream of the inputs' device).  The library switches to that device for
    the duration of each call (r3g_device_guard), so a pipeline on cuda:1 works without torch.cuda.set_device(1).
    A tensor argument is passed as its address (_ptr; argument i is the i-th after the context), None as NULL and
    anything else as it is.  A failed call raises R3GError with the library's return code."""
    if not anchor.is_cuda:
        raise RuntimeError("r3g ops need CUDA tensors: there is no CPU fallback")
    dev = anchor.get_device()
    ctx = _abi.get_context(dev)
    ptrs = list(args)
    for i in _PTR_ARGS[name]:
        if isinstance(ptrs[i], torch.Tensor):
            ptrs[i] = _ptr(ptrs[i], dev, name, i + 1)
    ctx.check(getattr(ctx.lib, "r3g_" + name)(ctx.handle, *ptrs, torch.cuda.current_stream(dev).cuda_stream))


def _out(op, out, shape, dtype, like, contiguous=False, rows=False):
    """The buffer `op` writes.  None: a new `dtype` tensor of `shape` on `like`'s device.  Otherwise `out`, once it is
    checked to be a `dtype` tensor on that device of exactly `shape` with unit inner stride (contiguous=True: fully
    contiguous, for kernels given no leading dimension).  rows=True asks only for the rows x width of `shape`, for a
    buffer whose layout _rows then describes."""
    if out is None:
        return torch.empty(shape, device=like.device, dtype=dtype)
    if rows:
        ok = out.shape[-1] == shape[-1] and out.numel() == math.prod(shape)
    else:
        ok = out.shape == shape and (out.is_contiguous() if contiguous else out.stride()[-1] == 1)
    if not ok or out.dtype != dtype or out.get_device() != like.get_device():
        raise ValueError(f"{op}: out must be {'contiguous ' if contiguous else ''}{dtype} {tuple(shape)} on "
                         f"{like.device}, got {out.dtype} {tuple(out.shape)} strides {out.stride()} on {out.device}")
    return out


def _f16(t, name):
    if t.dtype != torch.float16:
        raise TypeError(f"{name} must be float16, got {t.dtype}")
    return t


def _rows(t, name, segments=True):
    """Describe an activation as segmented rows.  Accepts [..., W] contiguous, a 2-D strided view [M, W], or a
    3-D view [S, L, W] whose segments are `stride(0)` apart (e.g. X[:, Lt:, :] of a joint txt+img buffer; not with
    segments=False, for kernels that take one row stride).  Row 0 is at t's address.
    Returns (rows, width, ld, seg_len, seg_stride_rows)."""
    if t.stride()[-1] != 1:
        raise ValueError(f"{name}: innermost stride must be 1")
    w = t.shape[-1]
    if t.dim() == 1:
        return 1, w, w, 0, 0
    if t.is_contiguous():
        return t.numel() // w, w, w, 0, 0
    if t.dim() == 2:
        return t.shape[0], w, t.stride(0), 0, 0
    if t.dim() == 3:
        S, L, _ = t.shape
        ld = t.stride(1)
        if S == 1:
            return L, w, ld, 0, 0
        if segments:
            if t.stride(0) % ld:
                raise ValueError(f"{name}: segment stride must be a multiple of the row stride")
            return S * L, w, ld, L, t.stride(0) // ld
    raise ValueError(f"{name}: cannot describe as {'(segmented)' if segments else 'evenly spaced'} rows without a copy")


def _merge_seg(xs, ys, name):
    """x and y must agree on the segmentation (or one of them is unsegmented)."""
    (xl, xst, xrows), (yl, yst) = xs, ys
    if xl == 0 and yl == 0:
        return 0, 0, 0
    L = xl or yl
    if (xl and yl and xl != yl) or xrows % L:
        raise ValueError(f"{name}: input and output segment lengths differ")
    return L, (xst if xl else L), (yst if yl else L)


QKN_RMS, QKN_LAYERNORM = 1, 2


def _linear_args(dev, x, w, bias=None, *, out=None, act=ACT_NONE, act_cols=None, gate=None, gate_rows=0, residual=None,
                 ls_gamma=None, out_dtype=torch.float16, qk_norm=None):
    """Build one r3g_linear_args whose tensors live on CUDA device `dev`; returns (struct, out tensor)."""
    _f16(x, "x"); _f16(w, "w")
    M, K, ldx, xl, xst = _rows(x, "x")
    N = w.shape[0]
    if w.shape[1] != K or not w.is_contiguous():
        raise ValueError("w must be contiguous [N, K]")
    if out is not None and out.dtype in (torch.float16, torch.float32):
        out_dtype = out.dtype       # the kernel writes whichever of the two `out` holds; out_dtype types a new out
    out = _out("linear", out, (*x.shape[:-1], N), out_dtype, x, rows=True)
    _, _, ldy, yl, yst = _rows(out, "out")
    seg_len, xs, ys = _merge_seg((xl, xst, M), (yl, yst), "linear")
    a = _abi.LinearArgs()
    a.x, a.ldx = _ptr(x, dev, "linear", "x"), ldx
    a.w, a.bias = _ptr(w, dev, "linear", "w"), _ptr(bias, dev, "linear", "bias")
    a.y, a.ldy = _ptr(out, dev, "linear", "out"), ldy
    a.M, a.N, a.K = M, N, K
    a.seg_len, a.x_seg_stride, a.y_seg_stride = seg_len, xs, ys
    a.act = act
    a.act_col0, a.act_col1 = act_cols if act_cols is not None else (0, N)
    if ls_gamma is not None and (residual is None or residual.dtype != torch.float32):
        raise ValueError("linear: ls_gamma scales the float32-residual form only; pass a float32 residual")
    if gate is not None:
        _f16(gate, "gate")
        a.gate, a.gate_ld, a.gate_rows = _ptr(gate, dev, "linear", "gate"), gate.stride(0), gate_rows
    if residual is not None:
        if residual.dtype == torch.float32:
            a.residual_f32 = 1
            if ls_gamma is not None:
                if ls_gamma.dtype != torch.float32 or ls_gamma.numel() != N:
                    raise TypeError("ls_gamma must be float32 [N]")
                a.ls_gamma = _ptr(ls_gamma, dev, "linear", "ls_gamma")
        else:
            _f16(residual, "residual")
        _, _, ldr, rl, rst = _rows(residual, "residual")
        if ldr != ldy or (rl, rst) != (yl, yst):
            raise ValueError("residual must share out's geometry")
        a.residual = _ptr(residual, dev, "linear", "residual")
    a.out_f32 = 1 if out.dtype == torch.float32 else 0
    if qk_norm is not None:
        a.qkn_mode, a.qkn_q_col0, a.qkn_cols = qk_norm["mode"], qk_norm["q_col0"], qk_norm["cols"]
        a.qkn_k_col0 = qk_norm["k_col0"] if qk_norm.get("k_col0") is not None else -1
        a.qkn_eps = float(qk_norm["eps"])
        for name in ("q_w", "q_b", "k_w", "k_b"):
            t = qk_norm.get(name)
            if t is not None:
                _f16(t, name)
                if t.numel() != 64 or not t.is_contiguous():
                    raise ValueError(f"qk_norm {name} must be a contiguous fp16 [64]")
                setattr(a, "qkn_" + name, _ptr(t, dev, "linear", "qk_norm " + name))
    return a, out


def linear(x, w, bias=None, **kw):
    """Y = epilogue(X W^T + bias); see r3g_linear in include/r3g.h.

    x: [..., K] or a strided [M, K] / [S, L, K] view, w: [N, K] contiguous, out: same row structure, width N.
    gate: [B, N] view with unit inner stride, applied to logical rows b = r // gate_rows.
    residual must be the same view geometry as out (and may be out itself).
    qk_norm: dict(mode=QKN_RMS|QKN_LAYERNORM, q_col0, k_col0 (None: q only), cols, eps, q_w, q_b, k_w, k_b) -- the per-head
    q/k normalisation fused into the epilogue (see qkn_* in include/r3g.h).
    """
    a, out = _linear_args(x.get_device(), x, w, bias, **kw)
    _launch("linear", x, C.byref(a))
    return out


def linear_group(*problems):
    """One to three independent linears in ONE launch (r3g_linear_args.group_next): each problem is a dict of linear()'s
    arguments (x, w, bias, out, ...).  Results are those of linear(**p) for each p, returned in order; the tiles of all
    problems share one grid -- the img and txt streams of a DoubleStreamBlock fill the machine together."""
    if not 1 <= len(problems) <= 3:
        raise ValueError(f"linear_group: 1 to 3 problems, got {len(problems)}")
    dev = problems[0]["x"].get_device()
    args, outs = zip(*[_linear_args(dev, **p) for p in problems])
    for a, nxt in zip(args, args[1:]):
        a.group_next = C.addressof(nxt)
    _launch("linear", problems[0]["x"], C.byref(args[0]))
    return outs


def linear_pair(first, second):
    """linear_group of two problems: the results of linear(**first), linear(**second) from one launch."""
    return linear_group(first, second)


MOE_ROUTE, MOE_GROUPED, MOE_COMBINE = 1, 2, 3


def _moe_buf(t, dev, name, dtype, numel):
    """A contiguous `dtype` buffer of at least `numel` elements on cuda:dev, as its address."""
    if t.dtype != dtype or not t.is_contiguous() or t.numel() < numel:
        raise ValueError(f"moe: {name} must be a contiguous {dtype} buffer of at least {numel} elements, got "
                         f"{t.dtype} {tuple(t.shape)}")
    return _ptr(t, dev, "linear", name)


def moe_route(x, w, *, top_k, cap, slot_x, slot_scale, counts, ids, weights, slots, out=None):
    """MoEGate.forward and the dispatch of its rows (r3g_linear moe_mode 1, include/r3g.h).  x: [M, K] rows, w: the gate
    weight [E, K] (E <= 64); out: fp16 [M, E] logits.  Writes ids / slots int32 [M, top_k], weights fp16 [M, top_k],
    counts int32 [E], and each chosen (row, expert) copy of x into slot_x [E * cap, K] with its weight in slot_scale."""
    dev = x.get_device()
    a, out = _linear_args(dev, x, w, out=out)
    E, K, M = w.shape[0], w.shape[1], a.M
    a.moe_mode, a.moe_experts, a.moe_top_k, a.moe_cap = MOE_ROUTE, E, top_k, cap
    a.moe_counts = _moe_buf(counts, dev, "counts", torch.int32, E)
    a.moe_ids = _moe_buf(ids, dev, "ids", torch.int32, M * top_k)
    a.moe_weights = _moe_buf(weights, dev, "weights", torch.float16, M * top_k)
    a.moe_slots = _moe_buf(slots, dev, "slots", torch.int32, M * top_k)
    a.moe_slot_x = _moe_buf(slot_x, dev, "slot_x", torch.float16, E * cap * K)
    a.moe_slot_scale = _moe_buf(slot_scale, dev, "slot_scale", torch.float16, E * cap)
    _launch("linear", x, C.byref(a))
    return out


def moe_grouped(x, w, bias=None, *, counts, experts, out, act=ACT_NONE, row_scale=None):
    """G = w.shape[0] GEMMs in one launch (r3g_linear moe_mode 2): x [G * cap, K] holds one cap-row segment per group,
    w [G, N, K], bias [G, N]; group g < experts has counts[g] rows (read on the device), the others cap; out [G * cap,
    N] receives fp16(act(x w[g]^T + bias[g])), times row_scale[row] (fp16 [G * cap]) after the rounding if given."""
    G, N, K = w.shape
    if x.dim() != 2 or x.shape[0] % G or not w.is_contiguous():
        raise ValueError("moe_grouped: x must be [G * cap, K] and w a contiguous [G, N, K]")
    dev = x.get_device()
    if bias is not None and (tuple(bias.shape) != (G, N) or not bias.is_contiguous()):
        raise ValueError(f"moe_grouped: bias must be a contiguous [{G}, {N}]")
    cap = x.shape[0] // G
    if out is None or tuple(out.shape) != (G * cap, N):
        raise ValueError(f"moe_grouped: out must be [{G * cap}, {N}]")
    # group 0's operands describe the launch; the kernel addresses group g at g times their sizes
    a, _ = _linear_args(dev, x[:cap], w[0], None if bias is None else bias[0], out=out[:cap], act=act)
    a.moe_mode, a.moe_groups, a.moe_experts, a.moe_cap = MOE_GROUPED, G, experts, cap
    if experts:
        a.moe_counts = _moe_buf(counts, dev, "counts", torch.int32, experts)
    if row_scale is not None:
        a.moe_slot_scale = _moe_buf(row_scale, dev, "row_scale", torch.float16, G * cap)
    _launch("linear", x, C.byref(a))
    return out


def moe_combine(x, w, bias, *, slot_y, ids, slots, residual, out):
    """The shared expert's second Linear with the MoE sum and the block residual fused (r3g_linear moe_mode 3):
    out = fp16(residual + fp16(routed + fp16(x w^T + bias))), routed = the fp16 sum, in increasing expert order, of the
    rows slots[r] of slot_y (the weighted expert outputs)."""
    dev = x.get_device()
    a, out = _linear_args(dev, x, w, bias, out=out, residual=residual)
    top_k = ids.shape[-1]
    a.moe_mode, a.moe_top_k = MOE_COMBINE, top_k
    a.moe_ids = _moe_buf(ids, dev, "ids", torch.int32, a.M * top_k)
    a.moe_slots = _moe_buf(slots, dev, "slots", torch.int32, a.M * top_k)
    if slot_y.shape[-1] != a.N or not slot_y.is_contiguous() or slot_y.dtype != torch.float16:
        raise ValueError(f"moe_combine: slot_y must be a contiguous fp16 [*, {a.N}]")
    a.moe_slot_y = _ptr(slot_y, dev, "linear", "slot_y")
    _launch("linear", x, C.byref(a))
    return out


def attention(q, k, v, out=None, scale=None, windows=None):
    """softmax(q k^T * scale) v.  q: [B, Lq, H, 64] views (any strides with unit inner stride), k/v: [B, Lk, H, 64].
    Returns/writes out: [B, Lq, H, 64] ("B L (H D)" when contiguous).
    windows: None, or one (row0, length, k0_count) per batch (self-attention, B <= 2): batch b computes only the query
    rows [row0, row0 + length), over all keys; rows of out outside a window are left as they were.  k0_count > 1 first
    overwrites the k0_count - 1 rows of k and v before row0 with row0's k and v (see r3g_attention in r3g.h)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _f16(t, n)
        if t.dim() != 4 or t.shape[-1] != 64 or t.stride(-1) != 1:
            raise ValueError(f"{n} must be [B, L, H, 64] with unit inner stride")
    B, Lq, H, _ = q.shape
    Lk = k.shape[1]
    out = _out("attention", out, (B, Lq, H, 64), torch.float16, q)
    dev = q.get_device()
    a = _abi.AttentionArgs()
    a.q, a.q_sb, a.q_sl, a.q_sh = _ptr(q, dev, "attention", "q"), q.stride(0), q.stride(1), q.stride(2)
    a.k, a.k_sb, a.k_sl, a.k_sh = _ptr(k, dev, "attention", "k"), k.stride(0), k.stride(1), k.stride(2)
    a.v, a.v_sb, a.v_sl, a.v_sh = _ptr(v, dev, "attention", "v"), v.stride(0), v.stride(1), v.stride(2)
    a.o, a.o_sb, a.o_sl, a.o_sh = _ptr(out, dev, "attention", "out"), out.stride(0), out.stride(1), out.stride(2)
    a.B, a.H, a.Lq, a.Lk = B, H, Lq, Lk
    a.scale = float(scale if scale is not None else 64 ** -0.5)
    if windows is not None:
        if len(windows) != B:
            raise ValueError(f"attention: {len(windows)} windows for {B} batches")
        for b, (r0, n, cnt) in enumerate(windows):
            a.win_row0[b], a.win_len[b], a.win_k0_count[b] = r0, n, cnt
    _launch("attention", q, C.byref(a))
    return out


def layernorm(x, weight=None, bias=None, eps=1e-6, scale=None, shift=None, rows_per_batch=0, out=None):
    """LayerNorm over the last dim (+ optional (1+scale)*y+shift modulation with per-batch [B, width] vectors).
    x / out may be segmented views (see _rows)."""
    _f16(x, "x")
    rows, width, ldx, xl, xst = _rows(x, "x")
    out = _out("layernorm", out, x.shape, torch.float16, x, rows=True)
    _, _, ldy, yl, yst = _rows(out, "out")
    seg_len, xs, ys = _merge_seg((xl, xst, rows), (yl, yst), "layernorm")
    mod_ld = scale.stride(0) if scale is not None else 0
    _launch("layernorm", x, x, ldx, out, ldy, rows, width, float(eps), weight, bias, scale, shift, mod_ld,
            int(rows_per_batch), seg_len, xs, ys)
    return out


def layernorm_f32in(x, weight, bias, eps=1e-5, out=None):
    """LayerNorm of a float32 [rows, width] stream into fp16 (VGGT blocks keep the residual stream in fp32)."""
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise TypeError("x must be contiguous float32")
    width = x.shape[-1]
    rows = x.numel() // width
    out = _out("layernorm_f32in", out, x.shape, torch.float16, x, rows=True)
    ldy = _rows(out, "out", segments=False)[2]
    _launch("layernorm_f32in", x, x, width, out, ldy, rows, width, float(eps), weight, bias)
    return out


def qk_norm_rope_(qkv, heads, eps, q_w, q_b, k_w, k_b, rope_freq, tokens_per_frame, n_special, patches_w):
    """In place on a packed fp16 [rows, 3*H*64] (3,H,D) projection: q/k LayerNorm (if weights) + 2-D RoPE (if freq>0)."""
    _f16(qkv, "qkv")
    if not qkv.is_contiguous():
        raise ValueError("qkv must be contiguous")
    ld = qkv.shape[-1]
    rows = qkv.numel() // ld
    _launch("qk_norm_rope", qkv, qkv, ld, rows, heads, float(eps), q_w, q_b, k_w, k_b, float(rope_freq),
            int(tokens_per_frame), int(n_special), int(patches_w))
    return qkv


def patchify(images, patch, mean=None, std=None, out_ld=None):
    """images float32 [N,3,H,W] -> fp16 [N*(H/p)*(W/p), out_ld] rows in Conv2d weight order (zero padded)."""
    if images.dtype != torch.float32 or images.dim() != 4 or images.shape[1] != 3:
        raise TypeError("images must be float32 [N,3,H,W]")
    images = images.contiguous()
    N, _, H, W = images.shape
    kk = 3 * patch * patch
    out_ld = out_ld or ((kk + 7) // 8) * 8
    out = torch.empty(N * (H // patch) * (W // patch), out_ld, device=images.device, dtype=torch.float16)
    m = (C.c_float * 3)(*(mean if mean is not None else (0.0, 0.0, 0.0)))
    sd = (C.c_float * 3)(*(std if std is not None else (1.0, 1.0, 1.0)))
    _launch("patchify", images, images, out, out_ld, N, H, W, int(patch), C.cast(m, C.c_void_p),
            C.cast(sd, C.c_void_p))
    return out


def qk_norm_(buf, heads, q_off, k_off, head_stride, mode, eps, q_w, q_b=None, k_w=None, k_b=None):
    """In-place per-head RMS (mode 0: QKNorm, rounded before the scale) / LayerNorm (mode 1) / nn.RMSNorm (mode 2: one
    rounding) of q (and k) inside a packed buffer of rows
    ([rows, ld] or a segmented [S, L, ld] view)."""
    _f16(buf, "buf")
    rows, _, ld, sl, sst = _rows(buf, "buf")
    _launch("qk_norm", buf, buf, ld, rows, heads, q_off, k_off, head_stride, mode, float(eps), q_w, q_b, k_w, k_b,
            sl, sst)
    return buf


def gemv(w, bias, vec, silu_in=False, silu_out=False, out=None, residual=None):
    """out[b] = W . act(vec[b]) + bias for B <= 8 rows; with residual ([B, N] fp16, it may be out itself)
    out[b] = fp16(that) + residual[b], rounded again."""
    _f16(w, "w"); _f16(vec, "vec")
    B, K = vec.shape
    N = w.shape[0]
    out = _out("gemv", out, (B, N), torch.float16, vec)
    if residual is not None and (residual.dtype != torch.float16 or residual.shape != out.shape
                                 or residual.stride() != out.stride()):
        raise ValueError(f"gemv: residual must be float16 {tuple(out.shape)} with out's strides {out.stride()}, got "
                         f"{residual.dtype} {tuple(residual.shape)} strides {residual.stride()}")
    _launch("gemv", vec, w, bias, vec, vec.stride(0), out, out.stride(0), residual, B, N, K, int(silu_in),
            int(silu_out))
    return out


def swiglu(x, F, out=None):
    """out[:, j] = silu(x[:, j]) * x[:, F + j]  (fp16 roundings of Dinov2SwiGLUFFN); x [M, 2F] -> out [M, F]."""
    _f16(x, "x")
    rows, width, ldx, _, _ = _rows(x, "x", segments=False)
    if width < 2 * F:
        raise ValueError("swiglu: x must hold 2F columns")
    out = _out("swiglu", out, (*x.shape[:-1], F), torch.float16, x, rows=True)
    ldo = _rows(out, "out", segments=False)[2]
    _launch("swiglu", x, x, ldx, out, ldo, rows, int(F))
    return out


def timestep_embedding(t, dim=256, time_factor=1000.0, max_period=10000.0, out=None):
    _f16(t, "t")
    out = _out("timestep_embedding", out, (t.shape[0], dim), torch.float16, t, contiguous=True)
    _launch("timestep_embedding", t, t, out, t.shape[0], dim, float(time_factor), float(max_period))
    return out


def cfg_euler_step_(x, v, guidance, dsigma, x_dup=None):
    """x <- x + dsigma * (v_uncond + g (v_cond - v_uncond)) with v = cat(cond, uncond) (v twice x's size), or
    x <- x + dsigma * v with guidance ignored when v is x's size (a model run without CFG).  x_dup, when given,
    receives x as many times as v holds samples: the next step's model input."""
    _f16(x, "x"); _f16(v, "v")
    n = x.numel()
    nb = v.numel() // n if n else 0
    if v.numel() != nb * n or nb not in (1, 2) or not (x.is_contiguous() and v.is_contiguous()):
        raise ValueError(f"cfg_euler_step_: v must be contiguous with {n} (no CFG) or 2 * {n} (cond, uncond) elements, "
                         f"got {tuple(v.shape)}")
    if x_dup is not None and (x_dup.dtype != torch.float16 or x_dup.numel() != nb * n or not x_dup.is_contiguous()):
        raise ValueError(f"cfg_euler_step_: x_dup must be contiguous float16 with {nb} * {n} elements, got {x_dup.dtype} "
                         f"{tuple(x_dup.shape)} with strides {x_dup.stride()}")
    _launch("cfg_euler_step", x, x, v, x_dup, n, nb, float(guidance), float(dsigma))
    return x


def grid_fourier(out, start, count, R, bounds6, num_freqs, include_pi):
    """Fourier features of the dense grid points [start, start+count) -> out, contiguous fp16 [count, >= 3+6F]: the
    kernel zero-pads every row to its full width."""
    _out("grid_fourier", out, (int(count), out.shape[-1]), torch.float16, out, contiguous=True)
    b = (C.c_float * 6)(*[float(v) for v in bounds6])
    _launch("grid_fourier", out, out, out.stride(0), int(start), int(count), int(R), C.cast(b, C.c_void_p),
            int(num_freqs), int(include_pi))
    return out


def points_fourier(queries, out, num_freqs, include_pi):
    """Fourier features of explicit fp16 query points [n, 3] -> out, contiguous [n, >= 3+6F] (zero padded)."""
    _f16(queries, "queries")
    q = queries.contiguous()
    _out("points_fourier", out, (q.shape[0], out.shape[-1]), torch.float16, q, contiguous=True)
    _launch("points_fourier", q, q, out, out.stride(0), q.shape[0], int(num_freqs), int(include_pi))
    return out


def points_fourier_f32(queries, out, num_freqs, include_pi):
    """Fourier features of explicit FLOAT32 query points [n, 3] (float32 arithmetic, fp16 result; FlashVDM levels)."""
    if queries.dtype != torch.float32:
        raise TypeError("queries must be float32")
    q = queries.contiguous()
    _out("points_fourier_f32", out, (q.shape[0], out.shape[-1]), torch.float16, q, contiguous=True)
    _launch("points_fourier_f32", q, q, out, out.stride(0), q.shape[0], int(num_freqs), int(include_pi))
    return out


def lnpost_dot(x, ln_w, ln_b, w_out, b_out, out, eps=1e-5):
    """ln_post + output_proj of the geo decoder: one float32 logit per row of x into out, contiguous [rows].
    x: fp16 rows with one row stride; ln_w, ln_b, w_out: fp16 [width]; b_out: fp16 [1] or None."""
    _f16(x, "x")
    rows, width, ldx, _, _ = _rows(x, "x", segments=False)
    for t, name in ((ln_w, "ln_w"), (ln_b, "ln_b"), (w_out, "w_out")):
        if _f16(t, name).numel() != width:
            raise ValueError(f"lnpost_dot: {name} must hold width = {width} values, got {t.numel()}")
    if b_out is not None:
        _f16(b_out, "b_out")
    _out("lnpost_dot", out, (rows,), torch.float32, x, contiguous=True)
    _launch("lnpost_dot", x, x, ldx, rows, width, float(eps), ln_w, ln_b, w_out, b_out, out)
    return out


def im2col3x3(x, stride=1, relu_in=False, out=None):
    """x fp16 NHWC [N,H,W,C] -> rows [N*Ho*Wo, 9*C] for a 3x3 / padding-1 convolution as a GEMM (see r3g.h)."""
    _f16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise ValueError("im2col3x3: x must be a contiguous NHWC tensor")
    N, H, W, Cc = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    out = _out("im2col3x3", out, (N * Ho * Wo, 9 * Cc), torch.float16, x, contiguous=True)
    _launch("im2col3x3", x, x, out, N, H, W, Cc, int(stride), int(relu_in))
    return out, Ho, Wo


def bilinear_nhwc(x, Ho, Wo, out=None):
    """F.interpolate(..., mode='bilinear', align_corners=True) on an fp16 NHWC tensor."""
    _f16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise ValueError("bilinear_nhwc: x must be a contiguous NHWC tensor")
    N, Hi, Wi, Cc = x.shape
    out = _out("bilinear_nhwc", out, (N, int(Ho), int(Wo), Cc), torch.float16, x, contiguous=True)
    _launch("bilinear_nhwc", x, x, out, N, Hi, Wi, int(Ho), int(Wo), Cc)
    return out


def _f32(t, name):
    if t is not None and (t.dtype != torch.float32 or t.stride(-1) != 1):
        raise TypeError(f"{name} must be float32 with unit inner stride")
    return t


def gemv_f32(w16, bias, vec, out=None, residual=None, gamma=None, silu_in=False, gelu_out=False):
    """out[b] = residual[b] + gamma * g(W . a(vec[b]) + bias): fp16 weights, float32 everything else (see r3g.h)."""
    _f16(w16, "w")
    for t, n in ((bias, "bias"), (vec, "vec"), (residual, "residual"), (gamma, "gamma")):
        _f32(t, n)
    B, K = vec.shape
    N = w16.shape[0]
    out = _out("gemv_f32", out, (B, N), torch.float32, vec)
    if residual is not None and residual.stride(0) != out.stride(0):
        raise ValueError("gemv_f32: residual must share out's row stride")
    _launch("gemv_f32", vec, w16, bias, vec, vec.stride(0), out, out.stride(0), residual, gamma, B, N, K, int(silu_in),
            int(gelu_out))
    return out


def layernorm_f32(x, weight=None, bias=None, eps=1e-5, shift=None, scale=None, gate=None, out=None):
    """float32 LayerNorm over the last dim of [rows, width]; with shift / scale / gate: gate * (LN(x)(1+scale)+shift) + x."""
    _f32(x, "x")
    rows, width = x.shape
    out = _out("layernorm_f32", out, x.shape, torch.float32, x)
    mod_ld = scale.stride(0) if scale is not None else 0
    _launch("layernorm_f32", x, x, x.stride(0), out, out.stride(0), rows, width, float(eps), _f32(weight, "weight"),
            _f32(bias, "bias"), _f32(shift, "shift"), _f32(scale, "scale"), _f32(gate, "gate"), mod_ld)
    return out


def small_attention_f32(qkv, B, S, H, D, out=None):
    """qkv float32 [B*S, 3*H*D] laid out (3, H, D) -> [B*S, H*D]; softmax over the S tokens of each batch element."""
    _f32(qkv, "qkv")
    if not qkv.is_contiguous() or qkv.shape != (B * S, 3 * H * D):
        raise ValueError("small_attention_f32: qkv must be contiguous [B*S, 3*H*D]")
    out = _out("small_attention_f32", out, (B * S, H * D), torch.float32, qkv, contiguous=True)
    _launch("small_attention_f32", qkv, qkv, out, B, S, H, D, float(D) ** -0.5)
    return out


def closed_form_inverse_se3(se3):
    """numpy branch of vggt/vggt/utils/geometry.py:120-169: [R t]^-1 = [R^T, -R^T t], written into np.eye(4)
    (so the result is float64 holding float32-computed entries)."""
    se3 = np.asarray(se3)
    R, T = se3[:, :3, :3], se3[:, :3, 3:]
    Rt = np.transpose(R, (0, 2, 1))
    inv = np.tile(np.eye(4), (len(R), 1, 1))
    inv[:, :3, :3] = Rt
    inv[:, :3, 3:] = -np.matmul(Rt, T)
    return inv


def unproject(depth, extrinsic, intrinsic, out_dtype=torch.float64, out=None):
    """depth: CUDA float32 [S,H,W]; extrinsic [S,3,4] / intrinsic [S,3,3]: host numpy float32 (cam from world).
    out: optional preallocated [S,H,W,3] tensor of `out_dtype` (a 1.6 GB float64 result is worth reusing)."""
    S, H, W = depth.shape
    c2w = np.ascontiguousarray(closed_form_inverse_se3(np.asarray(extrinsic))[:, :3, :].astype(np.float64))
    k = np.ascontiguousarray(np.asarray(intrinsic, dtype=np.float32).reshape(S, 9))
    out = _out("unproject", out, (S, H, W, 3), out_dtype, depth, contiguous=True)
    _launch("unproject", depth, depth.contiguous(), c2w.ctypes.data_as(C.c_void_p), k.ctypes.data_as(C.c_void_p), out,
            S, H, W, 1 if out_dtype == torch.float64 else 0)
    return out


class MarchingCubesError(RuntimeError):
    pass


_WS = {}


def _workspace(kind, device, nbytes):
    """One cached byte workspace per kind ("mc", "decimate") and device, grown when a call needs more and never shrunk:
    not re-requested from the allocator per object (marching cubes: 0.39 GB at 257^3, 3.0 GB at 513^3, sized for the
    worst case of every cell crossed).  The kinds stay apart: the marching-cubes one carries r3g_mc_count's state to
    r3g_mc_extract."""
    ws = _WS.get((kind, device))
    if ws is None or ws.numel() < nbytes:
        ws = _WS[kind, device] = torch.empty(max(nbytes, 1), device=device, dtype=torch.uint8)
    return ws


def marching_cubes(grid, level=0.0, bounds=None):
    """grid: CUDA float32 [n0,n1,n2].  Returns (verts float32 [V,3], faces int32 [F,3]) CUDA tensors in
    skimage's output convention.  Raises ValueError / RuntimeError like skimage.measure.marching_cubes."""
    return _extract_surface(grid, level, _abi.R3G_MC_LEWINER, bounds)


def dual_marching_cubes(grid):
    """r3g's dual marching cubes at level 0 (include/r3g.h, R3G_MC_DUAL): grid CUDA float32 [n0,n1,n2] of logits.
    Returns (verts float32 [V,3] in [0, 1]^3, array-axis order; faces int32 [F,3] with normals towards increasing
    values) CUDA tensors.  Raises RuntimeError when no cell is crossed."""
    return _extract_surface(grid, 0.0, _abi.R3G_MC_DUAL, None)


def _extract_surface(grid, level, method, bounds):
    if grid.dtype != torch.float32 or grid.dim() != 3:
        raise TypeError("grid must be float32 [n0,n1,n2]")
    grid = grid.contiguous()
    n0, n1, n2 = grid.shape
    ws_bytes = _abi.load_library().r3g_mc_workspace_bytes(n0, n1, n2)
    ws = _workspace("mc", grid.device, ws_bytes)
    nv, nf = C.c_int64(0), C.c_int64(0)
    try:
        _launch("mc_count", grid, grid, n0, n1, n2, float(level), method, ws, ws_bytes, C.byref(nv), C.byref(nf))
    except _abi.R3GError as e:
        if e.code == _abi.R3G_E_LEVEL:
            raise ValueError("Surface level must be within volume data range.") from None
        if e.code == _abi.R3G_E_NOSURFACE:
            raise RuntimeError("No surface found at the given iso value.") from None
        raise
    # capacities rounded up to 32 MiB so that the caching allocator can hand back the block of the previous object
    # (a fresh cudaMalloc of ~100 MB costs ~100 ms on this box; meshes of successive objects differ by a few percent)
    q = 32 << 20
    cap_v = (-(-(nv.value * 12) // q) * q) // 12 + 1
    cap_f = (-(-(nf.value * 12) // q) * q) // 12 + 1
    # the library gets the whole buffers: a dual mesh of a grid without interior edges has no face, and an empty slice
    # would pass a null address
    verts = torch.empty(cap_v, 3, device=grid.device, dtype=torch.float32)
    faces = torch.empty(cap_f, 3, device=grid.device, dtype=torch.int32)
    bptr = C.c_void_p(0)
    if bounds is not None:
        barr = (C.c_double * 6)(*[float(v) for v in bounds])
        bptr = C.cast(barr, C.c_void_p)
    _launch("mc_extract", grid, grid, n0, n1, n2, float(level), method, bptr, ws, ws_bytes, verts, faces)
    return verts[:nv.value], faces[:nf.value]


def mesh_components(faces, num_vertices):
    """labels int32 [num_vertices]: the smallest vertex index of each vertex's connected component (see r3g.h)."""
    if faces.dtype != torch.int32 or faces.dim() != 2 or faces.shape[1] != 3:
        raise TypeError("faces must be int32 [F, 3]")
    f = faces.contiguous()
    labels = torch.empty(int(num_vertices), device=faces.device, dtype=torch.int32)
    _launch("mesh_components", f, f, f.shape[0], int(num_vertices), labels)
    return labels


def mesh_decimate(verts, faces, target):
    """Quadric edge-collapse decimation to `target` faces (see include/r3g.h): verts CUDA float32 [V, 3], faces
    CUDA int32 [F, 3] on the same device.  Returns (verts float32 [V', 3], faces int32 [F', 3], rounds) on that device,
    F' in {target - 1, target} when the collapse rules allow it, else the smallest mesh they allow.  The workspace is
    cached per device like the marching-cubes one."""
    if verts.dtype != torch.float32 or verts.dim() != 2 or verts.shape[1] != 3:
        raise TypeError("verts must be float32 [V, 3]")
    if faces.dtype != torch.int32 or faces.dim() != 2 or faces.shape[1] != 3:
        raise TypeError("faces must be int32 [F, 3]")
    if int(target) < 0:
        raise ValueError(f"mesh_decimate: target must be >= 0, got {target}")
    v, f = verts.contiguous(), faces.contiguous()
    nv, nf = v.shape[0], f.shape[0]
    ws_bytes = _abi.load_library().r3g_decimate_workspace_bytes(nv, nf)
    if ws_bytes == 0 and nv and nf:
        raise ValueError(f"mesh_decimate: {nv} vertices / {nf} faces exceed the int32 index range")
    ws = _workspace("decimate", v.device, ws_bytes)
    v_out = torch.empty_like(v)
    f_out = torch.empty_like(f)
    nv_out, nf_out, rounds = C.c_int64(0), C.c_int64(0), C.c_int64(0)
    _launch("mesh_decimate", v, v, nv, f, nf, int(target), ws, ws_bytes, v_out, f_out, C.byref(nv_out), C.byref(nf_out),
            C.byref(rounds))
    return v_out[:nv_out.value], f_out[:nf_out.value], rounds.value


def mc_classify(grid, level=0.0):
    grid = grid.contiguous()
    n0, n1, n2 = grid.shape
    out = torch.empty((n0 - 1) * (n1 - 1) * (n2 - 1), device=grid.device, dtype=torch.uint8)
    _launch("mc_classify", grid, grid, n0, n1, n2, float(level), out)
    return out.view(n0 - 1, n1 - 1, n2 - 1)
