"""Torch-tensor front end of the C ABI (include/r3g.h).  Torch is plumbing only: it owns device memory
and the stream; every computation below happens in libr3g.so.  No fallback paths."""
import ctypes as C
import os
import time

import numpy as np
import torch

from . import _abi

ACT_NONE, ACT_GELU_TANH, ACT_GELU_ERF, ACT_RELU = 0, 1, 2, 3


def _ctx(t):
    """The r3g context of the tensor's device and torch's current stream OF THAT DEVICE, which the launch goes to.  The
    library switches to that device for the duration of each call (r3g_device_guard), so a pipeline on cuda:1 works
    without torch.cuda.set_device(1)."""
    if not t.is_cuda:
        raise RuntimeError("r3g ops need CUDA tensors: there is no CPU fallback")
    dev = t.device.index
    return _abi.get_context(dev), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _f16(t, name):
    if t.dtype != torch.float16:
        raise TypeError(f"{name} must be float16, got {t.dtype}")
    return t


def _rows(t, name):
    """Describe an activation as segmented rows.  Accepts [..., W] contiguous, a 2-D strided view [M, W], or a
    3-D view [S, L, W] whose segments are `stride(0)` apart (e.g. X[:, Lt:, :] of a joint txt+img buffer).
    Returns (data_ptr_tensor, rows, width, ld, seg_len, seg_stride_rows)."""
    if t.stride(-1) != 1:
        raise ValueError(f"{name}: innermost stride must be 1")
    w = t.shape[-1]
    if t.dim() == 1:
        return t, 1, w, w, 0, 0
    if t.is_contiguous():
        t2 = t.reshape(-1, w)
        return t2, t2.shape[0], w, w, 0, 0
    if t.dim() == 2:
        return t, t.shape[0], w, t.stride(0), 0, 0
    if t.dim() == 3:
        S, L, _ = t.shape
        ld = t.stride(1)
        if S == 1:
            return t, L, w, ld, 0, 0
        if t.stride(0) % ld:
            raise ValueError(f"{name}: segment stride must be a multiple of the row stride")
        return t, S * L, w, ld, L, t.stride(0) // ld
    raise ValueError(f"{name}: cannot describe as (segmented) rows without a copy")


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


def _linear_args(x, w, bias=None, *, out=None, act=ACT_NONE, act_cols=None, gate=None, gate_rows=0, residual=None,
                 ls_gamma=None, out_dtype=torch.float16, qk_norm=None):
    """Build one r3g_linear_args; returns (struct, out tensor, tensors the struct points into)."""
    _f16(x, "x"); _f16(w, "w")
    x2, M, K, ldx, xl, xst = _rows(x, "x")
    N = w.shape[0]
    if w.shape[1] != K or not w.is_contiguous():
        raise ValueError("w must be contiguous [N, K]")
    if out is None:
        out = torch.empty(*x.shape[:-1], N, device=x.device, dtype=out_dtype)
    o2, Mo, No, ldy, yl, yst = _rows(out, "out")
    if No != N or Mo != M:
        raise ValueError(f"out has shape {tuple(out.shape)}, expected {M} rows x {N}")
    seg_len, xs, ys = _merge_seg((xl, xst, M), (yl, yst), "linear")
    keep = [x2, w, bias, o2, gate, residual, ls_gamma]
    a = _abi.LinearArgs()
    a.x, a.ldx, a.w, a.bias = x2.data_ptr(), ldx, w.data_ptr(), (bias.data_ptr() if bias is not None else None)
    a.y, a.ldy = o2.data_ptr(), ldy
    a.M, a.N, a.K = M, N, K
    a.seg_len, a.x_seg_stride, a.y_seg_stride = seg_len, xs, ys
    a.act = act
    a.act_col0, a.act_col1 = act_cols if act_cols is not None else (0, N)
    if gate is not None:
        _f16(gate, "gate")
        a.gate, a.gate_ld, a.gate_rows = gate.data_ptr(), gate.stride(0), gate_rows
    if residual is not None:
        if residual.dtype == torch.float32:
            a.residual_f32 = 1
            if ls_gamma is not None:
                if ls_gamma.dtype != torch.float32 or ls_gamma.numel() != N:
                    raise TypeError("ls_gamma must be float32 [N]")
                a.ls_gamma = ls_gamma.data_ptr()
        else:
            _f16(residual, "residual")
        r2, _, _, ldr, rl, rst = _rows(residual, "residual")
        if ldr != ldy or (rl, rst) != (yl, yst):
            raise ValueError("residual must share out's geometry")
        a.residual = r2.data_ptr()
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
                setattr(a, "qkn_" + name, t.data_ptr())
                keep.append(t)
    return a, out, keep


def linear(x, w, bias=None, **kw):
    """Y = epilogue(X W^T + bias); see r3g_linear in include/r3g.h.

    x: [..., K] or a strided [M, K] / [S, L, K] view, w: [N, K] contiguous, out: same row structure, width N.
    gate: [B, N] view with unit inner stride, applied to logical rows b = r // gate_rows.
    residual must be the same view geometry as out (and may be out itself).
    qk_norm: dict(mode=QKN_RMS|QKN_LAYERNORM, q_col0, k_col0 (None: q only), cols, eps, q_w, q_b, k_w, k_b) -- the per-head
    q/k normalisation fused into the epilogue (see qkn_* in include/r3g.h).
    """
    ctx, stream = _ctx(x)
    a, out, _keep = _linear_args(x, w, bias, **kw)
    ctx.check(ctx.lib.r3g_linear(ctx.handle, C.byref(a), stream))
    return out


def linear_pair(first, second):
    """Two independent linears in ONE launch (r3g_linear_args.group_next): `first` / `second` are dicts of linear()'s
    arguments (x, w, bias, out, ...).  Results are those of linear(**first), linear(**second); the tiles of both problems
    share one persistent grid -- the img and txt streams of a DoubleStreamBlock fill the machine together."""
    ctx, stream = _ctx(first["x"])
    if second["x"].device != first["x"].device:
        raise ValueError("linear_pair: both problems must live on the same device")
    a, out_a, _ka = _linear_args(**first)
    b, out_b, _kb = _linear_args(**second)
    a.group_next = C.addressof(b)
    ctx.check(ctx.lib.r3g_linear(ctx.handle, C.byref(a), stream))
    return out_a, out_b


def attention(q, k, v, out=None, scale=None):
    """softmax(q k^T * scale) v.  q: [B, Lq, H, 64] views (any strides with unit inner stride), k/v: [B, Lk, H, 64].
    Returns/writes out: [B, Lq, H, 64] ("B L (H D)" when contiguous)."""
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _f16(t, n)
        if t.dim() != 4 or t.shape[-1] != 64 or t.stride(-1) != 1:
            raise ValueError(f"{n} must be [B, L, H, 64] with unit inner stride")
    ctx, stream = _ctx(q)
    B, Lq, H, _ = q.shape
    Lk = k.shape[1]
    if out is None:
        out = torch.empty(B, Lq, H, 64, device=q.device, dtype=torch.float16)
    a = _abi.AttentionArgs()
    a.q, a.q_sb, a.q_sl, a.q_sh = q.data_ptr(), q.stride(0), q.stride(1), q.stride(2)
    a.k, a.k_sb, a.k_sl, a.k_sh = k.data_ptr(), k.stride(0), k.stride(1), k.stride(2)
    a.v, a.v_sb, a.v_sl, a.v_sh = v.data_ptr(), v.stride(0), v.stride(1), v.stride(2)
    a.o, a.o_sb, a.o_sl, a.o_sh = out.data_ptr(), out.stride(0), out.stride(1), out.stride(2)
    a.B, a.H, a.Lq, a.Lk = B, H, Lq, Lk
    a.scale = float(scale if scale is not None else 64 ** -0.5)
    ctx.check(ctx.lib.r3g_attention(ctx.handle, C.byref(a), stream))
    return out


def layernorm(x, weight=None, bias=None, eps=1e-6, scale=None, shift=None, rows_per_batch=0, out=None):
    """LayerNorm over the last dim (+ optional (1+scale)*y+shift modulation with per-batch [B, width] vectors).
    x / out may be segmented views (see _rows)."""
    _f16(x, "x")
    ctx, stream = _ctx(x)
    x2, rows, width, ldx, xl, xst = _rows(x, "x")
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    o2, orow, _, ldy, yl, yst = _rows(out, "out")
    if orow != rows:
        raise ValueError("layernorm: out has a different number of rows")
    seg_len, xs, ys = _merge_seg((xl, xst, rows), (yl, yst), "layernorm")
    mod_ld = scale.stride(0) if scale is not None else 0
    ctx.check(ctx.lib.r3g_layernorm(ctx.handle, _p(x2), ldx, _p(o2), ldy, rows, width, float(eps), _p(weight),
                                    _p(bias), _p(scale), _p(shift), mod_ld, int(rows_per_batch), seg_len, xs, ys,
                                    stream))
    return out


def layernorm_f32in(x, weight, bias, eps=1e-5, out=None):
    """LayerNorm of a float32 [rows, width] stream into fp16 (VGGT blocks keep the residual stream in fp32)."""
    if x.dtype != torch.float32 or not x.is_contiguous():
        raise TypeError("x must be contiguous float32")
    ctx, stream = _ctx(x)
    width = x.shape[-1]
    rows = x.numel() // width
    if out is None:
        out = torch.empty(x.shape, device=x.device, dtype=torch.float16)
    ctx.check(ctx.lib.r3g_layernorm_f32in(ctx.handle, _p(x), width, _p(out), out.stride(-2) if out.dim() > 1 else width,
                                          rows, width, float(eps), _p(weight), _p(bias), stream))
    return out


def qk_norm_rope_(qkv, heads, eps, q_w, q_b, k_w, k_b, rope_freq, tokens_per_frame, n_special, patches_w):
    """In place on a packed fp16 [rows, 3*H*64] (3,H,D) projection: q/k LayerNorm (if weights) + 2-D RoPE (if freq>0)."""
    _f16(qkv, "qkv")
    ctx, stream = _ctx(qkv)
    if not qkv.is_contiguous():
        raise ValueError("qkv must be contiguous")
    ld = qkv.shape[-1]
    rows = qkv.numel() // ld
    ctx.check(ctx.lib.r3g_qk_norm_rope(ctx.handle, _p(qkv), ld, rows, heads, float(eps), _p(q_w), _p(q_b), _p(k_w),
                                       _p(k_b), float(rope_freq), int(tokens_per_frame), int(n_special),
                                       int(patches_w), stream))
    return qkv


def patchify(images, patch, mean=None, std=None, out_ld=None):
    """images float32 [N,3,H,W] -> fp16 [N*(H/p)*(W/p), out_ld] rows in Conv2d weight order (zero padded)."""
    if images.dtype != torch.float32 or images.dim() != 4 or images.shape[1] != 3:
        raise TypeError("images must be float32 [N,3,H,W]")
    images = images.contiguous()
    ctx, stream = _ctx(images)
    N, _, H, W = images.shape
    kk = 3 * patch * patch
    out_ld = out_ld or ((kk + 7) // 8) * 8
    out = torch.empty(N * (H // patch) * (W // patch), out_ld, device=images.device, dtype=torch.float16)
    m = (C.c_float * 3)(*(mean if mean is not None else (0.0, 0.0, 0.0)))
    sd = (C.c_float * 3)(*(std if std is not None else (1.0, 1.0, 1.0)))
    ctx.check(ctx.lib.r3g_patchify(ctx.handle, _p(images), _p(out), out_ld, N, H, W, int(patch), C.cast(m, C.c_void_p),
                                   C.cast(sd, C.c_void_p), stream))
    return out


def qk_norm_(buf, heads, q_off, k_off, head_stride, mode, eps, q_w, q_b=None, k_w=None, k_b=None):
    """In-place per-head RMS (mode 0) / LayerNorm (mode 1) of q (and k) inside a packed buffer of rows
    ([rows, ld] or a segmented [S, L, ld] view)."""
    _f16(buf, "buf")
    ctx, stream = _ctx(buf)
    b2, rows, _, ld, sl, sst = _rows(buf, "buf")
    ctx.check(ctx.lib.r3g_qk_norm(ctx.handle, _p(b2), ld, rows, heads, q_off, k_off, head_stride, mode, float(eps),
                                  _p(q_w), _p(q_b), _p(k_w), _p(k_b), sl, sst, stream))
    return buf


def gemv(w, bias, vec, silu_in=False, silu_out=False, out=None):
    """out[b] = W . act(vec[b]) + bias for B <= 8 rows."""
    _f16(w, "w"); _f16(vec, "vec")
    ctx, stream = _ctx(vec)
    B, K = vec.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty(B, N, device=vec.device, dtype=torch.float16)
    ctx.check(ctx.lib.r3g_gemv(ctx.handle, _p(w), _p(bias), _p(vec), vec.stride(0), _p(out), out.stride(0), B, N, K,
                               int(silu_in), int(silu_out), stream))
    return out


def swiglu(x, F, out=None):
    """out[:, j] = silu(x[:, j]) * x[:, F + j]  (fp16 roundings of Dinov2SwiGLUFFN); x [M, 2F] -> out [M, F]."""
    _f16(x, "x")
    ctx, stream = _ctx(x)
    x2, rows, width, ldx, _, _ = _rows(x, "x")
    if width < 2 * F:
        raise ValueError("swiglu: x must hold 2F columns")
    if out is None:
        out = torch.empty(*x.shape[:-1], F, device=x.device, dtype=torch.float16)
    o2, orow, _, ldo, _, _ = _rows(out, "out")
    ctx.check(ctx.lib.r3g_swiglu(ctx.handle, _p(x2), ldx, _p(o2), ldo, rows, int(F), stream))
    return out


def timestep_embedding(t, dim=256, time_factor=1000.0, max_period=10000.0, out=None):
    _f16(t, "t")
    ctx, stream = _ctx(t)
    if out is None:
        out = torch.empty(t.shape[0], dim, device=t.device, dtype=torch.float16)
    ctx.check(ctx.lib.r3g_timestep_embedding(ctx.handle, _p(t), _p(out), t.shape[0], dim, float(time_factor),
                                             float(max_period), stream))
    return out


def cfg_euler_step_(x, v, guidance, dsigma, x_dup=None):
    """x <- x + dsigma * (v_uncond + g (v_cond - v_uncond)); v = cat(cond, uncond)."""
    _f16(x, "x"); _f16(v, "v")
    ctx, stream = _ctx(x)
    n = x.numel()
    if v.numel() != 2 * n or not (x.is_contiguous() and v.is_contiguous()):
        raise ValueError("v must hold cond and uncond predictions, contiguous")
    ctx.check(ctx.lib.r3g_cfg_euler_step(ctx.handle, _p(x), _p(v), _p(x_dup), n, float(guidance), float(dsigma),
                                         stream))
    return x


def grid_fourier(out, start, count, R, bounds6, num_freqs, include_pi):
    ctx, stream = _ctx(out)
    b = (C.c_float * 6)(*[float(v) for v in bounds6])
    ctx.check(ctx.lib.r3g_grid_fourier(ctx.handle, _p(out), out.stride(0), int(start), int(count), int(R),
                                       C.cast(b, C.c_void_p), int(num_freqs), int(include_pi), stream))
    return out


def points_fourier(queries, out, num_freqs, include_pi):
    """Fourier features of explicit fp16 query points [n, 3] -> out [n, >= 3+6F] (zero padded)."""
    _f16(queries, "queries")
    ctx, stream = _ctx(queries)
    q = queries.contiguous()
    ctx.check(ctx.lib.r3g_points_fourier(ctx.handle, _p(q), _p(out), out.stride(0), q.shape[0], int(num_freqs),
                                         int(include_pi), stream))
    return out


def points_fourier_f32(queries, out, num_freqs, include_pi):
    """Fourier features of explicit FLOAT32 query points [n, 3] (float32 arithmetic, fp16 result; FlashVDM levels)."""
    if queries.dtype != torch.float32:
        raise TypeError("queries must be float32")
    ctx, stream = _ctx(queries)
    q = queries.contiguous()
    ctx.check(ctx.lib.r3g_points_fourier_f32(ctx.handle, _p(q), _p(out), out.stride(0), q.shape[0], int(num_freqs),
                                             int(include_pi), stream))
    return out


def lnpost_dot(x, ln_w, ln_b, w_out, b_out, out, eps=1e-5):
    ctx, stream = _ctx(x)
    x2, rows, width, ldx, _, _ = _rows(x, "x")
    ctx.check(ctx.lib.r3g_lnpost_dot(ctx.handle, _p(x2), ldx, rows, width, float(eps), _p(ln_w), _p(ln_b), _p(w_out),
                                     _p(b_out), _p(out), stream))
    return out


def im2col3x3(x, stride=1, relu_in=False, out=None):
    """x fp16 NHWC [N,H,W,C] -> rows [N*Ho*Wo, 9*C] for a 3x3 / padding-1 convolution as a GEMM (see r3g.h)."""
    _f16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise ValueError("im2col3x3: x must be a contiguous NHWC tensor")
    ctx, stream = _ctx(x)
    N, H, W, Cc = x.shape
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    if out is None:
        out = torch.empty(N * Ho * Wo, 9 * Cc, device=x.device, dtype=torch.float16)
    ctx.check(ctx.lib.r3g_im2col3x3(ctx.handle, _p(x), _p(out), N, H, W, Cc, int(stride), int(relu_in), stream))
    return out, Ho, Wo


def bilinear_nhwc(x, Ho, Wo, out=None):
    """F.interpolate(..., mode='bilinear', align_corners=True) on an fp16 NHWC tensor."""
    _f16(x, "x")
    if x.dim() != 4 or not x.is_contiguous():
        raise ValueError("bilinear_nhwc: x must be a contiguous NHWC tensor")
    ctx, stream = _ctx(x)
    N, Hi, Wi, Cc = x.shape
    if out is None:
        out = torch.empty(N, Ho, Wo, Cc, device=x.device, dtype=torch.float16)
    ctx.check(ctx.lib.r3g_bilinear_nhwc(ctx.handle, _p(x), _p(out), N, Hi, Wi, int(Ho), int(Wo), Cc, stream))
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
    ctx, stream = _ctx(vec)
    B, K = vec.shape
    N = w16.shape[0]
    if out is None:
        out = torch.empty(B, N, device=vec.device, dtype=torch.float32)
    if residual is not None and residual.stride(0) != out.stride(0):
        raise ValueError("gemv_f32: residual must share out's row stride")
    ctx.check(ctx.lib.r3g_gemv_f32(ctx.handle, _p(w16), _p(bias), _p(vec), vec.stride(0), _p(out), out.stride(0),
                                   _p(residual), _p(gamma), B, N, K, int(silu_in), int(gelu_out), stream))
    return out


def layernorm_f32(x, weight=None, bias=None, eps=1e-5, shift=None, scale=None, gate=None, out=None):
    """float32 LayerNorm over the last dim of [rows, width]; with shift / scale / gate: gate * (LN(x)(1+scale)+shift) + x."""
    _f32(x, "x")
    ctx, stream = _ctx(x)
    rows, width = x.shape
    if out is None:
        out = torch.empty_like(x)
    mod_ld = scale.stride(0) if scale is not None else 0
    ctx.check(ctx.lib.r3g_layernorm_f32(ctx.handle, _p(x), x.stride(0), _p(out), out.stride(0), rows, width, float(eps),
                                        _p(_f32(weight, "weight")), _p(_f32(bias, "bias")), _p(_f32(shift, "shift")),
                                        _p(_f32(scale, "scale")), _p(_f32(gate, "gate")), mod_ld, stream))
    return out


def small_attention_f32(qkv, B, S, H, D, out=None):
    """qkv float32 [B*S, 3*H*D] laid out (3, H, D) -> [B*S, H*D]; softmax over the S tokens of each batch element."""
    _f32(qkv, "qkv")
    ctx, stream = _ctx(qkv)
    if not qkv.is_contiguous() or qkv.shape != (B * S, 3 * H * D):
        raise ValueError("small_attention_f32: qkv must be contiguous [B*S, 3*H*D]")
    if out is None:
        out = torch.empty(B * S, H * D, device=qkv.device, dtype=torch.float32)
    ctx.check(ctx.lib.r3g_small_attention_f32(ctx.handle, _p(qkv), _p(out), B, S, H, D, float(D) ** -0.5, stream))
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
    ctx, stream = _ctx(depth)
    S, H, W = depth.shape
    c2w = np.ascontiguousarray(closed_form_inverse_se3(np.asarray(extrinsic))[:, :3, :].astype(np.float64))
    k = np.ascontiguousarray(np.asarray(intrinsic, dtype=np.float32).reshape(S, 9))
    if out is None:
        out = torch.empty(S, H, W, 3, device=depth.device, dtype=out_dtype)
    elif out.shape != (S, H, W, 3) or out.dtype != out_dtype or not out.is_contiguous():
        raise ValueError("unproject: out must be a contiguous [S,H,W,3] tensor of out_dtype")
    ctx.check(ctx.lib.r3g_unproject(ctx.handle, _p(depth.contiguous()), c2w.ctypes.data_as(C.c_void_p),
                                    k.ctypes.data_as(C.c_void_p), _p(out), S, H, W,
                                    1 if out_dtype == torch.float64 else 0, stream))
    return out


class MarchingCubesError(RuntimeError):
    pass


_MC_WS = {}


def _mc_workspace(device, nbytes):
    """One cached marching-cubes workspace per device (0.39 GB at 257^3, 3.0 GB at 513^3; sized for the worst case of every
    cell crossed): not re-requested from the allocator per object."""
    ws = _MC_WS.get(device)
    if ws is None or ws.numel() < nbytes:
        ws = torch.empty(nbytes, device=device, dtype=torch.uint8)
        _MC_WS[device] = ws
    return ws


def marching_cubes(grid, level=0.0, bounds=None):
    """grid: CUDA float32 [n0,n1,n2].  Returns (verts float32 [V,3], faces int32 [F,3]) CUDA tensors in
    skimage's output convention.  Raises ValueError / RuntimeError like skimage.measure.marching_cubes."""
    if grid.dtype != torch.float32 or grid.dim() != 3:
        raise TypeError("grid must be float32 [n0,n1,n2]")
    grid = grid.contiguous()
    ctx, stream = _ctx(grid)
    n0, n1, n2 = grid.shape
    ws_bytes = ctx.lib.r3g_mc_workspace_bytes(n0, n1, n2)
    dbg = os.environ.get("R3G_DEBUG_TIMING") == "1"
    if dbg:
        torch.cuda.synchronize()
        t0 = time.perf_counter()
    ws = _mc_workspace(grid.device, ws_bytes)
    if dbg:
        t1 = time.perf_counter()
    nv, nf = C.c_int64(0), C.c_int64(0)
    rc = ctx.lib.r3g_mc_count(ctx.handle, _p(grid), n0, n1, n2, float(level), _p(ws), ws_bytes, C.byref(nv),
                              C.byref(nf), stream)
    if rc == _abi.R3G_E_LEVEL:
        raise ValueError("Surface level must be within volume data range.")
    if rc == _abi.R3G_E_NOSURFACE:
        raise RuntimeError("No surface found at the given iso value.")
    ctx.check(rc)
    if dbg:
        t2 = time.perf_counter()
    # capacities rounded up to 32 MiB so that the caching allocator can hand back the block of the previous object
    # (a fresh cudaMalloc of ~100 MB costs ~100 ms on this box; meshes of successive objects differ by a few percent)
    q = 32 << 20
    cap_v = (-(-(nv.value * 12) // q) * q) // 12 + 1
    cap_f = (-(-(nf.value * 12) // q) * q) // 12 + 1
    verts = torch.empty(cap_v, 3, device=grid.device, dtype=torch.float32)[:nv.value]
    faces = torch.empty(cap_f, 3, device=grid.device, dtype=torch.int32)[:nf.value]
    if dbg:
        t3 = time.perf_counter()
    bptr = C.c_void_p(0)
    if bounds is not None:
        barr = (C.c_double * 6)(*[float(v) for v in bounds])
        bptr = C.cast(barr, C.c_void_p)
    ctx.check(ctx.lib.r3g_mc_extract(ctx.handle, _p(grid), n0, n1, n2, float(level), bptr, _p(ws), ws_bytes,
                                     _p(verts), _p(faces), stream))
    if dbg:
        torch.cuda.synchronize()
        t4 = time.perf_counter()
        print(f"[r3g mc] ws {1e3 * (t1 - t0):.2f} ms, count {1e3 * (t2 - t1):.2f} ms, alloc {1e3 * (t3 - t2):.2f} ms, "
              f"extract {1e3 * (t4 - t3):.2f} ms, V={nv.value} F={nf.value}", flush=True)
    return verts, faces


def mesh_components(faces, num_vertices):
    """labels int32 [num_vertices]: the smallest vertex index of each vertex's connected component (see r3g.h)."""
    if faces.dtype != torch.int32 or faces.dim() != 2 or faces.shape[1] != 3:
        raise TypeError("faces must be int32 [F, 3]")
    ctx, stream = _ctx(faces)
    f = faces.contiguous()
    labels = torch.empty(int(num_vertices), device=faces.device, dtype=torch.int32)
    ctx.check(ctx.lib.r3g_mesh_components(ctx.handle, _p(f), f.shape[0], int(num_vertices), _p(labels), stream))
    return labels


def mc_classify(grid, level=0.0):
    grid = grid.contiguous()
    ctx, stream = _ctx(grid)
    n0, n1, n2 = grid.shape
    out = torch.empty((n0 - 1) * (n1 - 1) * (n2 - 1), device=grid.device, dtype=torch.uint8)
    ctx.check(ctx.lib.r3g_mc_classify(ctx.handle, _p(grid), n0, n1, n2, float(level), _p(out), stream))
    return out.view(n0 - 1, n1 - 1, n2 - 1)
