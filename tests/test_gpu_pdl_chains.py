"""GPU: programmatic dependent launch (PDL).  Every kernel launched through r3g_launch_pdl may start while the kernel
before it in the stream is still running, and must call pdl_wait() before it touches memory another kernel produces or
still reads.  The kernel tests elsewhere feed each r3g kernel from torch kernels, which never trigger early, so a
misplaced wait would pass them.  Here:

1. Chains: a producer r3g launch followed directly on the same stream by a consumer r3g launch, run three ways that
   must agree bit for bit -- serialized (a synchronize between the two: the reference), back to back (PDL overlap
   possible) and captured into a CUDA graph and replayed (a programmatic edge inside the graph).  Before every run the
   producer's output is NaN and the consumer's out= buffer another non-finite pattern, so a consumer that reads its
   input before the producer wrote it, or writes a buffer the producer still reads, changes the result.  CHAINS covers
   every instantiation of every PDL kernel (CONSUMERS, kept equal to the launches in csrc/ by tests/test_pdl_launches.py)
   as a consumer, every early-triggering kernel as a producer, each activation operand read after the wait and each
   consumer writing over the producer's input; the pairs the models launch are listed with their source lines.
2. Whole forwards (DiT + one CFG step, VAE + SDF grid, FlashVDM, DINOv2 conditioner, VGGT aggregator, camera and DPT
   heads) run eager and graph-replayed with PDL on here and with R3G_PDL=0 in a subprocess: equal bits.  None of the
   kernels uses atomics, so equal bits are the requirement.

Run as a script (`python tests/test_gpu_pdl_chains.py --forwards OUT.pt`) it writes the forwards' outputs to OUT.pt."""
import collections
import contextlib
import os
import subprocess
import sys

if __name__ == "__main__":
    _ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for _p in (_ROOT, os.path.join(_ROOT, "3d-re-gen_b200"), os.path.join(_ROOT, "oracle")):
        if _p not in sys.path:
            sys.path.insert(0, _p)

import numpy as np
import pytest
import torch

DEV = "cuda"
F16, F32 = torch.float16, torch.float32
NAN, NEG_INF = float("nan"), float("-inf")

# Every kernel (with each template instantiation) that csrc/ launches through r3g_launch_pdl.
CONSUMERS = (
    "linear_kernel<128>", "linear_kernel<256>",
    "kv_fill_kernel", "attention_kernel",
    "layernorm_kernel<4>", "layernorm_kernel<8>",
    "lnpost_dot_kernel<4>", "lnpost_dot_kernel<8>",
    "gemv_kernel<1>", "gemv_kernel<2>", "gemv_kernel<4>", "gemv_kernel<8>",
    "swiglu_kernel",
    "gemv_f32_kernel<1>", "gemv_f32_kernel<2>", "gemv_f32_kernel<4>", "gemv_f32_kernel<8>",
    "layernorm_f32_kernel",
    "small_attention_f32_kernel<1>", "small_attention_f32_kernel<2>", "small_attention_f32_kernel<4>",
    "small_attention_f32_kernel<8>",
    "im2col3x3_kernel",
    "bilinear_nhwc_kernel",
)
# The r3g entry point each kernel is launched by, and the activation operands it reads after its wait.
ENTRY = {"linear_kernel": "linear", "kv_fill_kernel": "attention", "attention_kernel": "attention",
         "layernorm_kernel": "layernorm", "lnpost_dot_kernel": "lnpost_dot", "gemv_kernel": "gemv",
         "swiglu_kernel": "swiglu", "gemv_f32_kernel": "gemv_f32", "layernorm_f32_kernel": "layernorm_f32",
         "small_attention_f32_kernel": "small_attention_f32", "im2col3x3_kernel": "im2col3x3",
         "bilinear_nhwc_kernel": "bilinear_nhwc"}
ACTIVATION_OPERANDS = {
    "linear": {"x", "gate", "residual"}, "attention": {"q", "k", "v"}, "layernorm": {"x", "scale", "shift"},
    "lnpost_dot": {"x"}, "gemv": {"vec", "residual"}, "swiglu": {"x"}, "gemv_f32": {"vec", "residual"},
    "layernorm_f32": {"x", "shift", "scale", "gate"}, "small_attention_f32": {"qkv"}, "im2col3x3": {"x"},
    "bilinear_nhwc": {"x"}}
# The kernels that call pdl_trigger() right after their wait, so that the next kernel's CTAs start under their tail
# (by entry point; kv_fill runs inside r3g_attention).  linear_kernel and attention_kernel trigger at exit only.
EARLY_TRIGGERING = ("kv_fill", "im2col3x3", "bilinear_nhwc", "gemv_f32", "layernorm_f32", "small_attention_f32",
                    "layernorm", "gemv", "swiglu", "lnpost_dot")


def _ops():
    from r3g import ops
    return ops


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------------------ chains
class Chain:
    """The buffers of one chain, what each holds before a run (a tensor to copy in, or a fill value), and the two
    launches.  check(before, after) checks the consumer's result against a float64 mirror, given every buffer just
    before the consumer ran and just after; `finite` lists views that must end finite (the producer's output the
    consumer reads and the consumer's output), so that a chain cannot pass by comparing NaN with NaN."""

    def __init__(self, seed):
        self.t, self.init, self.seed = {}, {}, seed * 1000
        self.producer = self.consumer = self.check = None
        self.finite = []

    def randn(self, *shape, std=1.0, mean=0.0, dtype=F16):
        self.seed += 1
        g = torch.Generator(device=DEV).manual_seed(self.seed)
        return (mean + std * torch.randn(*shape, generator=g, device=DEV)).to(dtype)

    def inp(self, name, *shape, std=1.0, dtype=F16):
        """A buffer restored to the same random contents before every run."""
        v = self.randn(*shape, std=std, dtype=dtype)
        self.t[name], self.init[name] = v.clone(), v
        return self.t[name]

    def buf(self, name, *shape, value=NAN, dtype=F16):
        """A buffer filled with `value` before every run."""
        self.t[name], self.init[name] = torch.empty(*shape, device=DEV, dtype=dtype), value
        return self.t[name]

    def reset(self):
        for k, v in self.init.items():
            if isinstance(v, torch.Tensor):
                self.t[k].copy_(v)
            else:
                self.t[k].fill_(v)

    def snap(self):
        return {k: v.clone() for k, v in self.t.items()}


Spec = collections.namedtuple("Spec", "name producer entry consumers reads war source side_stream build")
CHAINS = []


def chain(producer, entry, consumers, reads=(), war=False, source=None, side_stream=False):
    """Registers a chain builder.  producer / entry: the r3g entry points of the two launches; consumers: the kernels
    the second launch runs; reads: the consumer's activation operands that the producer wrote; war: the consumer writes
    a buffer the producer reads; source: where a model launches this pair."""
    def deco(fn):
        CHAINS.append(Spec(fn.__name__, producer, entry, tuple(consumers), tuple(reads), war, source, side_stream, fn))
        return fn
    return deco


def _gemm_tile_n(problems):
    from test_gpu_kernel_bounds import gemm_tile_n
    return gemm_tile_n(problems, _sms())


def _check_linear(got, x, w, b=None, what="", **kw):
    import fp16_ref as R
    R.check_bound(got, *R.linear(x, w, b, **kw), what)


def _check_attention(o, q, k, v, what, rows=None):
    """o, q: [B, Lq, H, 64], k, v: [B, Lk, H, 64]; rows: per batch, the query rows computed (default all)."""
    import fp16_ref as R
    for bi in range(q.shape[0]):
        r0, r1 = rows[bi] if rows else (0, q.shape[1])
        for h in range(q.shape[2]):
            R.check_bound(o[bi, r0:r1, h], *R.attention(q[bi, r0:r1, h], k[bi, :, h], v[bi, :, h]), f"{what} b={bi} h={h}")


# --- linear
@chain("layernorm", "linear", ["linear_kernel<128>"], reads=("x", "residual"))
def chain_layernorm_to_linear128_residual():
    ops, c = _ops(), Chain(1)
    M, W = 65536, 128
    x, Y, O = c.inp("x", M, W), c.buf("y", M, W), c.buf("o", M, W, value=NEG_INF)
    lw, lb = c.randn(W, mean=1.0, std=0.1), c.randn(W, std=0.1)
    w, b = c.randn(W, W, std=W ** -0.5), c.randn(W)
    assert _gemm_tile_n([(M, W, 0)]) == 128
    c.producer = lambda: ops.layernorm(x, lw, lb, eps=1e-6, out=Y)
    c.consumer = lambda: ops.linear(Y, w, b, residual=Y, out=O)
    c.check = lambda bf, af: _check_linear(af["o"], bf["y"], w, b, "linear<128> residual", residual=bf["y"])
    c.finite = [Y, O]
    return c


@chain("swiglu", "linear", ["linear_kernel<256>"], reads=("x",), source="conditioner.py:121-122 (MLP gate -> out "
       "projection with LayerScale gate and residual in place)")
def chain_swiglu_to_linear256_gated_residual():
    ops, c = _ops(), Chain(2)
    M, F, N = 4864, 1024, 1024
    hid, G, X = c.inp("hid", M, 2 * F), c.buf("g", M, F), c.inp("X", M, N)
    w, b, ls = c.randn(N, F, std=F ** -0.5), c.randn(N), c.randn(1, N, mean=0.5, std=0.1)
    assert _gemm_tile_n([(M, N, 0)]) == 256
    c.producer = lambda: ops.swiglu(hid, F, out=G)
    c.consumer = lambda: ops.linear(G, w, b, gate=ls, gate_rows=M, residual=X, out=X)
    c.check = lambda bf, af: _check_linear(af["X"], bf["g"], w, b, "linear<256> gated residual", gate=ls, gate_rows=M,
                                           residual=bf["X"])
    c.finite = [G, X]
    return c


@chain("gemv", "linear", ["linear_kernel<128>"], reads=("gate",), source="dit.py:224,269-271 (the modulation GEMV "
       "gives the gate of the gated residual projection)")
def chain_gemv_to_linear_gate():
    ops, c = _ops(), Chain(3)
    B, L, H, K = 2, 1000, 128, 4096
    vec, mods = c.inp("vec", B, K), c.buf("mods", B, 3 * H)
    x, X = c.inp("x", B, L, H), c.inp("X", B, L, H)
    wm, bm = c.randn(3 * H, K, std=K ** -0.5), c.randn(3 * H)
    w, b = c.randn(H, H, std=H ** -0.5), c.randn(H)
    gate = mods[:, H:2 * H]
    c.producer = lambda: ops.gemv(wm, bm, vec, silu_in=True, out=mods)
    c.consumer = lambda: ops.linear(x, w, b, gate=gate, gate_rows=L, residual=X, out=X)
    c.check = lambda bf, af: _check_linear(af["X"].view(-1, H), bf["x"].view(-1, H), w, b, "linear gate from gemv",
                                           gate=bf["mods"][:, H:2 * H], gate_rows=L, residual=bf["X"].view(-1, H))
    c.finite = [mods, X]
    return c


@chain("layernorm_f32", "linear", ["linear_kernel<128>"], reads=("residual",), side_stream=True,
       source="vggt.py:66 form (LayerScale residual on the float32 stream)")
def chain_layernorm_f32_to_linear_f32_residual():
    ops, c = _ops(), Chain(4)
    M, N, K = 4096, 128, 256
    r, Y = c.inp("r", M, N, dtype=F32), c.buf("y", M, N, dtype=F32)
    x = c.inp("x", M, K)
    w, b, ls = c.randn(N, K, std=K ** -0.5), c.randn(N), c.randn(N, mean=0.5, std=0.1, dtype=F32)
    c.producer = lambda: ops.layernorm_f32(r, eps=1e-5, out=Y)
    c.consumer = lambda: ops.linear(x, w, b, residual=Y, ls_gamma=ls, out=Y)
    c.check = lambda bf, af: _check_linear(af["y"], bf["x"], w, b, "linear fp32 residual + LayerScale",
                                           residual=bf["y"], ls_gamma=ls)
    c.finite = [Y]
    return c


@chain("layernorm", "linear", ["linear_kernel<128>"], reads=("x",), war=True,
       source="dit.py:253-262 (modulated LayerNorm of the txt stream -> the streams' grouped projection)")
def chain_layernorm_to_linear_group_over_its_input():
    ops, c = _ops(), Chain(5)
    B, Lt, Li, W = 2, 137, 307, 256
    L = Lt + Li
    A, XM = c.inp("A", B, L, W), c.buf("xm", B, L, W)
    sc, sh = c.inp("sc", B, W, std=0.2), c.inp("sh", B, W, std=0.2)
    wi, bi, wt, bt = c.randn(W, W, std=W ** -0.5), c.randn(W), c.randn(W, W, std=W ** -0.5), c.randn(W)
    c.producer = lambda: ops.layernorm(A, eps=1e-6, scale=sc, shift=sh, rows_per_batch=L, out=XM)
    # both streams read the normalised rows and overwrite the rows the LayerNorm reads (segmented, one launch)
    c.consumer = lambda: ops.linear_group(dict(x=XM[:, Lt:], w=wi, bias=bi, out=A[:, Lt:], act=ops.ACT_GELU_TANH),
                                          dict(x=XM[:, :Lt], w=wt, bias=bt, out=A[:, :Lt]))

    def check(bf, af):
        _check_linear(af["A"][:, Lt:].reshape(-1, W), bf["xm"][:, Lt:].reshape(-1, W), wi, bi, "group img", act=1)
        _check_linear(af["A"][:, :Lt].reshape(-1, W), bf["xm"][:, :Lt].reshape(-1, W), wt, bt, "group txt")
    c.check = check
    c.finite = [XM, A]
    return c


@chain("layernorm", "linear", ["linear_kernel<128>"], reads=("x",),
       source="dit.py:253-262 with the q/k RMS norm fused into the projection's epilogue")
def chain_dit_layernorm_to_qkv_pair():
    ops, c = _ops(), Chain(6)
    B, Lt, Li, H = 2, 137, 307, 128
    L = Lt + Li
    X, XM, QKV = c.inp("X", B, L, H), c.buf("xm", B, L, H), c.buf("qkv", B, L, 3 * H, value=NEG_INF)
    sc, sh = c.inp("sc", B, H, std=0.2), c.inp("sh", B, H, std=0.2)
    p = {s: (c.randn(3 * H, H, std=H ** -0.5), c.randn(3 * H), c.randn(64, mean=1.0, std=0.1),
             c.randn(64, mean=1.0, std=0.1)) for s in "it"}

    def qkv(s, o, n):
        w, b, qs, ks = p[s]
        return dict(x=XM[:, o:o + n], w=w, bias=b, out=QKV[:, o:o + n],
                    qk_norm=dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H, cols=H, eps=1e-6, q_w=qs, k_w=ks))
    c.producer = lambda: ops.layernorm(X[:, :Lt], eps=1e-6, scale=sc, shift=sh, rows_per_batch=Lt, out=XM[:, :Lt])
    c.init["xm"] = torch.zeros(B, L, H, device=DEV, dtype=F16)      # the img rows come from an earlier launch
    c.consumer = lambda: ops.linear_pair(qkv("i", Lt, Li), qkv("t", 0, Lt))
    c.finite = [XM, QKV]
    return c


# --- attention
@chain("layernorm", "attention", ["kv_fill_kernel", "attention_kernel"], reads=("q", "k", "v"),
       source="dit.py:268 (the collapsed unconditional sample: windows with a counted first key)")
def chain_layernorm_to_windowed_attention():
    ops, c = _ops(), Chain(7)
    B, Lt, Li, H = 2, 137, 307, 2
    L = Lt + Li
    src, QKV, O = c.inp("src", B * L, 3 * H * 64), c.buf("qkv", B, L, 3, H, 64), c.buf("o", B, L, H, 64, value=NEG_INF)
    wins = ((0, L, 1), (Lt - 1, Li + 1, Lt))
    c.producer = lambda: ops.layernorm(src, eps=1e-6, out=QKV.view(B * L, -1))
    c.consumer = lambda: ops.attention(QKV[:, :, 0], QKV[:, :, 1], QKV[:, :, 2], out=O, windows=wins)

    def check(bf, af):
        q = bf["qkv"]
        k, v = q[:, :, 1].clone(), q[:, :, 2].clone()
        k[1, :Lt - 1], v[1, :Lt - 1] = k[1, Lt - 1], v[1, Lt - 1]         # kv_fill's copies of the window's first key
        assert torch.equal(af["qkv"][:, :, 1], k) and torch.equal(af["qkv"][:, :, 2], v)
        _check_attention(af["o"], q[:, :, 0], k, v, "windowed attention", rows=[(0, L), (Lt - 1, L)])
    c.check = check
    c.finite = [QKV, O[0], O[1, Lt - 1:]]
    return c


@chain("swiglu", "attention", ["attention_kernel"], reads=("q", "k", "v"), war=True, side_stream=True)
def chain_swiglu_to_attention_over_its_input():
    ops, c = _ops(), Chain(8)
    B, L, H = 2, 700, 2
    F = 3 * H * 64
    hid, G = c.inp("hid", B * L, 2 * F), c.buf("g", B * L, F)
    qkv = G.view(B, L, 3, H, 64)
    out = hid[:, :H * 64].unflatten(0, (B, L)).unflatten(-1, (H, 64))    # over the gate half swiglu reads
    c.producer = lambda: ops.swiglu(hid, F, out=G)
    c.consumer = lambda: ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], out=out)

    def check(bf, af):
        q = bf["g"].view(B, L, 3, H, 64)
        o = af["hid"][:, :H * 64].reshape(B, L, H, 64)
        _check_attention(o, q[:, :, 0], q[:, :, 1], q[:, :, 2], "attention over swiglu's input")
    c.check = check
    c.finite = [G, hid]
    return c


@chain("linear", "attention", ["attention_kernel"], reads=("q",),
       source="vae.py:116-123 (c_q with the fused q LayerNorm -> cross attention over the latents, out in place)")
def chain_geo_c_q_to_attention():
    ops, c = _ops(), Chain(9)
    n, W, nl = 3000, 128, 48
    xn, q = c.inp("xn", n, W), c.buf("q", n, W)
    kv = c.inp("kv", 1, nl, W // 64, 2, 64)
    w, b = c.randn(W, W, std=W ** -0.5), c.randn(W)
    qw, qb = c.randn(64, mean=1.0, std=0.1), c.randn(64, std=0.1)
    q4 = q.view(1, n, W // 64, 64)
    c.producer = lambda: ops.linear(xn, w, b, out=q, qk_norm=dict(mode=ops.QKN_LAYERNORM, q_col0=0, k_col0=None,
                                                                  cols=W, eps=1e-6, q_w=qw, q_b=qb))
    c.consumer = lambda: ops.attention(q4, kv[:, :, :, 0], kv[:, :, :, 1], out=q4)
    c.check = lambda bf, af: _check_attention(af["q"].view(q4.shape), bf["q"].view(q4.shape), bf["kv"][:, :, :, 0],
                                              bf["kv"][:, :, :, 1], "geo cross attention")
    c.finite = [q]
    return c


@chain("linear", "attention", ["attention_kernel"], reads=("q", "k", "v"),
       source="dit.py:262-268 (the streams' qkv projection -> joint attention, out over q)")
def chain_dit_qkv_to_attention():
    ops, c = _ops(), Chain(10)
    B, L, H, nh = 2, 444, 128, 2
    XM, QKV = c.inp("xm", B, L, H), c.buf("qkv", B, L, 3 * H)
    w, b = c.randn(3 * H, H, std=H ** -0.5), c.randn(3 * H)
    q4 = QKV.view(B, L, 3, nh, 64)
    c.producer = lambda: ops.linear(XM, w, b, out=QKV)
    c.consumer = lambda: ops.attention(q4[:, :, 0], q4[:, :, 1], q4[:, :, 2], out=q4[:, :, 0])

    def check(bf, af):
        q = bf["qkv"].view(B, L, 3, nh, 64)
        _check_attention(af["qkv"].view(B, L, 3, nh, 64)[:, :, 0], q[:, :, 0], q[:, :, 1], q[:, :, 2], "dit attention")
    c.check = check
    c.finite = [QKV]
    return c


# --- layernorm
@chain("swiglu", "layernorm", ["layernorm_kernel<4>"], reads=("x",))
def chain_swiglu_to_layernorm_affine():
    ops, c = _ops(), Chain(11)
    M, F = 16384, 1024
    hid, G, Y = c.inp("hid", M, 2 * F), c.buf("g", M, F), c.buf("y", M, F, value=NEG_INF)
    lw, lb = c.randn(F, mean=1.0, std=0.1), c.randn(F, std=0.1)
    c.producer = lambda: ops.swiglu(hid, F, out=G)
    c.consumer = lambda: ops.layernorm(G, lw, lb, eps=1e-6, out=Y)
    c.finite = [G, Y]
    return c


@chain("gemv", "layernorm", ["layernorm_kernel<4>"], reads=("scale", "shift"),
       source="dit.py:224,253 (the modulation GEMV gives the LayerNorm's scale / shift)")
def chain_gemv_to_layernorm_modulated():
    ops, c = _ops(), Chain(12)
    B, L, W, K = 2, 3000, 512, 4096
    vec, mods = c.inp("vec", B, K), c.buf("mods", B, 2 * W)
    x, Y = c.inp("x", B, L, W), c.buf("y", B, L, W, value=NEG_INF)
    wm, bm = c.randn(2 * W, K, std=K ** -0.5), c.randn(2 * W)
    c.producer = lambda: ops.gemv(wm, bm, vec, silu_in=True, out=mods)
    c.consumer = lambda: ops.layernorm(x, eps=1e-6, shift=mods[:, :W], scale=mods[:, W:], rows_per_batch=L, out=Y)
    c.finite = [mods, Y]
    return c


@chain("layernorm", "layernorm", ["layernorm_kernel<4>"], reads=("x",),
       source="dit.py:251-253 (the img stream's modulated LayerNorm, then the txt stream's: segmented rows)")
def chain_layernorm_to_layernorm_segmented():
    ops, c = _ops(), Chain(13)
    B, Lt, Li, W = 2, 1370, 3072, 256
    L = Lt + Li
    X, Y, XM = c.inp("X", B, L, W), c.buf("y", B, L, W), c.buf("xm", B, L, W, value=NEG_INF)
    sc, sh = c.inp("sc", B, W, std=0.2), c.inp("sh", B, W, std=0.2)
    c.producer = lambda: ops.layernorm(X, eps=1e-6, scale=sc, shift=sh, rows_per_batch=L, out=Y)
    c.consumer = lambda: ops.layernorm(Y[:, :Lt], eps=1e-6, scale=sc, shift=sh, rows_per_batch=Lt, out=XM[:, :Lt])
    c.finite = [Y, XM[:, :Lt]]
    return c


@chain("bilinear_nhwc", "layernorm", ["layernorm_kernel<8>"], reads=("x",))
def chain_bilinear_to_layernorm_wide():
    ops, c = _ops(), Chain(14)
    N, Hi, Wi, C, Ho, Wo = 1, 40, 48, 2048, 64, 80
    x, Y, Z = c.inp("x", N, Hi, Wi, C), c.buf("y", N, Ho, Wo, C), c.buf("z", N * Ho * Wo, C, value=NEG_INF)
    lw, lb = c.randn(C, mean=1.0, std=0.1), c.randn(C, std=0.1)
    c.producer = lambda: ops.bilinear_nhwc(x, Ho, Wo, out=Y)
    c.consumer = lambda: ops.layernorm(Y.view(-1, C), lw, lb, eps=1e-6, out=Z)
    c.finite = [Y, Z]
    return c


@chain("swiglu", "layernorm", ["layernorm_kernel<4>"], war=True)
def chain_swiglu_then_layernorm_in_place_over_its_input():
    ops, c = _ops(), Chain(15)
    M, F = 16384, 512
    hid, G = c.inp("hid", M, 2 * F), c.buf("g", M, F)
    lw, lb = c.randn(F, mean=1.0, std=0.1), c.randn(F, std=0.1)
    c.producer = lambda: ops.swiglu(hid, F, out=G)
    c.consumer = lambda: ops.layernorm(hid[:, :F], lw, lb, eps=1e-6, out=hid[:, :F])
    c.finite = [G, hid]
    return c


@chain("linear", "layernorm", ["layernorm_kernel<4>"], reads=("x",),
       source="vae.py:113-114 (query_proj -> ln_1 of a geo-decoder chunk)")
def chain_geo_query_proj_to_ln1():
    ops, c = _ops(), Chain(16)
    n, W = 8000, 128
    emb, x, xn = c.inp("emb", n, 64), c.buf("x", n, W), c.buf("xn", n, W, value=NEG_INF)
    w, b = c.randn(W, 64, std=0.125), c.randn(W)
    lw, lb = c.randn(W, mean=1.0, std=0.1), c.randn(W, std=0.1)
    c.producer = lambda: ops.linear(emb, w, b, out=x)
    c.consumer = lambda: ops.layernorm(x, lw, lb, eps=1e-6, out=xn)
    c.finite = [x, xn]
    return c


@chain("linear", "layernorm", ["layernorm_kernel<4>"], reads=("x",),
       source="dit.py:269-274 (gated residual projection in place -> the next modulated LayerNorm)")
def chain_dit_proj_to_layernorm():
    ops, c = _ops(), Chain(17)
    B, L, H = 2, 444, 128
    src, X, XM = c.inp("src", B, L, H), c.inp("X", B, L, H), c.buf("xm", B, L, H, value=NEG_INF)
    gate, sc, sh = c.inp("gate", B, H, std=0.5), c.inp("sc", B, H, std=0.2), c.inp("sh", B, H, std=0.2)
    w, b = c.randn(H, H, std=H ** -0.5), c.randn(H)
    c.producer = lambda: ops.linear(src, w, b, gate=gate, gate_rows=L, residual=X, out=X)
    c.consumer = lambda: ops.layernorm(X, eps=1e-6, scale=sc, shift=sh, rows_per_batch=L, out=XM)
    c.finite = [X, XM]
    return c


# --- lnpost_dot
def _lnpost(c, W):
    return (c.randn(W, mean=1.0, std=0.1), c.randn(W, std=0.1), c.randn(W, std=W ** -0.5), c.randn(1))


def _check_lnpost(out, x, p, what):
    import fp16_ref as R
    R.check_bound(out, *R.lnpost_dot(x, *p, eps=1e-5), what)


@chain("layernorm", "lnpost_dot", ["lnpost_dot_kernel<4>"], reads=("x",))
def chain_layernorm_to_lnpost_dot():
    ops, c = _ops(), Chain(18)
    n, W = 65536, 1024
    x, Y, out = c.inp("x", n, W), c.buf("y", n, W), c.buf("out", n, value=NEG_INF, dtype=F32)
    lw, lb, p = c.randn(W, mean=1.0, std=0.1), c.randn(W, std=0.1), _lnpost(c, W)
    c.producer = lambda: ops.layernorm(x, lw, lb, eps=1e-6, out=Y)
    c.consumer = lambda: ops.lnpost_dot(Y, *p, out, eps=1e-5)
    c.check = lambda bf, af: _check_lnpost(af["out"], bf["y"], p, "lnpost_dot<4>")
    c.finite = [Y, out]
    return c


@chain("swiglu", "lnpost_dot", ["lnpost_dot_kernel<8>"], reads=("x",))
def chain_swiglu_to_lnpost_dot_wide():
    ops, c = _ops(), Chain(19)
    n, F = 8192, 2048
    hid, G, out = c.inp("hid", n, 2 * F), c.buf("g", n, F), c.buf("out", n, value=NEG_INF, dtype=F32)
    p = _lnpost(c, F)
    c.producer = lambda: ops.swiglu(hid, F, out=G)
    c.consumer = lambda: ops.lnpost_dot(G, *p, out, eps=1e-5)
    c.check = lambda bf, af: _check_lnpost(af["out"], bf["g"], p, "lnpost_dot<8>")
    c.finite = [G, out]
    return c


@chain("layernorm_f32", "lnpost_dot", ["lnpost_dot_kernel<4>"], war=True)
def chain_layernorm_f32_then_lnpost_dot_over_its_input():
    ops, c = _ops(), Chain(20)
    rows, width, n, W = 4, 1 << 21, 4096, 256
    r, Y = c.inp("r", rows, width, dtype=F32), c.buf("y", rows, width, dtype=F32)
    x = c.inp("x", n, W)
    p = _lnpost(c, W)
    out = r.view(-1)[:n]                       # the first values of row 0, which the LayerNorm reads in every pass
    c.producer = lambda: ops.layernorm_f32(r, eps=1e-5, out=Y)
    c.consumer = lambda: ops.lnpost_dot(x, *p, out, eps=1e-5)
    c.check = lambda bf, af: _check_lnpost(af["r"].view(-1)[:n], bf["x"], p, "lnpost_dot over layernorm_f32's input")
    c.finite = [Y, r]
    return c


@chain("linear", "lnpost_dot", ["lnpost_dot_kernel<4>"], reads=("x",),
       source="vae.py:129-130 (mlp_proj with the residual in place -> ln_post + output_proj)")
def chain_geo_mlp_proj_to_lnpost_dot():
    ops, c = _ops(), Chain(21)
    n, W = 8000, 128
    h, x, out = c.inp("h", n, 4 * W), c.inp("x", n, W), c.buf("out", n, value=NEG_INF, dtype=F32)
    w, b, p = c.randn(W, 4 * W, std=(4 * W) ** -0.5), c.randn(W), _lnpost(c, W)
    c.producer = lambda: ops.linear(h, w, b, out=x, residual=x)
    c.consumer = lambda: ops.lnpost_dot(x, *p, out, eps=1e-5)
    c.check = lambda bf, af: _check_lnpost(af["out"], bf["x"], p, "geo lnpost_dot")
    c.finite = [x, out]
    return c


# --- gemv
@chain("gemv", "gemv", ["gemv_kernel<1>"], reads=("vec",),
       source="dit.py:214-215 (time_in: in_layer with SiLU -> out_layer), one sample")
def chain_gemv_to_gemv_b1():
    ops, c = _ops(), Chain(22)
    K, N, N2 = 4096, 8192, 1024
    temb, v0, vec = c.inp("temb", 1, K), c.buf("v0", 1, N), c.buf("vec", 1, N2, value=NEG_INF)
    w1, b1, w2, b2 = c.randn(N, K, std=K ** -0.5), c.randn(N), c.randn(N2, N, std=N ** -0.5), c.randn(N2)
    c.producer = lambda: ops.gemv(w1, b1, temb, silu_out=True, out=v0)
    c.consumer = lambda: ops.gemv(w2, b2, v0, out=vec)
    c.finite = [v0, vec]
    return c


@chain("gemv", "gemv", ["gemv_kernel<2>"], reads=("vec",),
       source="dit.py:215-224 (time_in.out_layer -> the modulation GEMV with SiLU on its input), CFG batch")
def chain_gemv_to_gemv_b2_silu_in():
    ops, c = _ops(), Chain(23)
    K, N, N2 = 1024, 4096, 8192
    v0, vec, mods = c.inp("v0", 2, K), c.buf("vec", 2, N), c.buf("mods", 2, N2, value=NEG_INF)
    w1, b1, w2, b2 = c.randn(N, K, std=K ** -0.5), c.randn(N), c.randn(N2, N, std=N ** -0.5), c.randn(N2)
    c.producer = lambda: ops.gemv(w1, b1, v0, out=vec)
    c.consumer = lambda: ops.gemv(w2, b2, vec, silu_in=True, out=mods)
    c.finite = [vec, mods]
    return c


@chain("swiglu", "gemv", ["gemv_kernel<4>"], reads=("vec",), war=True)
def chain_swiglu_to_gemv_b3_over_its_input():
    ops, c = _ops(), Chain(24)
    M, F, N = 8192, 2048, 2048
    hid, G = c.inp("hid", M, 2 * F), c.buf("g", M, F)
    w, b = c.randn(N, F, std=F ** -0.5), c.randn(N)
    out = hid[:3, :N]                          # over rows swiglu reads
    c.producer = lambda: ops.swiglu(hid, F, out=G)
    c.consumer = lambda: ops.gemv(w, b, G[M - 3:], out=out)        # the last rows swiglu writes
    c.finite = [G, hid]
    return c


@chain("layernorm", "gemv", ["gemv_kernel<8>"], reads=("vec",))
def chain_layernorm_to_gemv_b6():
    ops, c = _ops(), Chain(25)
    M, K, N = 32768, 1024, 8192
    x, Y, out = c.inp("x", M, K), c.buf("y", M, K), c.buf("out", 6, N, value=NEG_INF)
    w, b = c.randn(N, K, std=K ** -0.5), c.randn(N)
    c.producer = lambda: ops.layernorm(x, eps=1e-6, out=Y)
    c.consumer = lambda: ops.gemv(w, b, Y[M - 6:], out=out)        # the last rows the LayerNorm writes
    c.finite = [Y, out]
    return c


@chain("gemv", "gemv", ["gemv_kernel<2>"], reads=("vec", "residual"),
       source="dit.py:220-223 (guidance_in: in_layer -> out_layer added to vec in place, residual aliasing out)")
def chain_gemv_to_gemv_residual_alias():
    ops, c = _ops(), Chain(26)
    K, N = 256, 1024
    gemb, P = c.inp("gemb", 2, K), c.buf("p", 2, 2 * N)
    w1, b1, w2, b2 = c.randn(2 * N, K, std=K ** -0.5), c.randn(2 * N), c.randn(N, N, std=N ** -0.5), c.randn(N)
    vec = P[:, N:]
    c.producer = lambda: ops.gemv(w1, b1, gemb, silu_out=True, out=P)
    c.consumer = lambda: ops.gemv(w2, b2, P[:, :N], residual=vec, out=vec)
    c.finite = [P]
    return c


@chain("gemv", "linear", ["linear_kernel<128>"], source="dit.py:224-225 (the modulation GEMV -> latent_in)")
def chain_dit_mods_to_latent_in():
    ops, c = _ops(), Chain(27)
    K, N, B, Li, H = 1024, 6144, 2, 3072, 128
    vec, mods = c.inp("vec", B, K), c.buf("mods", B, N)
    x, img = c.inp("x", B, Li, 64), c.buf("img", B, Li, H, value=NEG_INF)
    wm, bm, w, b = c.randn(N, K, std=K ** -0.5), c.randn(N), c.randn(H, 64, std=0.125), c.randn(H)
    c.producer = lambda: ops.gemv(wm, bm, vec, silu_in=True, out=mods)
    c.consumer = lambda: ops.linear(x, w, b, out=img)
    c.check = lambda bf, af: _check_linear(af["img"].view(-1, H), bf["x"].view(-1, 64), w, b, "latent_in")
    c.finite = [mods, img]
    return c


# --- swiglu
@chain("layernorm", "swiglu", ["swiglu_kernel"], reads=("x",), war=True, side_stream=True)
def chain_layernorm_to_swiglu_over_its_input():
    ops, c = _ops(), Chain(28)
    M, F = 16384, 512
    A, Y = c.inp("A", M, 2 * F), c.buf("y", M, 2 * F)
    c.producer = lambda: ops.layernorm(A, eps=1e-6, out=Y)
    c.consumer = lambda: ops.swiglu(Y, F, out=A[:, F:])

    def check(bf, af):
        import fp16_ref as R
        R.check_bound(af["A"][:, F:], *R.swiglu(bf["y"], F), "swiglu")
    c.check = check
    c.finite = [Y, A]
    return c


# --- gemv_f32 (the camera head's float32 GEMVs)
@chain("layernorm_f32", "gemv_f32", ["gemv_f32_kernel<1>"], reads=("vec",), war=True)
def chain_layernorm_f32_to_gemv_f32_over_its_input():
    ops, c = _ops(), Chain(29)
    width, K, N = 1 << 22, 2048, 4096
    r, Y = c.inp("r", 1, width, dtype=F32), c.buf("y", 1, width, dtype=F32)
    w, b = c.randn(N, K, std=K ** -0.5), c.randn(N, dtype=F32)
    c.producer = lambda: ops.layernorm_f32(r, eps=1e-5, out=Y)
    c.consumer = lambda: ops.gemv_f32(w, b, Y[:, :K], out=r[:, :N])   # the first values the LayerNorm writes, and reads
    c.finite = [Y, r]
    return c


@chain("small_attention_f32", "gemv_f32", ["gemv_f32_kernel<2>"], reads=("vec",),
       source="vggt_heads.py:125-126 (trunk attention -> proj with LayerScale residual)")
def chain_camera_attention_to_proj():
    ops, c = _ops(), Chain(30)
    S, H, D = 2, 16, 128
    C = H * D
    qkv, o = c.inp("qkv", S, 3 * C, dtype=F32), c.buf("o", S, C, dtype=F32)
    x, out = c.inp("x", S, C, dtype=F32), c.buf("out", S, C, value=NEG_INF, dtype=F32)
    w, b, gm = c.randn(C, C, std=C ** -0.5), c.randn(C, dtype=F32), c.randn(C, mean=0.5, std=0.1, dtype=F32)
    c.producer = lambda: ops.small_attention_f32(qkv, 1, S, H, D, out=o)
    c.consumer = lambda: ops.gemv_f32(w, b, o, residual=x, gamma=gm, out=out)
    c.finite = [o, out]
    return c


@chain("gemv_f32", "gemv_f32", ["gemv_f32_kernel<4>"], reads=("vec", "residual"),
       source="vggt_heads.py:128-129 (fc1 with GELU -> fc2 with LayerScale residual)")
def chain_camera_fc1_to_fc2():
    ops, c = _ops(), Chain(31)
    B, K, N, C = 4, 2048, 8192, 2048
    x, P = c.inp("x", B, K, dtype=F32), c.buf("p", B, N + C, dtype=F32)
    Q = c.buf("q", B, N + C, value=NEG_INF, dtype=F32)
    w1, b1 = c.randn(N + C, K, std=K ** -0.5), c.randn(N + C, dtype=F32)
    w2, b2, gm = c.randn(C, N, std=N ** -0.5), c.randn(C, dtype=F32), c.randn(C, mean=0.5, std=0.1, dtype=F32)
    c.producer = lambda: ops.gemv_f32(w1, b1, x, gelu_out=True, out=P)
    c.consumer = lambda: ops.gemv_f32(w2, b2, P[:, :N], residual=P[:, N:], gamma=gm, out=Q[:, :C])
    c.finite = [P, Q[:, :C]]
    return c


@chain("lnpost_dot", "gemv_f32", ["gemv_f32_kernel<8>"], reads=("vec",))
def chain_lnpost_dot_to_gemv_f32_b8():
    ops, c = _ops(), Chain(32)
    n, W, N = 32768, 1024, 1024
    x, lg, out = c.inp("x", n, W), c.buf("lg", n, dtype=F32), c.buf("out", 8, N, value=NEG_INF, dtype=F32)
    p = _lnpost(c, W)
    w, b = c.randn(N, n // 8, std=(n // 8) ** -0.5), c.randn(N, dtype=F32)
    c.producer = lambda: ops.lnpost_dot(x, *p, lg, eps=1e-5)
    c.consumer = lambda: ops.gemv_f32(w, b, lg.view(8, n // 8), silu_in=True, out=out)
    c.finite = [lg, out]
    return c


@chain("layernorm_f32", "gemv_f32", ["gemv_f32_kernel<2>"], reads=("vec",),
       source="vggt_heads.py:123-124 (norm1 -> qkv)")
def chain_camera_norm1_to_qkv():
    ops, c = _ops(), Chain(33)
    S, C = 2, 2048
    x, h, qkv = c.inp("x", S, C, dtype=F32), c.buf("h", S, C, dtype=F32), c.buf("qkv", S, 3 * C, value=NEG_INF, dtype=F32)
    lw, lb = c.randn(C, mean=1.0, std=0.1, dtype=F32), c.randn(C, std=0.1, dtype=F32)
    w, b = c.randn(3 * C, C, std=C ** -0.5), c.randn(3 * C, dtype=F32)
    c.producer = lambda: ops.layernorm_f32(x, lw, lb, eps=1e-5, out=h)
    c.consumer = lambda: ops.gemv_f32(w, b, h, out=qkv)
    c.finite = [h, qkv]
    return c


# --- layernorm_f32
@chain("gemv_f32", "layernorm_f32", ["layernorm_f32_kernel"], reads=("x",),
       source="vggt_heads.py:126-127 (proj with LayerScale residual -> norm2)")
def chain_camera_proj_to_norm2():
    ops, c = _ops(), Chain(34)
    S, C = 2, 2048
    o, x, x2 = c.inp("o", S, C, dtype=F32), c.inp("x", S, C, dtype=F32), c.buf("x2", S, C, dtype=F32)
    h = c.buf("h", S, C, value=NEG_INF, dtype=F32)
    w, b, gm = c.randn(C, C, std=C ** -0.5), c.randn(C, dtype=F32), c.randn(C, mean=0.5, std=0.1, dtype=F32)
    lw, lb = c.randn(C, mean=1.0, std=0.1, dtype=F32), c.randn(C, std=0.1, dtype=F32)
    c.producer = lambda: ops.gemv_f32(w, b, o, residual=x, gamma=gm, out=x2)
    c.consumer = lambda: ops.layernorm_f32(x2, lw, lb, eps=1e-5, out=h)
    c.finite = [x2, h]
    return c


@chain("gemv_f32", "layernorm_f32", ["layernorm_f32_kernel"], reads=("shift", "scale", "gate"),
       source="vggt_heads.py:118-120 (poseLN_modulation -> the gated, modulated LayerNorm)")
def chain_camera_modulation_to_gated_layernorm():
    ops, c = _ops(), Chain(35)
    S, C = 2, 2048
    emb, mod = c.inp("emb", S, C, dtype=F32), c.buf("mod", S, 3 * C, dtype=F32)
    x0, x = c.inp("x0", S, C, dtype=F32), c.buf("x", S, C, value=NEG_INF, dtype=F32)
    w, b = c.randn(3 * C, C, std=C ** -0.5), c.randn(3 * C, dtype=F32)
    c.producer = lambda: ops.gemv_f32(w, b, emb, silu_in=True, out=mod)
    c.consumer = lambda: ops.layernorm_f32(x0, eps=1e-6, shift=mod[:, :C], scale=mod[:, C:2 * C], gate=mod[:, 2 * C:],
                                           out=x)
    c.finite = [mod, x]
    return c


@chain("lnpost_dot", "layernorm_f32", ["layernorm_f32_kernel"], reads=("x",), war=True)
def chain_lnpost_dot_to_layernorm_f32_over_its_input():
    ops, c = _ops(), Chain(36)
    n, W, rows = 65536, 1024, 128
    x, lg = c.inp("x", n, W), c.buf("lg", n, dtype=F32)
    p = _lnpost(c, W)
    y = x.view(F32)[:rows]                        # float32 rows laid over the first fp16 rows lnpost_dot reads
    c.producer = lambda: ops.lnpost_dot(x, *p, lg, eps=1e-5)
    c.consumer = lambda: ops.layernorm_f32(lg.view(rows, n // rows), eps=1e-5, out=y)
    c.finite = [lg, y]
    return c


# --- small_attention_f32, every head width
def _small_attention_chain(seed, D, producer):
    ops, c = _ops(), Chain(seed)
    B, S, H = (1, 2, 4) if producer == "gemv_f32" else (8, 64, 2)
    M, Wq = B * S, 3 * H * D
    out = c.buf("out", M, H * D, value=NEG_INF, dtype=F32)
    if producer == "gemv_f32":
        K = 2048
        x, qkv = c.inp("x", M, K, dtype=F32), c.buf("qkv", M, Wq, dtype=F32)
        w, b = c.randn(Wq, K, std=K ** -0.5), c.randn(Wq, dtype=F32)
        c.producer = lambda: ops.gemv_f32(w, b, x, out=qkv)
        c.consumer = lambda: ops.small_attention_f32(qkv, B, S, H, D, out=out)
    else:
        # the attention's output overwrites the start of the LayerNorm's input
        x, qkv = c.inp("x", M, Wq, dtype=F32), c.buf("qkv", M, Wq, dtype=F32)
        o = x.view(-1)[:M * H * D].view(M, H * D)
        c.producer = lambda: ops.layernorm_f32(x, eps=1e-5, out=qkv)
        c.consumer = lambda: ops.small_attention_f32(qkv, B, S, H, D, out=o)
        out = o
    c.finite = [qkv, out]
    return c


for _i, (_D, _prod) in enumerate(((32, "layernorm_f32"), (64, "gemv_f32"), (128, "gemv_f32"), (256, "layernorm_f32"))):
    def _build(_D=_D, _prod=_prod, _i=_i):
        return _small_attention_chain(40 + _i, _D, _prod)
    _build.__name__ = f"chain_{_prod}_to_small_attention_f32_d{_D}"
    chain(_prod, "small_attention_f32", [f"small_attention_f32_kernel<{_D // 32}>"], reads=("qkv",),
          war=_prod == "layernorm_f32",
          source="vggt_heads.py:124-125 (qkv -> trunk attention)" if _D == 128 else None)(_build)


# --- im2col3x3 / bilinear_nhwc (the DPT head)
@chain("bilinear_nhwc", "im2col3x3", ["im2col3x3_kernel"], reads=("x",))
def chain_bilinear_to_im2col_stride1():
    ops, c = _ops(), Chain(50)
    N, Hi, Wi, C, Ho, Wo = 2, 64, 64, 128, 128, 128
    x, Y = c.inp("x", N, Hi, Wi, C), c.buf("y", N, Ho, Wo, C)
    cols = c.buf("cols", N * Ho * Wo, 9 * C, value=NEG_INF)
    c.producer = lambda: ops.bilinear_nhwc(x, Ho, Wo, out=Y)
    c.consumer = lambda: ops.im2col3x3(Y, stride=1, out=cols)
    c.finite = [Y, cols]
    return c


@chain("layernorm", "im2col3x3", ["im2col3x3_kernel"], reads=("x",), war=True)
def chain_layernorm_to_im2col_stride2_over_its_input():
    ops, c = _ops(), Chain(51)
    N, H, W, C = 2, 96, 96, 256
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    A, Y = c.inp("A", N * H * W * 3, C), c.buf("y", N * H * W * 3, C)
    cols = A.view(-1)[:N * Ho * Wo * 9 * C].view(N * Ho * Wo, 9 * C)
    c.producer = lambda: ops.layernorm(A, eps=1e-6, out=Y)
    c.consumer = lambda: ops.im2col3x3(Y[:N * H * W].view(N, H, W, C), stride=2, relu_in=True, out=cols)
    c.finite = [Y, A]
    return c


@chain("im2col3x3", "bilinear_nhwc", ["bilinear_nhwc_kernel"], reads=("x",))
def chain_im2col_to_bilinear_up():
    ops, c = _ops(), Chain(52)
    N, H, W, C = 2, 64, 64, 64
    x, cols = c.inp("x", N, H, W, C), c.buf("cols", N * H * W, 9 * C)
    out = c.buf("out", N, 2 * H, 2 * W, 9 * C, value=NEG_INF)
    c.producer = lambda: ops.im2col3x3(x, out=cols)
    c.consumer = lambda: ops.bilinear_nhwc(cols.view(N, H, W, 9 * C), 2 * H, 2 * W, out=out)
    c.finite = [cols, out]
    return c


@chain("layernorm", "bilinear_nhwc", ["bilinear_nhwc_kernel"], reads=("x",), war=True, side_stream=True)
def chain_layernorm_to_bilinear_down_over_its_input():
    ops, c = _ops(), Chain(53)
    N, H, W, C, Ho, Wo = 2, 128, 128, 256, 37, 45
    A, Y = c.inp("A", N * H * W, C), c.buf("y", N * H * W, C)
    out = A.view(-1)[:N * Ho * Wo * C].view(N, Ho, Wo, C)
    c.producer = lambda: ops.layernorm(A, eps=1e-6, out=Y)
    c.consumer = lambda: ops.bilinear_nhwc(Y.view(N, H, W, C), Ho, Wo, out=out)
    c.finite = [Y, A]
    return c


@chain("im2col3x3", "linear", ["linear_kernel<128>"], reads=("x",),
       source="vggt_heads.py:315-317 (a fusion stage's 3x3 convolution: im2col -> GEMM with ReLU)")
def chain_dpt_im2col_to_conv():
    ops, c = _ops(), Chain(54)
    N, H, W, C = 2, 28, 28, 32
    x, cols = c.inp("x", N, H, W, C), c.buf("cols", N * H * W, 9 * C)
    y = c.buf("y", N * H * W, C, value=NEG_INF)
    w, b = c.randn(C, 9 * C, std=(9 * C) ** -0.5), c.randn(C)
    c.producer = lambda: ops.im2col3x3(x, out=cols)
    c.consumer = lambda: ops.linear(cols, w, b, act=ops.ACT_RELU, out=y)
    c.check = lambda bf, af: _check_linear(af["y"], bf["cols"], w, b, "dpt conv1", act=3)
    c.finite = [cols, y]
    return c


@chain("linear", "im2col3x3", ["im2col3x3_kernel"], reads=("x",),
       source="vggt_heads.py:331-332 (conv1's GEMM -> conv2's im2col)")
def chain_dpt_conv1_to_im2col():
    ops, c = _ops(), Chain(55)
    N, H, W, C = 2, 28, 28, 32
    cols, y = c.inp("cols", N * H * W, 9 * C), c.buf("y", N * H * W, C)
    cols2 = c.buf("cols2", N * H * W, 9 * C, value=NEG_INF)
    w, b = c.randn(C, 9 * C, std=(9 * C) ** -0.5), c.randn(C)
    c.producer = lambda: ops.linear(cols, w, b, act=ops.ACT_RELU, out=y)
    c.consumer = lambda: ops.im2col3x3(y.view(N, H, W, C), out=cols2)
    c.finite = [y, cols2]
    return c


@chain("linear", "bilinear_nhwc", ["bilinear_nhwc_kernel"], reads=("x",),
       source="vggt_heads.py:332,339 (conv2 with the skip as residual -> the stage's bilinear resampling)")
def chain_dpt_conv2_to_bilinear():
    ops, c = _ops(), Chain(56)
    N, H, W, C = 2, 28, 28, 32
    cols, skip, y = c.inp("cols", N * H * W, 9 * C), c.inp("skip", N * H * W, C), c.buf("y", N * H * W, C)
    out = c.buf("out", N, 2 * H, 2 * W, C, value=NEG_INF)
    w, b = c.randn(C, 9 * C, std=(9 * C) ** -0.5), c.randn(C)
    c.producer = lambda: ops.linear(cols, w, b, residual=skip, out=y)
    c.consumer = lambda: ops.bilinear_nhwc(y.view(N, H, W, C), 2 * H, 2 * W, out=out)
    c.finite = [y, out]
    return c


@chain("bilinear_nhwc", "linear", ["linear_kernel<128>"], reads=("x",),
       source="vggt_heads.py:339 (the stage's bilinear resampling -> out_conv, a 1x1 convolution)")
def chain_dpt_bilinear_to_out_conv():
    ops, c = _ops(), Chain(57)
    N, H, W, C = 2, 28, 28, 32
    x, up = c.inp("x", N, H, W, C), c.buf("up", N, 2 * H, 2 * W, C)
    y = c.buf("y", N * 4 * H * W, C, value=NEG_INF)
    w, b = c.randn(C, C, std=C ** -0.5), c.randn(C)
    c.producer = lambda: ops.bilinear_nhwc(x, 2 * H, 2 * W, out=up)
    c.consumer = lambda: ops.linear(up.view(-1, C), w, b, out=y)
    c.check = lambda bf, af: _check_linear(af["y"], bf["up"].view(-1, C), w, b, "dpt out_conv")
    c.finite = [up, y]
    return c


# ------------------------------------------------------------------------------------------------------ chain runs
def _same(a, b):
    """Bit equality (NaN payloads included)."""
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def run_serialized(c):
    c.reset()
    torch.cuda.synchronize()
    c.producer()
    torch.cuda.synchronize()
    before = c.snap()
    c.consumer()
    torch.cuda.synchronize()
    return before, c.snap()


def run_back_to_back(c, stream=None, sleep_cycles=2_000_000):
    """The two launches one after the other.  A torch sleep kernel before them holds the stream for about a
    millisecond, so that both are queued before the producer starts and the consumer can start under its tail however
    long the host takes between the two calls."""
    c.reset()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream) if stream is not None else contextlib.nullcontext():
        torch.cuda._sleep(sleep_cycles)
        c.producer()
        c.consumer()
    torch.cuda.synchronize()
    return c.snap()


def run_graph(c):
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        c.producer()
        c.consumer()
    c.reset()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    out = c.snap()
    del g
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("spec", CHAINS, ids=lambda s: s.name[len("chain_"):])
def test_chain_back_to_back_and_graph_equal_serialized(spec):
    c = spec.build()
    before, ref = run_serialized(c)
    for i, v in enumerate(c.finite):
        assert torch.isfinite(v).all(), f"{spec.name}: finite view {i} holds a non-finite value after the serialized run"
    if c.check is not None:
        c.check(before, ref)
    side = torch.cuda.Stream() if spec.side_stream else None
    for mode, got in (("back to back" + (" on a side stream" if side else ""), run_back_to_back(c, side)),
                      ("graph replay", run_graph(c))):
        for k in ref:
            assert _same(got[k], ref[k]), f"{spec.name}: buffer {k!r} differs from the serialized run ({mode})"


# -------------------------------------------------------------------------------------------- whole forwards, PDL off
# PDL kernels the forwards below do not reach (their shapes are too small); the chains above cover them.
NOT_REACHED_BY_FORWARDS = {"layernorm_kernel<8>", "lnpost_dot_kernel<8>", "gemv_kernel<1>", "gemv_kernel<4>",
                           "gemv_kernel<8>", "gemv_f32_kernel<1>", "gemv_f32_kernel<4>", "gemv_f32_kernel<8>",
                           "small_attention_f32_kernel<1>", "small_attention_f32_kernel<2>",
                           "small_attention_f32_kernel<8>"}


def _golden(name):
    root = os.path.dirname(os.path.abspath(__file__))
    return np.load(os.path.join(root, "golden", name))


def _sd(z, prefix="w:"):
    return {k[len(prefix):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(prefix)}


def forwards():
    """Seeded model forwards, eager and graph-replayed: name -> output tensor on the CPU."""
    import types
    from r3g.conditioner import DinoImageEncoder
    from r3g.dit import Hunyuan3DDiT
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline, ImageProcessorV2
    from r3g.scheduler import FlowMatchEulerDiscreteScheduler
    from r3g.vae import FlashVDMVolumeDecoding, ShapeVAE
    from r3g.vggt import Aggregator
    from r3g.vggt_heads import CameraHeadR3G, DPTHeadR3G, random_state_dict
    out = {}
    with torch.no_grad():
        # DiT: eager, eager with the collapsed unconditional text (kv_fill), and a 2-step CFG denoise (graph replay)
        z = _golden("dit_mini.npz")
        m = Hunyuan3DDiT(in_channels=64, context_in_dim=96, hidden_size=128, num_heads=2, depth=2, depth_single_blocks=2)
        m.load_state_dict(_sd(z))
        x, t = torch.from_numpy(z["x"]).cuda().half(), torch.from_numpy(z["t"]).cuda().half()
        cond = torch.from_numpy(z["cond"]).cuda().half()
        out["dit"] = m(x, t, {"main": cond}).clone()
        uncond = torch.cat([cond[:1], torch.zeros_like(cond[1:])])
        out["dit_collapsed"] = m(x, t, {"main": uncond}, uncond_txt_shared=True).clone()
        pipe = Hunyuan3DDiTFlowMatchingPipeline(
            vae=types.SimpleNamespace(latent_shape=tuple(x.shape[1:])), model=m,
            scheduler=FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000), conditioner=None,
            image_processor=ImageProcessorV2(size=512, border_ratio=0.15))
        lat0 = torch.randn((1,) + tuple(x.shape[1:]), generator=torch.manual_seed(7), dtype=torch.float16)
        out["dit_cfg_steps"] = pipe(cond={"main": uncond}, latents=lat0, num_inference_steps=2, guidance_scale=5.0,
                                    output_type="latent").clone()
        assert [k[-1] for k in pipe._graphs.entries] == [True], "the CFG step must run the collapsed branch"
        # ShapeVAE forward and the dense SDF grid (graph replay, then eager)
        z = _golden("vae_mini.npz")
        vae = ShapeVAE(num_latents=48, embed_dim=64, width=128, heads=int(z["cfg_heads"]),
                       num_decoder_layers=int(z["cfg_layers"]), num_freqs=8, include_pi=False, qkv_bias=False,
                       qk_norm=True)
        vae.load_state_dict(_sd(z))
        out["vae"] = vae(torch.from_numpy(z["z"]).cuda().half()).clone()
        lat = torch.from_numpy(z["latents"]).cuda().half()
        R = int(z["cfg_R"])
        out["sdf_graph"] = vae.volume_decoder(lat, vae.geo_decoder, bounds=1.01, num_chunks=100, octree_resolution=R).clone()
        vae.geo_decoder.use_cuda_graph = False
        out["sdf_eager"] = vae.volume_decoder(lat, vae.geo_decoder, bounds=1.01, num_chunks=100, octree_resolution=R).clone()
        # FlashVDM
        z = _golden("flashvdm_mini.npz")
        fv = ShapeVAE(num_latents=48, embed_dim=64, width=128, heads=int(z["cfg_heads"]), num_decoder_layers=0,
                      num_freqs=8, include_pi=False, qkv_bias=False, qk_norm=True)
        fv.geo_decoder.load(_sd(z))
        out["flashvdm"] = FlashVDMVolumeDecoding("mean")(
            torch.from_numpy(z["latents"]).cuda().half(), fv.geo_decoder, bounds=1.01,
            num_chunks=int(z["cfg_num_chunks"]), mc_level=0.0, octree_resolution=int(z["cfg_octree"]),
            min_resolution=int(z["cfg_min_resolution"]), enable_pbar=False).clone()
        # DINOv2 conditioner with the SwiGLU MLP, small random weights
        cfg = dict(hidden_size=192, num_hidden_layers=2, num_attention_heads=3, mlp_ratio=4, patch_size=14,
                   image_size=70, use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True, hidden_act="gelu",
                   layer_norm_eps=1e-6)
        torch.manual_seed(0)
        enc = DinoImageEncoder(config=cfg, image_size=70, device="cuda", dtype=torch.float16)
        assert enc.backend == "r3g"
        out["conditioner"] = enc(torch.rand(2, 3, 90, 90, generator=torch.manual_seed(1)) * 2 - 1).clone()
        # VGGT aggregator (graph replay, then eager)
        z = _golden("vggt_mini.npz")
        agg = Aggregator(img_size=56, patch_size=14, embed_dim=128, depth=2, num_heads=2, patch_embed="conv")
        agg.load_state_dict(_sd(z, "w:agg."))
        images = torch.from_numpy(z["agg_images"]).cuda()
        for mode in ("graph", "eager"):
            agg.use_cuda_graph = mode == "graph"
            for i, o in enumerate(agg(images)[0]):
                out[f"aggregator_{mode}_{i}"] = o.clone()
        # camera and DPT heads at the small geometry of tests/test_gpu_vggt.py (graph replay, then eager)
        sd = random_state_dict(7, embed_dim=128, depth=1, vit_depth=1, trunk_depth=2, features=32,
                               out_channels=(32, 64, 128, 128), img_size=56)
        cam = CameraHeadR3G({k: v for k, v in sd.items() if k.startswith("camera_head.")}, trunk_depth=2, num_heads=2)
        g = torch.Generator(device="cuda").manual_seed(2)
        toks = [torch.randn(1, 2, 7, 256, device="cuda", generator=g)]
        sd = random_state_dict(5, embed_dim=128, depth=1, vit_depth=1, trunk_depth=1, features=32,
                               out_channels=(32, 64, 128, 128), img_size=56)
        dpt = DPTHeadR3G({k: v.half().float() for k, v in sd.items() if k.startswith("depth_head.")},
                         intermediate_layer_idx=(0, 1, 0, 1))
        dtoks = [torch.randn(1, 2, 5 + 16, 256, device="cuda", generator=g) for _ in range(2)]
        imgs = torch.rand(1, 2, 3, 56, 56, device="cuda", generator=g)
        for mode in ("graph", "eager"):
            cam.use_cuda_graph = dpt.use_cuda_graph = mode == "graph"
            for i, o in enumerate(cam(toks)):
                out[f"camera_{mode}_{i}"] = o.clone()
            d, cf = dpt(dtoks, imgs, 5)
            out[f"dpt_depth_{mode}"], out[f"dpt_conf_{mode}"] = d.clone(), cf.clone()
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in out.items()}


def _pdl_kernels_in(names):
    """The CONSUMERS entries among profiler kernel names ('void (anonymous namespace)::gemv_kernel<2>(...)')."""
    import re
    found = set()
    for n in names:
        m = re.search(r"(\w+_kernel)(<(\d+)>)?\(", n)
        if m and m.group(1) in ENTRY:
            found.add(m.group(1) + (f"<{m.group(3)}>" if m.group(3) else ""))
    return found


@pytest.mark.gpu
def test_forwards_with_pdl_off_equal_pdl_on(tmp_path):
    from torch.profiler import ProfilerActivity, profile
    off = tmp_path / "pdl_off.pt"
    env = dict(os.environ, R3G_PDL="0")
    assert os.environ.get("R3G_PDL", "1")[:1] != "0", "this side of the comparison runs with PDL on"
    # the PDL-off process runs alongside this one
    r = subprocess.Popen([sys.executable, "-s", os.path.abspath(__file__), "--forwards", str(off)], env=env,
                         stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            first = forwards()
        second = forwards()
    finally:
        log, _ = r.communicate()
    assert r.returncode == 0, f"the R3G_PDL=0 run failed:\n{log}"
    reached = _pdl_kernels_in({e.name for e in prof.events() if e.device_type.name == "CUDA"})
    assert reached | NOT_REACHED_BY_FORWARDS == set(CONSUMERS) and not reached & NOT_REACHED_BY_FORWARDS, \
        f"PDL kernels reached: {sorted(reached)}"
    ref = torch.load(off)
    assert ref.keys() == first.keys() == second.keys()
    for k in first:
        assert torch.isfinite(first[k]).any(), k
        assert _same(first[k], second[k]), f"{k}: two PDL-on runs differ"
        assert _same(first[k], ref[k]), f"{k}: PDL on and R3G_PDL=0 differ"


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--forwards":
        torch.save(forwards(), sys.argv[2])
    else:
        sys.exit("usage: test_gpu_pdl_chains.py --forwards OUT.pt")
