"""GPU: r3g_linear's outputs, bit for bit.  A restructured GEMM (a persistent grid, another staging scheme) must keep
every output element's k16 accumulation order and its epilogue arithmetic, so the outputs of the cases below must hash
to the digests in tests/golden/gemm_persistent.json, recorded with tools/make_gemm_golden.py from the one-tile-per-CTA
kernel of gemm.cu.  The cases cover the bounds shapes, every epilogue, grouped launches, segmented A, one k-block, K not
a multiple of 64, fewer tiles than SMs and 2 * 132 + 1 tiles (H100 SXM), and the MoE grouped and combine modes, whose
kernel shares linear_kernel's operand ring."""

import hashlib
import json
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gemm_persistent.json")
DEV = "cuda"


def _randn(*shape, std=1.0, seed=0, mean=0.0, dtype=torch.float16):
    g = torch.Generator().manual_seed(seed)           # CPU generator: the same inputs on every machine
    return (torch.randn(*shape, generator=g) * std + mean).to(dtype).to(DEV)


def _inputs(M, N, K, seed):
    return _randn(M, K, seed=seed), _randn(N, K, std=K ** -0.5, seed=seed + 1), _randn(N, seed=seed + 2)


BOUNDS_SHAPES = [
    (1, 32, 8), (1, 128, 1016), (1, 256, 72), (1, 288, 56), (1, 3104, 5120),
    (127, 96, 56), (127, 128, 64), (127, 256, 5120), (127, 288, 8),
    (128, 32, 56), (128, 96, 5120), (128, 160, 72), (128, 256, 1016), (128, 3104, 64),
    (129, 32, 5120), (129, 96, 8), (129, 160, 1016), (129, 288, 64),
    (257, 96, 1016), (257, 128, 56), (257, 160, 64), (257, 256, 5120), (257, 288, 8), (257, 3104, 72),
    (8884, 32, 72), (8884, 96, 56), (8884, 128, 5120), (8884, 160, 8), (8884, 256, 64), (8884, 288, 1016),
    (8884, 3104, 1016),
]
EPILOGUE_SHAPES = [(1000, 160, 256), (8884, 256, 200), (2740, 1024, 1024)]
EPILOGUES = ["no_bias", "bias", "gelu_tanh", "gelu_erf", "relu", "gate1", "gate17", "gate63", "gate64", "gate100",
             "gate333", "residual", "fp32_out", "residual_f32", "residual_f32_gamma"]


def _epilogue(ops, name, M, N, K, seed=11):
    x, w, b = _inputs(M, N, K, seed)
    if name == "no_bias":
        return ops.linear(x, w)
    if name == "bias":
        return ops.linear(x, w, b)
    if name in ("gelu_tanh", "gelu_erf", "relu"):
        act = {"gelu_tanh": ops.ACT_GELU_TANH, "gelu_erf": ops.ACT_GELU_ERF, "relu": 3}[name]
        return ops.linear(x, w, b, act=act, act_cols=(32, N - 32))
    if name.startswith("gate"):
        gr = int(name[4:])
        out = _randn(M, N, seed=seed + 3)
        ops.linear(x, w, b, gate=_randn(-(-M // gr), N, seed=seed + 4), gate_rows=gr, residual=out, out=out)
        return out
    if name == "residual":
        out = _randn(M, N, seed=seed + 3)
        ops.linear(x, w, b, residual=out, out=out)
        return out
    if name == "fp32_out":
        return ops.linear(x, w, b, out_dtype=torch.float32)
    if name.startswith("residual_f32"):
        out = _randn(M, N, std=4.0, seed=seed + 5, dtype=torch.float32)
        g = _randn(N, std=0.5, mean=1.0, seed=seed + 6, dtype=torch.float32) if name.endswith("gamma") else None
        ops.linear(x, w, b, residual=out, out=out, ls_gamma=g)
        return out
    raise KeyError(name)


def _qk_norm(ops, mode, M, N, K, heads_cols, act_cols, seed):
    x, w, b = _inputs(M, N, K, seed)
    nw = {s: _randn(64, std=0.1, mean=1.0, seed=seed + 10 + i) for i, s in enumerate(("q_w", "q_b", "k_w", "k_b"))}
    qk = dict(mode=mode, q_col0=0, k_col0=heads_cols, cols=heads_cols, eps=1e-6, q_w=nw["q_w"], k_w=nw["k_w"])
    if mode == ops.QKN_LAYERNORM:
        qk.update(q_b=nw["q_b"], k_b=nw["k_b"])
    kw = dict(act=ops.ACT_GELU_TANH, act_cols=act_cols) if act_cols else {}
    return ops.linear(x, w, b, qk_norm=qk, **kw)


def _segmented(ops, seg_len, N=288, K=136, S=3):
    x, w, b = _inputs(S * seg_len, N, K, seed=seg_len)
    xbuf = torch.full((S, seg_len + 5, K + 16), 77.0, device=DEV, dtype=torch.float16)
    xbuf[:, 5:, 8:8 + K] = x.view(S, seg_len, K)
    ybuf = _randn(S, seg_len + 3, N + 32, seed=seg_len + 9)
    yv = ybuf[:, 3:, 16:16 + N]
    ops.linear(xbuf[:, 5:, 8:8 + K], w, b, out=yv, residual=yv, gate=_randn(S, N, seed=seg_len + 10), gate_rows=seg_len)
    return ybuf


def _group(ops, n):
    x0, w0, b0 = _inputs(700, 256, 128, seed=1)
    x1, w1, b1 = _inputs(333, 256, 64, seed=2)
    x2, w2, _ = _inputs(1, 256, 72, seed=3)
    out1 = _randn(333, 256, seed=4)
    probs = [dict(x=x0, w=w0, bias=b0, act=ops.ACT_GELU_TANH),
             dict(x=x1, w=w1, bias=b1, gate=_randn(1, 256, seed=5), gate_rows=333, residual=out1, out=out1),
             dict(x=x2, w=w2, bias=None, out_dtype=torch.float32)][:n]
    return list(ops.linear_group(*probs))


def _moe_grouped(ops, act, scaled, G=5, cap=300, N=392, K=1000, seed=51):
    """4 routed experts with a full-capacity, an empty, a 129-row (partial last tile) and a 5-row segment, and a last
    group of cap rows; N = 392 ends in a partial column tile.  Rows past a segment's count keep out's initial values."""
    x, b = _randn(G * cap, K, seed=seed), _randn(G, N, seed=seed + 1)
    w = _randn(G, N, K, std=K ** -0.5, seed=seed + 2)
    counts = torch.tensor([cap, 0, 129, 5], dtype=torch.int32, device=DEV)
    out = _randn(G * cap, N, seed=seed + 3)
    rs = _randn(G * cap, std=0.2, mean=0.5, seed=seed + 4) if scaled else None
    return ops.moe_grouped(x, w, b, counts=counts, experts=4, out=out, act=act, row_scale=rs)


def _moe_combine(ops, M=1000, N=256, K=512, E=4, seed=61):
    """The shared expert's fc2 + the top-2 expert sum + the residual, in place; each row's two experts are distinct and
    in either order."""
    x, w, b = _inputs(M, N, K, seed)
    g = torch.Generator().manual_seed(seed + 3)
    e0 = torch.randint(0, E, (M,), generator=g)
    e1 = (e0 + torch.randint(1, E, (M,), generator=g)) % E
    ids = torch.stack([e0, e1], 1)
    slots = ids * M + torch.arange(M)[:, None]
    out = _randn(M, N, seed=seed + 4)
    ops.moe_combine(x, w, b, slot_y=_randn(E * M, N, std=0.5, seed=seed + 5), ids=ids.int().to(DEV),
                    slots=slots.int().to(DEV), residual=out, out=out)
    return out


def cases():
    """{name: zero-argument callable returning the output tensor(s)} of every case."""
    from r3g import ops
    c = {}
    for M, N, K in BOUNDS_SHAPES:
        c[f"bounds_{M}x{N}x{K}"] = lambda M=M, N=N, K=K: ops.linear(*_inputs(M, N, K, seed=M * 7 + N * 3 + K))
        c[f"bounds_{M}x{N}x{K}_f32"] = lambda M=M, N=N, K=K: ops.linear(
            *_inputs(M, N, K, seed=M * 7 + N * 3 + K)[:2], None, out_dtype=torch.float32)
    for M, N, K in EPILOGUE_SHAPES:
        for name in EPILOGUES:
            c[f"epilogue_{name}_{M}x{N}x{K}"] = lambda name=name, M=M, N=N, K=K: _epilogue(ops, name, M, N, K)
    # the DiT's fused projections: q/k norm on two head ranges, the single block's linear1 with GELU beside them
    c["qk_rms_2740x3072x1024"] = lambda: _qk_norm(ops, ops.QKN_RMS, 2740, 3072, 1024, 1024, None, 31)
    c["qk_ln_2740x3072x1024"] = lambda: _qk_norm(ops, ops.QKN_LAYERNORM, 2740, 3072, 1024, 1024, None, 32)
    c["qk_rms_gelu_1000x768x1024"] = lambda: _qk_norm(ops, ops.QKN_RMS, 1000, 768, 1024, 256, (512, 768), 33)
    c["qk_rms_gelu_1000x640x256"] = lambda: _qk_norm(ops, ops.QKN_RMS, 1000, 640, 256, 128, (256, 640), 34)
    for seg_len in (1, 127, 129):
        c[f"segmented_{seg_len}"] = lambda seg_len=seg_len: _segmented(ops, seg_len)
    c["group_2"] = lambda: _group(ops, 2)
    c["group_3"] = lambda: _group(ops, 3)
    # one k-block, K not a multiple of 64, and tile counts around the SM count of an H100 SXM (132)
    for M, N, K in [(4096, 1024, 64), (4096, 1024, 200), (4864, 1024, 1000), (300, 384, 256),
                    (265 * 128, 128, 192), (133 * 128, 256, 320), (132 * 128, 256, 1024), (8884, 7168, 1024)]:
        c[f"tiles_{M}x{N}x{K}_gelu_erf"] = lambda M=M, N=N, K=K: ops.linear(
            *_inputs(M, N, K, seed=M + N + K), act=ops.ACT_GELU_ERF)
    # the MoE modes (moe_gemm_kernel): grouped with and without erf-GELU and the row scale, and combine
    for act in ("none", "gelu_erf"):
        for scaled in (False, True):
            c[f"moe_grouped_{act}{'_scaled' if scaled else ''}"] = lambda act=act, scaled=scaled: _moe_grouped(
                ops, ops.ACT_GELU_ERF if act == "gelu_erf" else ops.ACT_NONE, scaled)
    c["moe_combine_top2"] = lambda: _moe_combine(ops)
    return c


def digest(out):
    outs = out if isinstance(out, (list, tuple)) else [out]
    h = hashlib.sha256()
    for t in outs:
        h.update(t.contiguous().view(torch.uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def test_linear_matches_the_one_tile_per_cta_kernel_bit_for_bit():
    with open(GOLDEN) as f:
        golden = json.load(f)
    c = cases()
    assert set(c) == set(golden), sorted(set(c) ^ set(golden))
    bad = [name for name, fn in c.items() if digest(fn()) != golden[name]]
    torch.cuda.synchronize()
    assert not bad, f"{len(bad)} of {len(c)} cases differ: {bad}"
