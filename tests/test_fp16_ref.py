"""CPU: the float64 mirrors and the bound checker of oracle/fp16_ref.py (which the GPU kernel tests rely on) against
plain torch expressions of the same dtype flow, and the ops.py argument checks that refuse a call before any launch."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import fp16_ref as R


def _h(*shape, std=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * std).half()


def f16(t):
    return t.half().double()


# ------------------------------------------------------------------------------------------------- ulp16, check_bound
def test_ulp16_edges():
    cases = {0.0: 2 ** -24, 2 ** -24: 2 ** -24, 2 ** -14 - 2 ** -24: 2 ** -24, 2 ** -14: 2 ** -24, 1.0: 2 ** -10,
             1.999: 2 ** -10, 2.0: 2 ** -9, 2047.0: 1.0, 2048.0: 2.0, 32768.0: 32.0, 65504.0: 32.0, 1e6: 32.0}
    for x, u in cases.items():
        for s in (1.0, -1.0):
            assert R.ulp16(torch.tensor(s * x, dtype=torch.float64)).item() == u, (s * x, u)


def test_ulp16_matches_numpy_spacing_on_every_finite_fp16():
    bits = np.arange(0, 0x7bff, dtype=np.uint16)            # +0 up to the value below 65504
    v = bits.view(np.float16)
    got = R.ulp16(torch.from_numpy(v.astype(np.float64))).numpy()
    assert np.array_equal(got, np.spacing(v).astype(np.float64))


def test_check_bound_reports_the_worst_element():
    ref = torch.zeros(3, 4, dtype=torch.float64)
    bound = torch.full_like(ref, 0.1)
    got = ref.clone()
    got[1, 2] = 0.05
    assert R.check_bound(got, ref, bound, "ok") == pytest.approx(0.5)
    got[2, 3] = 0.3
    got[0, 0] = 0.2
    with pytest.raises(AssertionError, match=r"2 of 12 elements.*\(2, 3\).*err/bound 3"):
        R.check_bound(got, ref, bound, "two out")
    exact = torch.zeros_like(ref)
    assert R.check_bound(exact, ref, torch.zeros_like(ref), "bit exact") == 0.0
    nan = ref.clone()
    nan[0, 1] = float("nan")
    with pytest.raises(AssertionError, match="1 of 12"):
        R.check_bound(nan, ref, bound, "nan")


# ------------------------------------------------------------------------------------------------- mirrors
def test_linear_mirror_follows_the_documented_dtype_flow():
    M, N, K = 37, 64, 40
    x, w, b = _h(M, K, seed=1), _h(N, K, std=K ** -0.5, seed=2), _h(N, seed=3)
    lin = x.double() @ w.double().T + b.double()
    ref, bound = R.linear(x, w, b)
    assert torch.equal(ref, f16(lin))
    acc = R.wgmma_sum_bound(x, w)
    assert (bound <= R.ulp16(ref) + 2 * acc).all() and (bound > 0).any() and (bound == 0).any()
    R.check_bound(F.linear(x.float(), w.float(), b.float()).half(), ref, bound, "fp32 torch linear")
    ref, _ = R.linear(x, w, out_f32=True)
    assert torch.equal(ref, x.double() @ w.double().T)
    # activations on a column range, applied to the fp16-rounded Linear output
    for act, fn in ((1, lambda t: F.gelu(t, approximate="tanh")), (2, F.gelu), (3, F.relu)):
        ref, bound = R.linear(x, w, b, act=act, act_cols=(32, 64))
        pre = lin if act == 3 else f16(lin)
        assert torch.equal(ref[:, 32:], f16(fn(pre[:, 32:])))
        assert torch.equal(ref[:, :32], f16(lin[:, :32]))
    # gated fp16 residual: fp16(residual + fp16(gate * fp16(y)))
    res, gate = _h(M, N, seed=4), _h(3, N, seed=5)
    ref, bound = R.linear(x, w, b, gate=gate, gate_rows=13, residual=res)
    g = gate.double()[torch.arange(M) // 13]
    assert torch.equal(ref, f16(res.double() + f16(g * f16(lin))))
    y32 = F.linear(x.float(), w.float(), b.float()).half().float()
    R.check_bound((res.float() + (g.float() * y32).half().float()).half(), ref, bound, "gated residual")
    # fp32 residual stream: residual + ls_gamma * fp16(y), stored in float32
    r32 = torch.randn(M, N, generator=torch.Generator().manual_seed(6))
    gam = torch.rand(N, generator=torch.Generator().manual_seed(7))
    ref, bound = R.linear(x, w, b, residual=r32, ls_gamma=gam)
    assert torch.equal(ref, r32.double() + gam.double() * f16(lin))
    R.check_bound(r32 + gam * F.linear(x.float(), w.float(), b.float()).half().float(), ref, bound, "fp32 residual")


def test_linear_mirror_row_scale():
    M, N, K = 37, 64, 40
    x, w, b = _h(M, K, seed=1), _h(N, K, std=K ** -0.5, seed=2), _h(N, seed=3)
    s = torch.rand(M, generator=torch.Generator().manual_seed(4)).half()
    lin = x.double() @ w.double().T + b.double()
    for act, fn in ((0, lambda t: t), (2, F.gelu)):
        ref, bound = R.linear(x, w, b, act=act, row_scale=s)
        assert torch.equal(ref, f16(f16(fn(f16(lin))) * s.double()[:, None]))
        y = fn(F.linear(x.float(), w.float(), b.float()).half().float()).half()
        R.check_bound(y * s[:, None], ref, bound, f"row-scaled act={act}")


# ------------------------------------------------------------------------------------------------- MoE route / combine
def _route_logits_like_the_kernel(x, wg):
    """moe_route_kernel's logits in float32 torch: lane l adds its products x[8 l + 256 i + j] w[...] in (i, j) order
    (the products of fp16 values are exact, so fmaf is one rounded addition), then the xor-butterfly warp sum."""
    M, K = x.shape
    p = x.float()[:, None, :] * wg.float()[None, :, :]                 # [M, E, K], exact
    lanes = torch.zeros(M, wg.shape[0], 32)
    for k0 in range(0, K, 256):
        for j in range(8):
            cols = torch.arange(32) * 8 + k0 + j
            ok = cols < K
            lanes[..., ok] = lanes[..., ok] + p[..., cols[ok]]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[..., torch.arange(32) ^ o]
    return lanes[..., 0].half()


@pytest.mark.parametrize("K", [8, 1000, 1024])
def test_moe_logits_mirror(K):
    x, wg = _h(40, K, seed=K), _h(33, K, std=K ** -0.5, seed=K + 1)
    ref, bound = R.moe_logits(x, wg)
    assert torch.equal(ref, f16(x.double() @ wg.double().T))
    n = 8 * -(-K // 256) + 5
    assert (bound <= R.ulp16(ref) + 2 * n * 2.0 ** -24 * (x.double().abs() @ wg.double().abs().T)).all()
    R.check_bound(_route_logits_like_the_kernel(x, wg), ref, bound, f"kernel-order fp32 logits K={K}")
    R.check_bound((x.float() @ wg.float().T).half(), ref, bound, f"torch fp32 logits K={K}")


def _route_scores_like_the_kernel(logits):
    """moe_route_kernel's softmax in float32 torch: per-lane pairs (e, e + 32) added first, then the xor butterfly."""
    lg = logits.float()
    M, E = lg.shape
    ex = torch.exp(lg - lg.amax(dim=1, keepdim=True))
    pad = torch.zeros(M, 64)
    pad[:, :E] = ex
    s = pad[:, :32] + pad[:, 32:]
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, torch.arange(32) ^ o]
    return (ex * (1.0 / s[:, :1])).half()


def test_moe_scores_mirror():
    g = torch.Generator().manual_seed(5)
    lg = (torch.randn(400, 40, generator=g) * torch.rand(400, 1, generator=g) * 12).half()
    lg[0] = 0.0                                     # every score equal
    lg[1, 7] = 60.0                                 # the others underflow to fp16 0
    lg[2, :5] = -float("inf")                       # a logit of -inf: score 0
    lg[3, 3] = 65504.0
    lg[3, 4] = -65504.0                             # lg - mx is inexact in fp32
    sc = R.moe_scores(lg)
    p = torch.softmax(lg.double(), dim=1)
    assert torch.equal(sc.mid, f16(p))
    assert (sc.hi - sc.lo <= R.ulp16(sc.mid)).all() and (sc.hi > sc.lo).any()
    assert torch.equal(sc.mid[0], torch.full((40,), 0.025, dtype=torch.float64).half().double())
    assert (sc.hi[1, torch.arange(40) != 7] == 0).all() and (sc.lo[1, 7] == 1)
    assert (sc.hi[2, :5] == 0).all()
    for what, got in (("torch half softmax", torch.softmax(lg.float(), dim=1).half()),
                      ("kernel-order fp32 softmax", _route_scores_like_the_kernel(lg))):
        g64 = got.double()
        assert ((sc.lo <= g64) & (g64 <= sc.hi)).all(), what
    # where the k-th and (k+1)-th intervals are apart, the top k of the mirror is torch.topk's
    for k in (1, 2, 4):
        order = torch.sort(-sc.mid, dim=1, stable=True).indices
        kth = sc.lo.gather(1, order[:, k - 1:k])[:, 0]
        next_hi = sc.hi.gather(1, order[:, k:k + 1])[:, 0]
        clear = kth > next_hi
        assert clear.float().mean() > 0.5
        want = torch.topk(torch.softmax(lg.float(), dim=1), k, dim=1).indices
        assert torch.equal(order[clear, :k].sort(dim=1).values, want[clear].sort(dim=1).values)


def test_moe_combine_mirror_is_sequential_fp16_adds():
    M, N, K, E, k = 50, 24, 40, 5, 3
    x, w, b = _h(M, K, seed=1), _h(N, K, std=K ** -0.5, seed=2), _h(N, seed=3)
    g = torch.Generator().manual_seed(4)
    ids = torch.stack([torch.randperm(E, generator=g)[:k] for _ in range(M)]).int()
    cap = M + 3
    slots = (ids * cap + torch.randint(0, cap, (M, k), generator=g)).int()
    slot_y = _h(E * cap, N, std=2, seed=5)
    res = _h(M, N, std=4, seed=6)
    ref, bound = R.moe_combine(x, w, b, slot_y, ids, slots, res)
    shared = (x.double() @ w.double().T + b.double()).half()
    routed = torch.zeros(M, N, dtype=torch.float16)
    for r in range(M):
        for j in ids[r].long().argsort():
            routed[r] = routed[r] + slot_y[slots[r, j]]
    assert torch.equal(ref, (res + (routed + shared)).double())
    y32 = F.linear(x.float(), w.float(), b.float()).half()
    R.check_bound(res + (routed + y32), ref, bound, "fp32 torch shared expert")
    assert (bound == 0).float().mean() > 0.9 and (bound > 0).any()    # only near an fp16 rounding boundary


def test_wgmma_sum_bound_covers_a_truncating_blocked_sum():
    """A k16-blocked fp32 sum that truncates every addend to the block's largest exponent stays inside the bound."""
    x, w = _h(8, 96, seed=1), _h(8, 96, seed=2)
    bound = R.wgmma_sum_bound(x, w)
    exact = x.double() @ w.double().T
    acc = torch.zeros(8, 8, dtype=torch.float64)
    prods = x.double()[:, None, :] * w.double()[None, :, :]
    for k0 in range(0, 96, 16):
        terms = torch.cat([acc[..., None], prods[..., k0:k0 + 16]], dim=-1)
        e = torch.floor(torch.log2(terms.abs().amax(-1, keepdim=True).clamp_min(1e-300)))
        q = torch.exp2(e - 23)
        acc = R.f32((torch.trunc(terms / q) * q).sum(-1))
    assert ((acc - exact).abs() <= bound).all()


@pytest.mark.parametrize("Lq,Lk,scale", [(5, 1, None), (33, 200, None), (16, 300, 1.0)])
def test_attention_mirror_is_rounded_softmax(Lq, Lk, scale):
    q, k, v = _h(Lq, 64, seed=Lk), _h(Lk, 64, seed=Lk + 1), _h(Lk, 64, seed=Lk + 2)
    ref, bound = R.attention(q, k, v, scale)
    sc = 0.125 if scale is None else scale
    p = torch.softmax(q.double() @ k.double().T * sc, dim=-1)
    assert torch.equal(ref, f16(p @ v.double()))
    assert (bound > 0).all() and (bound <= 4 * R.ulp16(ref) + 1e-3).all()
    o32 = F.scaled_dot_product_attention(q.float()[None], k.float()[None], v.float()[None], scale=sc)[0]
    R.check_bound(o32.half(), ref, bound, "fp32 torch attention")
    if Lk == 1:
        assert torch.equal(ref, v.double().expand(Lq, 64))


def test_attention_mirror_row_chunks_agree():
    q, k, v = _h(70, 64, seed=1), _h(90, 64, seed=2), _h(90, 64, seed=3)
    a, b = R.attention(q, k, v), R.attention(q, k, v, row_chunk=16)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("b_out", [True, False])
def test_lnpost_dot_mirror(b_out):
    x = (3 + _h(9, 48, seed=1).float()).half()
    lw, lb = (1 + 0.1 * _h(48, seed=2).float()).half(), _h(48, std=0.1, seed=3)
    wo, bo = _h(1, 48, std=0.2, seed=4), (_h(1, seed=5) if b_out else None)
    ref, bound = R.lnpost_dot(x, lw, lb, wo, bo)
    h = f16(F.layer_norm(x.double(), (48,), lw.double(), lb.double(), 1e-5))
    want = f16(h @ wo.double().reshape(-1) + (bo.double() if b_out else 0.0))
    assert torch.equal(ref, want)
    assert ref.shape == (9,) and (bound <= 2 * R.ulp16(ref)).all()


def test_layernorm_f32in_mirror():
    x = torch.randn(6, 40, generator=torch.Generator().manual_seed(1)) * 2 + 1
    w, b = (1 + 0.1 * _h(40, seed=2).float()).half(), _h(40, std=0.1, seed=3)
    ref, bound = R.layernorm_f32in(x, w, b, eps=1e-6)
    assert torch.equal(ref, f16(F.layer_norm(x.double(), (40,), w.double(), b.double(), 1e-6)))
    assert (bound <= R.ulp16(ref)).all()
    R.check_bound(F.layer_norm(x, (40,), w.float(), b.float(), 1e-6).half(), ref, bound, "fp32 torch layer_norm")
    ref, _ = R.layernorm_f32in(x, eps=1e-6)
    assert torch.equal(ref, f16(F.layer_norm(x.double(), (40,), eps=1e-6)))


def test_swiglu_mirror():
    x = _h(20, 2 * 24 + 8, std=3, seed=1)
    x[0, :24] = 0.0
    x[1, :24] = -0.0
    x[2, :24] = -60000.0
    ref, bound = R.swiglu(x, 24)
    a, bb = x[:, :24].double(), x[:, 24:48].double()
    assert torch.equal(ref, f16(f16(F.silu(a)) * bb))
    assert ref.shape == (20, 24) and (ref[:3] == 0).all()
    flip = bound > 0           # only where the fp32 silu can cross an fp16 rounding boundary
    assert flip.float().mean() < 0.01


def test_patchify_mirror():
    img = torch.rand(2, 3, 4, 6, generator=torch.Generator().manual_seed(1))
    mean, std = (0.5, 0.4, 0.3), (0.2, 0.25, 0.3)
    out = R.patchify(img, 2, mean, std, out_ld=16)
    assert out.shape == (2 * 2 * 3, 16) and (out[:, 12:] == 0).all()
    for n in range(2):
        for py in range(2):
            for px in range(3):
                row = out[n * 6 + py * 3 + px]
                for c in range(3):
                    for dy in range(2):
                        for dx in range(2):
                            v = (img[n, c, 2 * py + dy, 2 * px + dx] - torch.tensor(mean[c])) / torch.tensor(std[c])
                            assert row[c * 4 + dy * 2 + dx] == v.half()


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("include_pi", [0, 1])
def test_points_fourier_mirror(include_pi, f32):
    q = torch.rand(7, 3, generator=torch.Generator().manual_seed(2)) * 2 - 1
    q = q if f32 else q.half()
    ref, bound = R.points_fourier(q, 3, include_pi, 24, f32_product=f32)
    x = q.double()
    cols = [f16(x)]
    e = []
    for d in range(3):
        for k in range(3):
            f = 2.0 ** k
            if include_pi:
                f = float(torch.tensor(f * math.pi, dtype=torch.float32).half())
            e.append(x[:, d] * f)
    e = torch.stack(e, 1)
    e = e.float().double() if f32 else f16(e)
    want = torch.cat(cols + [f16(torch.sin(e)), f16(torch.cos(e)), torch.zeros(7, 24 - 21, dtype=torch.float64)], 1)
    assert torch.equal(ref, want)
    assert (bound <= R.ulp16(ref)).all() and (bound[:, :3] == 0).all() and (bound[:, 21:] == 0).all()


# ------------------------------------------------------------------------------------------------- argument checks
@pytest.fixture
def ops(monkeypatch):
    from r3g import ops
    launched = []
    monkeypatch.setattr(ops, "_launch", lambda *a: launched.append(a))
    yield ops
    assert launched == []


def test_linear_refuses_a_stray_ls_gamma(ops):
    x, w = _h(4, 32), _h(64, 32)
    with pytest.raises(ValueError, match="ls_gamma"):
        ops.linear(x, w, ls_gamma=torch.ones(64))
    with pytest.raises(ValueError, match="ls_gamma"):
        ops.linear(x, w, residual=_h(4, 64), ls_gamma=torch.ones(64))


def test_lnpost_dot_and_swiglu_refuse_segmented_views(ops):
    buf = torch.zeros(3, 20, 64, dtype=torch.float16)
    ones = torch.ones(64, dtype=torch.float16)
    with pytest.raises(ValueError, match="rows"):
        ops.lnpost_dot(buf[:, 5:], ones, ones, ones, None, torch.zeros(45))
    with pytest.raises(ValueError, match="rows"):
        ops.swiglu(buf[:, 5:], 32)


def test_lnpost_dot_checks_dtypes_and_sizes(ops):
    x, ones = torch.zeros(5, 64, dtype=torch.float16), torch.ones(64, dtype=torch.float16)
    out = torch.zeros(5)
    with pytest.raises(TypeError, match="x must be float16"):
        ops.lnpost_dot(x.float(), ones, ones, ones, None, out)
    for i, name in enumerate(("ln_w", "ln_b", "w_out")):
        args = [ones, ones, ones]
        args[i] = ones.float()
        with pytest.raises(TypeError, match=name):
            ops.lnpost_dot(x, *args, None, out)
    with pytest.raises(TypeError, match="b_out"):
        ops.lnpost_dot(x, ones, ones, ones, torch.ones(1), out)
    with pytest.raises(ValueError, match="w_out must hold width = 64"):
        ops.lnpost_dot(x, ones, ones, torch.ones(1, 32, dtype=torch.float16), None, out)
