"""GPU: r3g_linear (with its MoE modes), r3g_attention and the row kernels against the float64 mirrors of
oracle/fp16_ref.py, element by element within the error bound its analysis gives (check_bound), at the shapes, strides
and epilogues where tiles, rings and masks change, plus the properties that hold bit for bit."""

import itertools

import pytest
import torch

import fp16_ref as R
from fp16_ref import check_bound

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _ops():
    from r3g import ops
    return ops


def _randn(*shape, std=1.0, seed=None, dtype=torch.float16):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return (torch.randn(*shape, generator=g, device=DEV) * std).to(dtype)


# ------------------------------------------------------------------------------------------------------ r3g_linear
def gemm_tile_n(problems, sms):
    """The output-tile width r3g_linear takes for a launch of `problems` ((M, N, seg_len) each) on `sms` SMs: 128 x 256
    tiles unless an N is below 256 or they leave more of the last wave idle than 128 x 128 tiles (end of gemm.cu)."""
    def tiles(tn):
        return sum((M // (s or M)) * -(-(s or M) // 128) * -(-N // tn) for M, N, s in problems)

    def eff(t, units):
        return t / (-(-t // units) * units)
    e256 = eff(tiles(256), sms) if min(N for _, N, _ in problems) >= 256 else 0.0
    return 256 if e256 > 0 and e256 >= eff(tiles(128), 2 * sms) else 128


LINEAR_SHAPES = [
    (1, 32, 8), (1, 128, 1016), (1, 256, 72), (1, 288, 56), (1, 3104, 5120),
    (127, 96, 56), (127, 128, 64), (127, 256, 5120), (127, 288, 8),
    (128, 32, 56), (128, 96, 5120), (128, 160, 72), (128, 256, 1016), (128, 3104, 64),
    (129, 32, 5120), (129, 96, 8), (129, 160, 1016), (129, 288, 64),
    (257, 96, 1016), (257, 128, 56), (257, 160, 64), (257, 256, 5120), (257, 288, 8), (257, 3104, 72),
    (8884, 32, 72), (8884, 96, 56), (8884, 128, 5120), (8884, 160, 8), (8884, 256, 64), (8884, 288, 1016),
    (8884, 3104, 1016),
]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def test_linear_shapes_reach_both_tile_widths():
    widths = {gemm_tile_n([(M, N, 0)], _sms()) for M, N, _ in LINEAR_SHAPES}
    assert widths == {128, 256}, widths


def _gemm_inputs(M, N, K, seed):
    x = _randn(M, K, seed=seed)
    w = _randn(N, K, std=K ** -0.5, seed=seed + 1)
    b = _randn(N, seed=seed + 2)
    return x, w, b


@pytest.mark.parametrize("M,N,K", LINEAR_SHAPES)
def test_linear_shapes(M, N, K):
    ops = _ops()
    x, w, b = _gemm_inputs(M, N, K, seed=M * 7 + N * 3 + K)
    what = f"linear {M}x{N}x{K} (BN={gemm_tile_n([(M, N, 0)], _sms())})"
    check_bound(ops.linear(x, w, b), *R.linear(x, w, b), what)
    check_bound(ops.linear(x, w, None, out_dtype=torch.float32), *R.linear(x, w, out_f32=True), what + " fp32 out")


def _epilogue_case(name, M, N, K, seed=11):
    """(linear kwargs, mirror kwargs, out tensor given or None) of one epilogue of the table."""
    x, w, b = _gemm_inputs(M, N, K, seed)
    res = _randn(M, N, seed=seed + 3)
    kw, ref = dict(), dict()
    if name == "no_bias":
        return x, w, None, kw, ref
    if name in ("gelu_tanh", "gelu_erf", "relu"):
        act = {"gelu_tanh": 1, "gelu_erf": 2, "relu": 3}[name]
        kw = dict(act=act, act_cols=(32, 96))
        return x, w, b, kw, dict(kw)
    if name.startswith("gate"):
        gr = int(name[4:])
        gate = _randn(-(-M // gr), N, seed=seed + 4)
        out = res.clone()
        kw = dict(gate=gate, gate_rows=gr, residual=out, out=out)
        return x, w, b, kw, dict(gate=gate, gate_rows=gr, residual=res)
    if name == "residual_alias":
        out = res.clone()
        return x, w, b, dict(residual=out, out=out), dict(residual=res)
    if name == "fp32_out":
        return x, w, b, dict(out_dtype=torch.float32), dict(out_f32=True)
    if name.startswith("residual_f32"):
        r32 = _randn(M, N, seed=seed + 5, dtype=torch.float32) * 4
        g = (1 + _randn(N, std=0.5, seed=seed + 6, dtype=torch.float32)) if name.endswith("gamma") else None
        out = r32.clone()
        return x, w, b, dict(residual=out, out=out, ls_gamma=g), dict(residual=r32, ls_gamma=g)
    raise KeyError(name)


EPILOGUES = ["no_bias", "gelu_tanh", "gelu_erf", "relu", "gate1", "gate17", "gate63", "gate64", "gate100", "gate333",
             "residual_alias", "fp32_out", "residual_f32", "residual_f32_gamma"]


@pytest.mark.parametrize("M,N,K", [(1000, 160, 256), (8884, 256, 200)])
@pytest.mark.parametrize("name", EPILOGUES)
def test_linear_epilogue_table(name, M, N, K):
    ops = _ops()
    x, w, b, kw, ref_kw = _epilogue_case(name, M, N, K)
    y = ops.linear(x, w, b, **kw)
    check_bound(y, *R.linear(x, w, b, **ref_kw), f"linear {name} {M}x{N}x{K} (BN={gemm_tile_n([(M, N, 0)], _sms())})")


@pytest.mark.parametrize("seg_len", [1, 127, 129])
def test_linear_segmented_strided_views(seg_len):
    """3 segments of seg_len rows read from a strided [S, L, K] view and written, with a per-segment gate and the
    output as residual, into a strided [S, L, N] view of a wider buffer; everything outside the view stays."""
    ops = _ops()
    S, K, N = 3, 136, 288
    x, w, b = _gemm_inputs(S * seg_len, N, K, seed=seg_len)
    xbuf = torch.full((S, seg_len + 5, K + 16), 77.0, device=DEV, dtype=torch.float16)
    xbuf[:, 5:, 8:8 + K] = x.view(S, seg_len, K)
    ybuf = _randn(S, seg_len + 3, N + 32, seed=seg_len + 9)
    before = ybuf.clone()
    yv = ybuf[:, 3:, 16:16 + N]
    res = yv.reshape(-1, N).clone()
    gate = _randn(S, N, seed=seg_len + 10)
    ops.linear(xbuf[:, 5:, 8:8 + K], w, b, out=yv, residual=yv, gate=gate, gate_rows=seg_len)
    check_bound(yv.reshape(-1, N), *R.linear(x, w, b, gate=gate, gate_rows=seg_len, residual=res),
                f"segmented seg_len={seg_len}")
    mask = torch.ones_like(ybuf, dtype=torch.bool)
    mask[:, 3:, 16:16 + N] = False
    assert torch.equal(ybuf[mask], before[mask])


def test_linear_group_of_three_epilogues():
    ops = _ops()
    x0, w0, b0 = _gemm_inputs(700, 256, 128, seed=1)
    x1, w1, b1 = _gemm_inputs(333, 256, 64, seed=2)
    x2, w2, b2 = _gemm_inputs(1, 256, 72, seed=3)
    r1 = _randn(333, 256, seed=4)
    g1 = _randn(1, 256, seed=5)
    out1 = r1.clone()
    y0, y1, y2 = ops.linear_group(dict(x=x0, w=w0, bias=b0, act=ops.ACT_GELU_TANH),
                                  dict(x=x1, w=w1, bias=b1, gate=g1, gate_rows=333, residual=out1, out=out1),
                                  dict(x=x2, w=w2, bias=None, out_dtype=torch.float32))
    check_bound(y0, *R.linear(x0, w0, b0, act=1), "group problem 0 (tanh-GELU)")
    check_bound(y1, *R.linear(x1, w1, b1, gate=g1, gate_rows=333, residual=r1), "group problem 1 (gated residual)")
    check_bound(y2, *R.linear(x2, w2, out_f32=True), "group problem 2 (fp32 out)")


@pytest.mark.parametrize("M,N,K", [(8884, 288, 64), (300, 3104, 1016)])
def test_linear_row_permutation_is_bit_exact(M, N, K):
    ops = _ops()
    x, w, b = _gemm_inputs(M, N, K, seed=21)
    perm = torch.randperm(M, generator=torch.Generator().manual_seed(3)).to(DEV)
    y = ops.linear(x, w, b, act=ops.ACT_GELU_ERF)
    yp = ops.linear(x[perm].contiguous(), w, b, act=ops.ACT_GELU_ERF)
    assert torch.equal(yp, y[perm])


def test_linear_refuses_gate_with_fp32_residual():
    ops = _ops()
    from r3g import _abi
    x, w, b = _gemm_inputs(64, 64, 64, seed=1)
    out = torch.zeros(64, 64, device=DEV)
    with pytest.raises(_abi.R3GError, match="gate"):
        ops.linear(x, w, b, gate=_randn(1, 64, seed=2), gate_rows=64, residual=out, out=out)
    torch.cuda.synchronize()
    assert not out.any()


# ------------------------------------------------------------------------------------------------------ r3g_attention
def check_attention(o, q, k, v, scale, what):
    """check_bound of every (b, h) of o [B, Lq, H, 64] against fp16_ref.attention; returns the largest ratio."""
    worst = 0.0
    for bi in range(q.shape[0]):
        for h in range(q.shape[2]):
            ref, bound = R.attention(q[bi, :, h], k[bi, :, h], v[bi, :, h], scale)
            worst = max(worst, check_bound(o[bi, :, h], ref, bound, f"{what} b={bi} h={h}"))
    return worst


def _strided_qkv(B, H, Lq, Lk, seed, q_std=1.0, k_std=1.0):
    """q a slice of a packed [B, Lq, 3, H, 64] buffer, k stored [B, H, Lk, 64], v [B, Lk, H, 72] cut to 64, and o a
    view into a wider [B, Lq, H, 80] buffer: four different stride patterns."""
    q = _randn(B, Lq, 3, H, 64, std=q_std, seed=seed)[:, :, 1]
    k = _randn(B, H, Lk, 64, std=k_std, seed=seed + 1).transpose(1, 2)
    v = _randn(B, Lk, H, 72, seed=seed + 2)[..., :64]
    obuf = torch.full((B, Lq, H, 80), 5.0, device=DEV, dtype=torch.float16)
    return q, k, v, obuf


ATTN_SHAPES = [(1, 1), (63, 127), (64, 128), (65, 129), (191, 383), (192, 384), (193, 385), (1, 8193), (193, 8193),
               (4442, 129), (65, 4442), (4442, 4442), (192, 1), (1, 385)]


@pytest.mark.parametrize("Lq,Lk", ATTN_SHAPES)
def test_attention_shapes_and_strides(Lq, Lk):
    ops = _ops()
    B, H = (2, 2) if Lq * Lk < 10 ** 6 else (1, 2)
    q, k, v, obuf = _strided_qkv(B, H, Lq, Lk, seed=Lq + Lk)
    o = obuf[..., 8:72]
    ops.attention(q, k, v, out=o)
    check_attention(o, q, k, v, None, f"attention Lq={Lq} Lk={Lk}")
    assert (obuf[..., :8] == 5).all() and (obuf[..., 72:] == 5).all()


@pytest.mark.parametrize("scale", [0.05, 1.0])
def test_attention_scales(scale):
    ops = _ops()
    q, k, v, _ = _strided_qkv(1, 2, 385, 1000, seed=3)
    check_attention(ops.attention(q, k, v, scale=scale), q, k, v, scale, f"attention scale={scale}")


def _tile_mass_v(Lk, H):
    j = torch.arange(Lk, device=DEV)
    v = ((j // 128) % 64)[:, None] == torch.arange(64, device=DEV)[None, :]
    return v.to(torch.float16)[None, :, None, :].expand(1, Lk, H, 64).contiguous()


@pytest.mark.parametrize("Lq,Lk", [(193, 4442), (64, 8193), (4442, 4442)])
def test_attention_tile_mass(Lq, Lk):
    """v[j, d] = (tile of key j mod 64 == d): o[:, d] is the softmax mass of key tile d (and d + 64), so a dropped,
    stale or mis-weighted tile, or P carried at less than fp16 precision, moves a whole column coherently."""
    ops = _ops()
    q = _randn(1, Lq, 2, 64, seed=Lk)
    k = _randn(1, Lk, 2, 64, seed=Lk + 1)
    v = _tile_mass_v(Lk, 2)
    o = ops.attention(q, k, v)
    check_attention(o, q, k, v, None, f"tile mass Lq={Lq} Lk={Lk}")


def test_attention_rising_max():
    """Every key tile holds larger logits than the one before, for every query: the running max and the alpha rescale
    change at every tile."""
    ops = _ops()
    Lq, Lk = 300, 4442
    u = _randn(64, seed=1, dtype=torch.float32)
    q = (u + 0.1 * _randn(1, Lq, 1, 64, seed=2, dtype=torch.float32)).half()
    t = (torch.arange(Lk, device=DEV) // 128).float()
    k = (0.05 * t[:, None] * u + 0.05 * _randn(Lk, 64, seed=3, dtype=torch.float32)).half()[None, :, None, :]
    v = _randn(1, Lk, 1, 64, seed=4)
    s = (q[0, :, 0].float() @ k[0, :, 0].float().T)[:, :34 * 128].view(Lq, 34, 128).amax(-1)
    assert (s[:, 1:] > s[:, :-1]).all()
    check_attention(ops.attention(q, k, v), q, k, v, None, "rising max")


def test_attention_large_logits():
    """|scale * s| up to about 80: most exponentials underflow (fp16 and fp32 subnormals, ex2 flush)."""
    ops = _ops()
    q = _randn(1, 500, 2, 64, std=1.3, seed=5)
    k = _randn(1, 3000, 2, 64, std=1.3, seed=6)
    v = _randn(1, 3000, 2, 64, seed=7)
    s = q[0, :, 0].float() @ k[0, :, 0].float().T
    assert s.abs().max() > 60
    check_attention(ops.attention(q, k, v, scale=1.0), q, k, v, 1.0, "large logits")


def test_attention_bit_exact_properties():
    ops = _ops()
    # one key: o == v
    q = _randn(2, 300, 3, 64, seed=1)
    k = _randn(2, 1, 3, 64, seed=2)
    v = _randn(2, 1, 3, 64, seed=3)
    assert torch.equal(ops.attention(q, k, v), v.expand(2, 300, 3, 64))
    # identical keys and values: P = 1 and the fp32 sum Lk * v is exact
    for Lk in (4442, 8192):
        k = _randn(1, 1, 2, 64, seed=Lk).expand(1, Lk, 2, 64).contiguous()
        v = _randn(1, 1, 2, 64, seed=Lk + 1).expand(1, Lk, 2, 64).contiguous()
        assert torch.equal(ops.attention(q[:1, :, :2], k, v), v[:, :1].expand(1, 300, 2, 64)), Lk
    # permuted query rows give permuted output rows
    q, k, v, _ = _strided_qkv(2, 3, 1000, 777, seed=9)
    o = ops.attention(q, k, v)
    perm = torch.randperm(1000, generator=torch.Generator().manual_seed(1)).to(DEV)
    assert torch.equal(ops.attention(q[:, perm], k, v), o[:, perm])
    # a (B, H) launch equals the per-(b, h) launches
    for bi in range(2):
        for h in range(3):
            oh = ops.attention(q[bi:bi + 1, :, h:h + 1], k[bi:bi + 1, :, h:h + 1], v[bi:bi + 1, :, h:h + 1])
            assert torch.equal(oh[0, :, 0], o[bi, :, h]), (bi, h)


@pytest.mark.parametrize("windows", [
    [(13, 100, 1), (0, 1, 1)],          # row0 not a multiple of 8; a window of one row
    [(40, 200, 1), (5, 200, 1)],        # 200 rows: two 192-row tiles, ending inside the last 64-row group
    [(30, 150, 7), (9, 1, 4)],          # k0_count > 1: copies of the first key, checked over explicit duplicates
])
def test_attention_windows(windows):
    ops = _ops()
    B, H, L = 2, 2, 517
    q = _randn(B, L, H, 64, seed=31)
    k = _randn(B, L, H, 64, seed=32)
    v = _randn(B, L, H, 64, seed=33)
    kd, vd = k.clone(), v.clone()
    for bi, (r0, n, cnt) in enumerate(windows):
        kd[bi, r0 - cnt + 1:r0] = k[bi, r0]
        vd[bi, r0 - cnt + 1:r0] = v[bi, r0]
    o = torch.full_like(q, 3.0)
    ops.attention(q, k, v, out=o, windows=windows)
    assert torch.equal(k, kd) and torch.equal(v, vd)     # the documented in-place key copies, nothing else
    for bi, (r0, n, cnt) in enumerate(windows):
        for h in range(H):
            ref, bound = R.attention(q[bi, r0:r0 + n, h], kd[bi, :, h], vd[bi, :, h])
            check_bound(o[bi, r0:r0 + n, h], ref, bound, f"window {bi} {(r0, n, cnt)} h={h}")
        outside = torch.ones(L, dtype=torch.bool, device=DEV)
        outside[r0:r0 + n] = False
        assert (o[bi, outside] == 3).all()


# ------------------------------------------------------------------------------------------------------ row kernels
@pytest.mark.parametrize("width,rows,offset", [(64, 7, 0.0), (1024, 100003, 0.0), (1032, 7, 0.0), (1032, 100003, 0.0),
                                               (2048, 1, 0.0), (1024, 1000, 50.0), (2048, 333, 200.0)])
@pytest.mark.parametrize("with_b_out", [True, False])
def test_lnpost_dot(width, rows, offset, with_b_out):
    ops = _ops()
    seed = width + rows
    xbuf = (offset + _randn(rows, width + 64, seed=seed, dtype=torch.float32)).half()
    x = xbuf[:, :width]                                   # ldx > width
    ln_w = (1 + _randn(width, std=0.1, seed=seed + 1, dtype=torch.float32)).half()
    ln_b = _randn(width, std=0.1, seed=seed + 2)
    w_out = _randn(1, width, std=width ** -0.5, seed=seed + 3)
    b_out = _randn(1, std=0.1, seed=seed + 4) if with_b_out else None
    out = torch.full((rows,), float("nan"), device=DEV)
    ops.lnpost_dot(x, ln_w, ln_b, w_out, b_out, out)
    ref, bound = R.lnpost_dot(x, ln_w, ln_b, w_out, b_out)
    check_bound(out, ref, bound, f"lnpost_dot width={width} rows={rows} offset={offset}")
    sure = ref.abs() > bound
    assert torch.equal(torch.sign(out.double())[sure], torch.sign(ref)[sure])


@pytest.mark.parametrize("width", [8, 1000, 2048])
@pytest.mark.parametrize("affine", [True, False])
@pytest.mark.parametrize("rows_kind", ["normal", "offset"])
def test_layernorm_f32in(width, affine, rows_kind):
    """rows_kind 'offset': rows 1000 + 0.01 N(0, 1), where E[x^2] - mean^2 in fp32 loses every digit of the variance."""
    ops = _ops()
    rows = 777
    z = _randn(rows, width, seed=width, dtype=torch.float32)
    x = 1000 + 0.01 * z if rows_kind == "offset" else 3 * z - 1
    w = (1 + _randn(width, std=0.2, seed=width + 1, dtype=torch.float32)).half() if affine else None
    b = _randn(width, std=0.2, seed=width + 2) if affine else None
    y = ops.layernorm_f32in(x, w, b, eps=1e-6)
    check_bound(y, *R.layernorm_f32in(x, w, b, eps=1e-6), f"layernorm_f32in width={width} {rows_kind}")


@pytest.mark.parametrize("F", [8, 344])
def test_swiglu(F):
    ops = _ops()
    rows = 1000
    xbuf = _randn(rows, 2 * F + 24, std=3.0, seed=F)
    a = xbuf[:, :F]
    a[0::7] = 0.0
    a[1::7] = -0.0
    a[2::7] = -a[2::7].abs() * 30                        # large negative: silu underflows to (-)0
    a[3::7, :4] = -65504.0
    x = xbuf[:, :2 * F]                                   # ldx > 2F
    obuf = torch.full((rows, F + 16), 9.0, device=DEV, dtype=torch.float16)
    out = obuf[:, :F]                                     # ldo > F
    ops.swiglu(x, F, out=out)
    ref, bound = R.swiglu(x, F)
    check_bound(out, ref, bound, f"swiglu F={F}")
    assert (obuf[:, F:] == 9).all()


@pytest.mark.parametrize("N,H,W,patch,out_ld", [(2, 28, 42, 14, 592), (3, 5, 7, 1, None)])
def test_patchify_bit_exact(N, H, W, patch, out_ld):
    ops = _ops()
    img = _randn(N, 3, H, W, seed=H * W, dtype=torch.float32) * 0.3 + 0.5
    mean, std = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
    got = ops.patchify(img, patch, mean=mean, std=std, out_ld=out_ld)
    ref = R.patchify(img, patch, mean, std, out_ld)
    assert got.shape == ref.shape and torch.equal(got, ref)


@pytest.mark.parametrize("f32", [False, True])
@pytest.mark.parametrize("include_pi", [0, 1])
@pytest.mark.parametrize("path", ["fast", "generic_F6", "generic_misaligned"])
def test_points_fourier(path, include_pi, f32):
    ops = _ops()
    n = 3001
    F, out_ld = (6, 40) if path == "generic_F6" else (8, 64)
    q = _randn(n, 3, std=0.6, seed=F + include_pi, dtype=torch.float32)
    q = q if f32 else q.half()
    buf = torch.full((n * out_ld + 4,), float("nan"), device=DEV, dtype=torch.float16)
    off = 4 if path == "generic_misaligned" else 0          # 8 bytes past 16-byte alignment
    out = buf[off:off + n * out_ld].view(n, out_ld)
    (ops.points_fourier_f32 if f32 else ops.points_fourier)(q, out, F, include_pi)
    ref, bound = R.points_fourier(q, F, include_pi, out_ld, f32_product=f32)
    check_bound(out, ref, bound, f"points_fourier {path} pi={include_pi} f32={f32}")
    assert (bound <= R.ulp16(ref)).all()
    assert (out[:, 3 + 6 * F:] == 0).all()


# ------------------------------------------------------------------------------------------------------ r3g_linear MoE
GUARD16 = -4320.0     # fp16 guard fill of the MoE output buffers (exact in fp16)
GUARD32 = -7          # int32 guard fill of ids / slots; counts past E are zero, see _route_bufs


def _bits(t):
    """fp16 as int16, so that NaNs compare by their bits."""
    return t.view(torch.int16) if t.dtype == torch.float16 else t


def _route_bufs(M, E, k, K, cap):
    """moe_route's output buffers as leading views of larger guard-filled ones.  The larger ones hold one spare
    segment of cap rows past slot_x / slot_scale's E * cap, 64 spare entries past ids / weights / slots, and 8 zeroed
    counters past counts: a kernel that routed a row to expert E would count it from 0 and write inside the spare
    segment, where the guards show it, instead of outside the allocation."""
    i32 = dict(device=DEV, dtype=torch.int32)
    h = dict(device=DEV, dtype=torch.float16)
    big = dict(counts=torch.zeros(E + 8, **i32), ids=torch.full((M * k + 64,), GUARD32, **i32),
               weights=torch.full((M * k + 64,), GUARD16, **h), slots=torch.full((M * k + 64,), GUARD32, **i32),
               slot_x=torch.full(((E + 1) * cap, K), GUARD16, **h),
               slot_scale=torch.full(((E + 1) * cap,), GUARD16, **h))
    views = dict(counts=big["counts"][:E], ids=big["ids"][:M * k].view(M, k), weights=big["weights"][:M * k].view(M, k),
                 slots=big["slots"][:M * k].view(M, k), slot_x=big["slot_x"][:E * cap],
                 slot_scale=big["slot_scale"][:E * cap])
    return big, views


def _route(x, wg, k, cap):
    """One route launch; the logits go to columns [2, 2 + E) of a guard-filled [M, E + 5] buffer."""
    M, K = x.shape
    E = wg.shape[0]
    big, v = _route_bufs(M, E, k, K, cap)
    lbuf = torch.full((M, E + 5), GUARD16, device=DEV, dtype=torch.float16)
    logits = _ops().moe_route(x, wg, top_k=k, cap=cap, out=lbuf[:, 2:2 + E], **v)
    return logits, lbuf, big, v


def _check_route_layout(x, E, k, cap, lbuf, big, v):
    """What holds whatever the scores: ids in [0, E) and distinct in a row, counts their bincount, slots in the id's
    segment at positions 0 .. count - 1 (a permutation), the slot rows copies of x with the weights as their scale, and
    every byte the route must not write still holding its guard."""
    M, K = x.shape
    ids, slots = v["ids"].long(), v["slots"].long()
    assert ((ids >= 0) & (ids < E)).all(), "expert id out of range"
    assert (ids.sort(dim=1).values.diff(dim=1) > 0).all(), "an expert taken twice in a row"
    counts = torch.bincount(ids.flatten(), minlength=E)
    assert torch.equal(v["counts"].long(), counts)
    assert torch.equal(slots // cap, ids)
    s = slots.flatten().sort().values
    start = torch.cumsum(counts, 0) - counts
    assert torch.equal(s % cap, torch.arange(M * k, device=DEV) - start[s // cap]), "segment positions"
    assert torch.equal(_bits(v["slot_x"][slots]), _bits(x)[:, None, :].expand(M, k, K))
    assert torch.equal(_bits(v["slot_scale"][slots]), _bits(v["weights"]))
    used = torch.zeros((E + 1) * cap, dtype=torch.bool, device=DEV)
    used[slots.flatten()] = True
    assert (big["slot_x"] == GUARD16).all(dim=1)[~used].all() and (big["slot_scale"][~used] == GUARD16).all()
    assert (big["counts"][E:] == 0).all()
    assert (big["ids"][M * k:] == GUARD32).all() and (big["slots"][M * k:] == GUARD32).all()
    assert (big["weights"][M * k:] == GUARD16).all()
    assert (lbuf[:, :2] == GUARD16).all() and (lbuf[:, 2 + E:] == GUARD16).all()


def _check_route_picks(logits, v, rows, what):
    """On `rows`, against the score intervals of the kernel's own logits: every weight in its expert's interval, no
    chosen interval wholly below an unchosen one, and the picks in the kernel's order (non-increasing weights, equal
    weights lower expert first)."""
    sc = R.moe_scores(logits[rows])
    ids, w = v["ids"][rows].long(), v["weights"][rows].double()
    assert ((sc.lo.gather(1, ids) <= w) & (w <= sc.hi.gather(1, ids))).all(), f"{what}: weight outside its interval"
    chosen = torch.zeros_like(sc.lo, dtype=torch.bool).scatter_(1, ids, True)
    lowest_chosen = torch.where(chosen, sc.hi, torch.full_like(sc.hi, float("inf"))).amin(dim=1)
    best_unchosen = torch.where(chosen, torch.full_like(sc.lo, -float("inf")), sc.lo).amax(dim=1)
    assert (lowest_chosen >= best_unchosen).all(), f"{what}: an expert chosen over a surely higher one"
    assert (w[:, 1:] <= w[:, :-1]).all(), f"{what}: picks out of order"
    tie = w[:, 1:] == w[:, :-1]
    assert (ids[:, 1:] > ids[:, :-1])[tie].all(), f"{what}: equal scores not lower expert first"


ROUTE_EK = [(1, 1), (8, 2), (4, 4), (33, 3), (64, 4)]


@pytest.mark.parametrize("layout", ["cap_M", "cap_M37_strided_x"])
@pytest.mark.parametrize("M", [1, 7, 8884])
@pytest.mark.parametrize("K", [8, 1000, 1024])
@pytest.mark.parametrize("E,k", ROUTE_EK)
def test_moe_route(E, k, K, M, layout):
    """E = 64 fills both score registers of every lane, E = 33 one lane's second register, E = 1 leaves 31 lanes idle;
    K = 8 and 1000 leave lanes idle in the last 256-column pass of the gate dot products."""
    seed = E * 7 + K + M
    strided = layout != "cap_M"
    cap = M + 37 if strided else M
    x = _randn(M, K + 24, seed=seed)[:, 8:8 + K] if strided else _randn(M, K, seed=seed)
    wg = _randn(E, K, std=2 * K ** -0.5, seed=seed + 1)
    logits, lbuf, big, v = _route(x, wg, k, cap)
    what = f"route E={E} k={k} K={K} M={M} {layout}"
    check_bound(logits, *R.moe_logits(x, wg), what + " logits")
    _check_route_picks(logits, v, slice(None), what)
    _check_route_layout(x, E, k, cap, lbuf, big, v)


@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_moe_route_ties_go_to_the_lower_expert(k):
    """Three pairs of identical gate rows, which dominate the others: across lanes (0 / 1), across one lane's two
    registers (3 / 35) and across the register boundary (31 / 32).  Their logits are bit-identical, so is every score;
    the lower expert of a pair comes first, and an odd k takes the lower one alone."""
    E, K, M = 64, 1000, 3000
    x = _randn(M, K, seed=k)
    wg = _randn(E, K, std=0.1 * K ** -0.5, seed=k + 1)
    strong = _randn(3, K, std=3 * K ** -0.5, seed=k + 2)
    pairs = [(0, 1), (3, 35), (31, 32)]
    for i, (a, b) in enumerate(pairs):
        wg[a] = strong[i]
        wg[b] = strong[i]
    logits, lbuf, big, v = _route(x, wg, k, M)
    check_bound(logits, *R.moe_logits(x, wg), f"ties k={k} logits")
    _check_route_picks(logits, v, slice(None), f"ties k={k}")
    _check_route_layout(x, E, k, M, lbuf, big, v)
    ids = v["ids"].long()

    def pos(e):     # expert e's pick position in each row, k where it is not picked
        hit = ids == e
        return torch.where(hit.any(dim=1), hit.int().argmax(dim=1), torch.full_like(ids[:, 0], k))
    for a, b in pairs:
        assert torch.equal(_bits(logits[:, a]), _bits(logits[:, b]))
        pa, pb = pos(a), pos(b)
        assert (pa < k).any(), (a, b)          # the pair is chosen on some rows
        assert (pa < pb)[pb < k].all(), f"expert {b} taken before or without its twin {a}"


@pytest.mark.parametrize("kind", ["all_equal", "underflow"])
@pytest.mark.parametrize("E,k", ROUTE_EK)
def test_moe_route_exact_orders(E, k, kind):
    """all_equal: one gate row for every expert, so every score ties: ids 0 .. k-1.  underflow: expert `hot` leads by
    about 64, every other score rounds to fp16 0 (and ties at 0): hot, then the lowest other experts."""
    M, K = 777, 1000
    hot = E - 1 - E // 3
    x = _randn(M, K, seed=E + k)
    if kind == "all_equal":
        wg = _randn(1, K, std=K ** -0.5, seed=E).expand(E, K).contiguous()
        want = list(range(k))
    else:
        x[:, :8] = 4.0
        wg = _randn(E, K, std=K ** -0.5, seed=E)
        wg[:, :8] = 0.0
        wg[hot, :8] = 2.0
        want = [hot] + [e for e in range(E) if e != hot][:k - 1]
    logits, lbuf, big, v = _route(x, wg, k, M)
    check_bound(logits, *R.moe_logits(x, wg), f"{kind} E={E} k={k} logits")
    _check_route_picks(logits, v, slice(None), f"{kind} E={E} k={k}")
    _check_route_layout(x, E, k, M, lbuf, big, v)
    assert torch.equal(v["ids"].long(), torch.tensor(want, device=DEV).expand(M, k))
    if kind == "underflow" and k > 1:
        assert (v["weights"][:, 1:] == 0).all() and (v["weights"][:, 0] == 1).all()


@pytest.mark.parametrize("E,k", [(1, 1), (8, 2), (33, 3), (64, 4)])
def test_moe_route_nonfinite_rows(E, k):
    """Rows with a NaN in x (in the first and in the last 256-column pass), a logit that rounds to +inf and one that
    rounds to -inf, among finite rows of one launch.  The NaN and +inf rows have only NaN scores: experts 0 .. k-1 with
    NaN weights (NaN ranks above every number, lower expert first).  The -inf expert's score is 0 (for E = 1 every
    logit is -inf and the row is a NaN row).  The finite rows route as in a launch without the others.  Every output is
    a leading view of a guard-filled buffer sized so that a route to expert E stays inside it and shows."""
    M, K = 300, 1000
    cap = M + 37
    hot = E // 2
    x = _randn(M, K, seed=E)
    x[:, :8] = 0.0
    wg = _randn(E, K, std=2 * K ** -0.5, seed=E + 1)
    wg[hot, :8] = 1000.0
    x[5, 3] = float("nan")
    x[150, 999] = float("nan")
    x[77, :8] = 10.0                 # logit of `hot` 80000 -> +inf
    x[231, :8] = -10.0               # -80000 -> -inf
    bad = [5, 77, 150, 231]
    logits, lbuf, big, v = _route(x, wg, k, cap)
    _check_route_layout(x, E, k, cap, lbuf, big, v)
    assert torch.isnan(logits[[5, 150]]).all()
    assert logits[77, hot] == float("inf") and logits[231, hot] == -float("inf")
    good = torch.ones(M, dtype=torch.bool, device=DEV)
    good[bad] = False
    ref, bound = R.moe_logits(x[good], wg)
    check_bound(logits[good], ref, bound, f"nonfinite E={E} logits of the finite rows")
    nan_rows = [5, 77, 150] + ([231] if E == 1 else [])
    for r in nan_rows:
        assert torch.equal(v["ids"][r].long(), torch.arange(k, device=DEV)), (r, v["ids"][r])
        assert torch.isnan(v["weights"][r]).all(), r
    scored = good.clone()
    if E > 1:
        scored[231] = True
        assert (v["weights"][231][v["ids"][231] == hot] == 0).all()
    _check_route_picks(logits, v, scored, f"nonfinite E={E} k={k}")
    _, _, _, alone = _route(x[good], wg, k, cap)
    assert torch.equal(v["ids"][good], alone["ids"]) and torch.equal(v["weights"][good], alone["weights"])


def _combine_layout(M, E, k, cap, seed):
    """ids [M, k]: k distinct experts per row, in every order for k = 3 and in 8 of the 24 for k = 4, row by row; slots
    into a cap-row segment per expert, at a random permutation of positions 0 .. count - 1 within each segment."""
    g = torch.Generator().manual_seed(seed)
    chosen = torch.rand(M, E, generator=g).argsort(dim=1)[:, :k].sort(dim=1).values
    orders = list(itertools.permutations(range(k)))
    if k == 4:
        orders = orders[::3]
    order = torch.tensor(orders)[torch.arange(M) % len(orders)]
    ids = chosen.gather(1, order)
    flat = ids.flatten()
    by_seg = (flat * (M * k) + torch.randperm(M * k, generator=g)).argsort()
    counts = torch.bincount(flat, minlength=E)
    start = torch.cumsum(counts, 0) - counts
    pos = torch.empty_like(flat)
    pos[by_seg] = torch.arange(M * k) - start[flat[by_seg]]
    return ids, (ids * cap + pos.view(M, k)), counts


@pytest.mark.parametrize("alias", [True, False])
@pytest.mark.parametrize("M", [1, 129, 8884])
@pytest.mark.parametrize("N", [8, 136, 392])
@pytest.mark.parametrize("k", [1, 2, 3, 4])
def test_moe_combine(k, N, M, alias):
    """The combine mode against its mirror: out (and the residual, when it is not out) a view into a wider buffer, the
    routed rows of slot_y in cap = M + 37 segments whose unused rows are NaN; N = 136 and 392 end in partial column
    tiles.  Moving rows inside each segment of slot_y, with slots moved to match, gives the same bits."""
    ops = _ops()
    E, K = 6, 256
    cap = M + 37
    seed = k * 1000 + N + M
    ids, slots, counts = _combine_layout(M, E, k, cap, seed)
    ids, slots = ids.int().to(DEV), slots.int().to(DEV)
    slot_y = torch.full((E * cap, N), float("nan"), device=DEV, dtype=torch.float16)
    used = slots.long().flatten()
    slot_y[used] = _randn(used.numel(), N, std=0.7, seed=seed + 1)
    x, w, b = _randn(M, K, seed=seed + 2), _randn(N, K, std=K ** -0.5, seed=seed + 3), _randn(N, seed=seed + 4)
    res = _randn(M, N, std=2.0, seed=seed + 5)
    ref, bound = R.moe_combine(x, w, b, slot_y, ids, slots, res)

    def run(slot_y, slots):
        obuf = torch.full((M, N + 24), GUARD16, device=DEV, dtype=torch.float16)
        out = obuf[:, 8:8 + N]
        if alias:
            out.copy_(res)
            residual = out
        else:
            rbuf = torch.full_like(obuf, GUARD16)
            residual = rbuf[:, 8:8 + N]
            residual.copy_(res)
        ops.moe_combine(x, w, b, slot_y=slot_y, ids=ids, slots=slots, residual=residual, out=out)
        outside = torch.ones_like(obuf, dtype=torch.bool)
        outside[:, 8:8 + N] = False
        assert (obuf[outside] == GUARD16).all()
        if not alias:
            assert torch.equal(residual, res)
        return out

    out = run(slot_y, slots)
    check_bound(out, ref, bound, f"combine k={k} N={N} M={M} alias={alias}")
    # reverse the rows of every segment: position p of expert e moves to count_e - 1 - p
    e, p = slots.long() // cap, slots.long() % cap
    moved = e * cap + counts.to(DEV)[e] - 1 - p
    slot_y2 = torch.full_like(slot_y, float("nan"))
    slot_y2[moved.flatten()] = slot_y[slots.long().flatten()]
    assert torch.equal(run(slot_y2, moved.int()), out)
