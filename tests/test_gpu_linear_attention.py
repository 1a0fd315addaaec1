"""GPU: the wgmma building blocks (r3g_linear, r3g_attention) against fp32 PyTorch on the same inputs.
Tolerances: fp16 inputs, fp32 accumulation, fp16 output rounding -> |err| <= 2^-10 * |y| + accumulation noise."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _check(y, ref, rel=2e-3, what=""):
    err = (y.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= rel * scale + 1e-3, f"{what}: err {err} vs scale {scale}"


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (300, 384, 256), (1, 64, 64), (129, 128, 1024), (2740, 3072, 1024),
                                   (8884, 1024, 5120), (77, 96, 72), (5000, 7168, 1024), (640, 64, 1024)])
def test_linear_plain(M, N, K):
    from r3g import ops
    torch.manual_seed(M + N + K)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).half()
    b = torch.randn(N, device="cuda").half()
    y = ops.linear(x, w, b)
    _check(y, F.linear(x.float(), w.float(), b.float()), what=f"{M}x{N}x{K}")
    y32 = ops.linear(x, w, None, out_dtype=torch.float32)
    _check(y32, F.linear(x.float(), w.float()), rel=1e-4, what="fp32 out")


def test_linear_epilogues():
    from r3g import ops
    torch.manual_seed(5)
    B, L, K, N = 2, 333, 256, 512
    x = torch.randn(B * L, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") / 16).half()
    b = (torch.randn(N, device="cuda") * 0.1).half()
    lin = F.linear(x.float(), w.float(), b.float())
    _check(ops.linear(x, w, b, act=ops.ACT_GELU_TANH), F.gelu(lin, approximate="tanh"), what="gelu tanh")
    _check(ops.linear(x, w, b, act=ops.ACT_GELU_ERF), F.gelu(lin), what="gelu erf")
    part = lin.clone(); part[:, 128:384] = F.gelu(lin[:, 128:384], approximate="tanh")
    _check(ops.linear(x, w, b, act=ops.ACT_GELU_TANH, act_cols=(128, 384)), part, what="gelu on a column range")
    res = torch.randn(B * L, N, device="cuda").half()
    gate = torch.randn(B, N, device="cuda").half()
    ref = res.float() + gate.float().repeat_interleave(L, 0) * lin
    out = res.clone()
    ops.linear(x, w, b, out=out, gate=gate, gate_rows=L, residual=out)
    _check(out, ref, what="gated residual in place")
    out2 = ops.linear(x, w, b, residual=res, out=torch.empty_like(res))
    _check(out2, res.float() + lin, what="plain residual")
    # segmented rows: two segments of L rows written into a joint [B, L+7, N] buffer at row offset 7 ...
    joint = torch.zeros(B, L + 7, N, device="cuda", dtype=torch.float16)
    ops.linear(x, w, b, out=joint[:, 7:])
    _check(joint[:, 7:].reshape(-1, N), lin, what="segmented output")
    assert (joint[:, :7] == 0).all()
    # ... and read back from a segmented input view, with the gated residual indexed by segment
    xin = torch.zeros(B, L + 5, K, device="cuda", dtype=torch.float16)
    xin[:, 5:] = x.view(B, L, K)
    xin[:, :5] = 77.0
    out3 = res.clone().view(B, L, N)
    ops.linear(xin[:, 5:], w, b, out=out3, gate=gate, gate_rows=L, residual=out3)
    _check(out3.view(-1, N), ref, what="segmented input + gated residual")
    # strided input / output views
    big = torch.randn(B * L, 1024, device="cuda").half()
    obig = torch.zeros(B * L, 2048, device="cuda", dtype=torch.float16)
    ops.linear(big[:, 512:768], w, b, out=obig[:, 1024:1536])
    _check(obig[:, 1024:1536], F.linear(big[:, 512:768].float(), w.float(), b.float()), what="strided views")
    assert (obig[:, :1024] == 0).all() and (obig[:, 1536:] == 0).all()


@pytest.mark.parametrize("B,H,Lq,Lk", [(1, 1, 128, 128), (1, 2, 200, 300), (2, 16, 4442, 4442), (1, 16, 1000, 3072),
                                       (2, 3, 1, 129), (1, 4, 257, 64)])
def test_attention(B, H, Lq, Lk):
    from r3g import ops
    torch.manual_seed(Lq + Lk)
    q = torch.randn(B, Lq, H, 64, device="cuda").half()
    k = torch.randn(B, Lk, H, 64, device="cuda").half()
    v = torch.randn(B, Lk, H, 64, device="cuda").half()
    o = ops.attention(q, k, v)
    ref = F.scaled_dot_product_attention(q.float().transpose(1, 2), k.float().transpose(1, 2),
                                         v.float().transpose(1, 2)).transpose(1, 2)
    err = (o.float() - ref).abs().max().item()
    assert err < 4e-3, f"attention err {err}"


def test_attention_packed_qkv_in_place():
    """q/k/v as strided views of one packed [B, L, 3, H, 64] buffer, output written over q (DiT layout)."""
    from r3g import ops
    torch.manual_seed(9)
    B, L, H = 2, 700, 4
    qkv = torch.randn(B, L, 3, H, 64, device="cuda").half()
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    ref = F.scaled_dot_product_attention(q.float().transpose(1, 2), k.float().transpose(1, 2),
                                         v.float().transpose(1, 2)).transpose(1, 2)
    kc, vc = k.clone(), v.clone()
    ops.attention(q, k, v, out=q)
    assert (q.float() - ref).abs().max().item() < 4e-3
    assert torch.equal(k, kc) and torch.equal(v, vc)
    # peaked softmax (large logits): running-max rescale path
    q2 = (torch.randn(1, 300, 1, 64, device="cuda") * 6).half()
    k2 = (torch.randn(1, 500, 1, 64, device="cuda") * 6).half()
    v2 = torch.randn(1, 500, 1, 64, device="cuda").half()
    ref2 = F.scaled_dot_product_attention(q2.float().transpose(1, 2), k2.float().transpose(1, 2),
                                          v2.float().transpose(1, 2)).transpose(1, 2)
    assert (ops.attention(q2, k2, v2).float() - ref2).abs().max().item() < 6e-3


@pytest.mark.parametrize("M,N,K,act", [(300, 384, 256, False), (1000, 3072, 1024, False), (777, 7168, 512, True)])
@pytest.mark.parametrize("mode", [1, 2])
def test_linear_fused_qk_norm(M, N, K, act, mode):
    """The q/k normalisation inside the GEMM epilogue (qkn_*) against the separate r3g_qk_norm pass and against torch:
    RMSNorm / LayerNorm over each 64-column head of the fp16 Linear output (hunyuan3ddit.py:83-104,
    attention_blocks.py:315-316)."""
    from r3g import ops
    torch.manual_seed(5)
    x = torch.randn(M, K, device="cuda").half()
    w = (torch.randn(N, K, device="cuda") / K ** 0.5).half()
    b = torch.randn(N, device="cuda").half()
    qw, kw = (1 + 0.1 * torch.randn(64, device="cuda")).half(), (1 + 0.1 * torch.randn(64, device="cuda")).half()
    qb, kb = (0.1 * torch.randn(64, device="cuda")).half(), (0.1 * torch.randn(64, device="cuda")).half()
    cols = 128 if N < 1024 else 1024
    q0, k0 = 0, N - 2 * cols if act else cols
    kw_act = dict(act=ops.ACT_GELU_TANH, act_cols=(cols, N - 2 * cols)) if act else {}
    qk = dict(mode=mode, q_col0=q0, k_col0=k0, cols=cols, eps=1e-6, q_w=qw, k_w=kw)
    if mode == 2:
        qk.update(q_b=qb, k_b=kb)
    fused = ops.linear(x, w, b, qk_norm=qk, **kw_act)
    plain = ops.linear(x, w, b, **kw_act)
    two_pass = plain.clone()
    ops.qk_norm_(two_pass, cols // 64, q0, k0, 64, mode - 1, 1e-6, qw, qb if mode == 2 else None, kw,
                 kb if mode == 2 else None)
    # torch reference on the fp16 Linear output
    ref = plain.float().clone()
    for c0, wv, bv in ((q0, qw, qb), (k0, kw, kb)):
        h = plain[:, c0:c0 + cols].float().view(M, cols // 64, 64)
        if mode == 1:
            rr = torch.rsqrt(h.pow(2).mean(-1, keepdim=True) + 1e-6)
            y = (h * rr).half().float() * wv.float()
        else:
            y = F.layer_norm(h, (64,), wv.float(), bv.float(), 1e-6)
        ref[:, c0:c0 + cols] = y.reshape(M, cols)
    untouched = torch.ones(N, dtype=torch.bool, device="cuda")
    untouched[q0:q0 + cols] = False
    untouched[k0:k0 + cols] = False
    assert torch.equal(fused[:, untouched], plain[:, untouched])          # other columns: the ordinary epilogue
    d = (fused.float() - two_pass.float()).abs()
    assert d.max().item() <= 4e-3 and (d > 0).float().mean().item() < 0.02  # fp32 sum order only: rare 1-ulp flips
    assert (fused.float() - ref).abs().max().item() <= 6e-3
