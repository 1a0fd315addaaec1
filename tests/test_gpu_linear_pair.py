"""GPU: two independent linears in one launch (r3g_linear_args.group_next) must give exactly the results of two
separate launches -- for every tile variant the dispatcher can pick, with segmented rows, different N / K per problem and
every epilogue of the DiT's DoubleStreamBlock (hunyuan3ddit.py:196-216)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(M, N, K, seed, seg=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(M, K, device="cuda", generator=g) * 0.5).half()
    w = (torch.randn(N, K, device="cuda", generator=g) * 0.05).half()
    b = (torch.randn(N, device="cuda", generator=g) * 0.1).half()
    return x, w, b


@pytest.mark.parametrize("shape", [
    dict(Ma=6144, Mb=2740, N=1024, K=1024),      # proj of a double block: 128 x 256 tiles
    dict(Ma=6144, Mb=2740, N=1024, K=4096),      # mlp.2: K = 4096
    dict(Ma=700, Mb=300, N=128, K=256),          # 128-wide tiles
    dict(Ma=300, Mb=200, N=64, K=64),            # N = 64: half-filled 128-wide tiles
    dict(Ma=1000, Mb=9, N=512, K=320),           # a tiny second problem
])
def test_pair_equals_two_launches(shape):
    from r3g import ops
    xa, wa, ba = _mk(shape["Ma"], shape["N"], shape["K"], 1)
    xb, wb, bb = _mk(shape["Mb"], shape["N"], shape["K"], 2)
    ya, yb = ops.linear(xa, wa, ba, act=ops.ACT_GELU_TANH), ops.linear(xb, wb, bb, act=ops.ACT_GELU_TANH)
    pa, pb = ops.linear_pair(dict(x=xa, w=wa, bias=ba, act=ops.ACT_GELU_TANH), dict(x=xb, w=wb, bias=bb, act=ops.ACT_GELU_TANH))
    assert torch.equal(ya, pa) and torch.equal(yb, pb)
    ref = torch.nn.functional.gelu(xa.float() @ wa.float().t() + ba.float(), approximate="tanh")
    assert (pa.float() - ref).abs().max().item() < 2e-2 * ref.abs().max().item()


def test_pair_of_stream_segments_with_gated_residual_and_qk_norm():
    """The DoubleStreamBlock form: both problems are row segments [B, L_s, .] of joint buffers, different N and K,
    gate * y + residual in place, and the fused q/k RMS norm on the qkv pair."""
    from r3g import ops
    B, Lt, Li, H = 2, 137, 307, 256
    L = Lt + Li
    g = torch.Generator(device="cuda").manual_seed(0)
    X = (torch.randn(B, L, H, device="cuda", generator=g)).half()
    QKV = torch.zeros(B, L, 3 * H, device="cuda", dtype=torch.float16)
    w = {s: (torch.randn(3 * H, H, device="cuda", generator=g) * 0.05).half() for s in "it"}
    b = {s: (torch.randn(3 * H, device="cuda", generator=g) * 0.1).half() for s in "it"}
    nq = {s: (1 + 0.1 * torch.randn(64, device="cuda", generator=g)).half() for s in "it"}
    nk = {s: (1 + 0.1 * torch.randn(64, device="cuda", generator=g)).half() for s in "it"}
    seg = {"i": (Lt, Li), "t": (0, Lt)}

    def call(s, out):
        o, n = seg[s]
        return dict(x=X[:, o:o + n], w=w[s], bias=b[s], out=out[:, o:o + n],
                    qk_norm=dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H, cols=H, eps=1e-6, q_w=nq[s], k_w=nk[s]))
    sep = torch.zeros_like(QKV)
    ops.linear(**call("i", sep)); ops.linear(**call("t", sep))
    ops.linear_pair(call("i", QKV), call("t", QKV))
    assert torch.equal(sep, QKV)
    # gated residual, written in place over the residual stream; the two problems have different K here
    gate = (torch.randn(B, 2 * H, device="cuda", generator=g)).half()
    wp = {"i": (torch.randn(H, H, device="cuda", generator=g) * 0.05).half(),
          "t": (torch.randn(H, 3 * H, device="cuda", generator=g) * 0.05).half()}
    bp = {s: (torch.randn(H, device="cuda", generator=g) * 0.1).half() for s in "it"}

    def call2(s, buf):
        o, n = seg[s]
        src = QKV[:, o:o + n, :H] if s == "i" else QKV[:, o:o + n]
        gt = gate[:, :H] if s == "i" else gate[:, H:]
        return dict(x=src, w=wp[s], bias=bp[s], out=buf[:, o:o + n], gate=gt, gate_rows=n, residual=buf[:, o:o + n])
    X1, X2 = X.clone(), X.clone()
    ops.linear(**call2("i", X1)); ops.linear(**call2("t", X1))
    ops.linear_pair(call2("i", X2), call2("t", X2))
    assert torch.equal(X1, X2) and not torch.equal(X1, X)


def test_dit_grouped_equals_ungrouped():
    from r3g.dit import Hunyuan3DDiT
    m = Hunyuan3DDiT(in_channels=64, context_in_dim=96, hidden_size=256, num_heads=4, depth=2, depth_single_blocks=1).init_random(3)
    torch.manual_seed(0)
    x = torch.randn(2, 300, 64, device="cuda").half()
    c = torch.randn(2, 77, 96, device="cuda").half()
    t = torch.tensor([0.4, 0.4], device="cuda").half()
    m.group_streams = True
    a = m(x, t, {"main": c}).clone()
    m.group_streams = False
    b = m(x, t, {"main": c}).clone()
    assert torch.equal(a, b)
