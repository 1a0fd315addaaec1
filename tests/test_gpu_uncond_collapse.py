"""GPU: the DiT's collapsed unconditional branch (Hunyuan3DDiT.forward, uncond_txt_shared) and the kernel features it
runs on -- three GEMM problems in one launch and windowed attention with a counted first key (include/r3g.h)."""
import types

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("Lt,Li,H", [(137, 307, 256), (1370, 3072, 1024)])
def test_group_of_three_equals_three_launches(Lt, Li, H):
    """The collapsed DoubleStreamBlock form: img rows of both batches (segmented), txt rows of batch 0, and batch 1's single
    text row -- with a gated residual in place, and the fused q/k RMS norm on the qkv projection."""
    from r3g import ops
    B, L = 2, Lt + Li
    g = torch.Generator(device="cuda").manual_seed(0)
    X = torch.randn(B, L, H, device="cuda", generator=g).half()
    w = {s: (torch.randn(3 * H, H, device="cuda", generator=g) * 0.05).half() for s in "it"}
    b = {s: (torch.randn(3 * H, device="cuda", generator=g) * 0.1).half() for s in "it"}
    nq = {s: (1 + 0.1 * torch.randn(64, device="cuda", generator=g)).half() for s in "it"}
    nk = {s: (1 + 0.1 * torch.randn(64, device="cuda", generator=g)).half() for s in "it"}
    gate = torch.randn(B, 2 * H, device="cuda", generator=g).half()
    wp = {s: (torch.randn(H, 3 * H, device="cuda", generator=g) * 0.05).half() for s in "it"}
    bp = {s: (torch.randn(H, device="cuda", generator=g) * 0.1).half() for s in "it"}
    probs = (("i", slice(None), Lt, Li), ("t", slice(0, 1), 0, Lt), ("t", slice(1, 2), Lt - 1, 1))

    def qkv(p, out):
        s, bs, o, n = p
        return dict(x=X[bs, o:o + n], w=w[s], bias=b[s], out=out[bs, o:o + n],
                    qk_norm=dict(mode=ops.QKN_RMS, q_col0=0, k_col0=H, cols=H, eps=1e-6, q_w=nq[s], k_w=nk[s]))

    def proj(p, src, buf):
        s, bs, o, n = p
        gt = (gate[:, :H] if s == "i" else gate[:, H:])[bs]
        return dict(x=src[bs, o:o + n], w=wp[s], bias=bp[s], out=buf[bs, o:o + n], gate=gt, gate_rows=n,
                    residual=buf[bs, o:o + n])
    sep, grp = torch.zeros(B, L, 3 * H, device="cuda", dtype=torch.float16), torch.zeros(B, L, 3 * H, device="cuda",
                                                                                          dtype=torch.float16)
    for p in probs:
        ops.linear(**qkv(p, sep))
    ops.linear_group(*[qkv(p, grp) for p in probs])
    assert torch.equal(sep, grp) and sep[1, Lt - 1].abs().sum() > 0 and not sep[1, :Lt - 1].any()
    X1, X2 = X.clone(), X.clone()
    for p in probs:
        ops.linear(**proj(p, sep, X1))
    ops.linear_group(*[proj(p, sep, X2) for p in probs])
    assert torch.equal(X1, X2) and not torch.equal(X1[1, Lt - 1], X[1, Lt - 1])
    assert torch.equal(X1[1, :Lt - 1], X[1, :Lt - 1])        # batch 1's other text rows are not touched


def test_group_rejects_more_than_three():
    from r3g import ops
    x = torch.randn(8, 64, device="cuda").half()
    w = torch.randn(64, 64, device="cuda").half()
    with pytest.raises(ValueError):
        ops.linear_group(*[dict(x=x, w=w)] * 4)


def test_windowed_attention_with_counted_first_key():
    """Batch 1's text rows [0, Lt) are Lt copies of one row.  Computing only its query window [Lt - 1, L), with the window's
    first key counted Lt times, must match full attention bit for bit, though k / v rows [0, Lt - 1) start out as
    garbage: the call fills them with row Lt - 1's.  Batch 0's window is the whole sequence."""
    from r3g import ops
    Lt, Li, H = 1370, 3072, 16
    L = Lt + Li
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(2, L, 3, H, 64, device="cuda", generator=g).half()
    qkv[1, :Lt - 1] = qkv[1, Lt - 1]
    full = ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2])
    dirty = qkv.clone()
    dirty[1, :Lt - 1] = torch.randn(Lt - 1, 3, H, 64, device="cuda", generator=g).half()
    out = torch.full((2, L, H, 64), 7.0, device="cuda", dtype=torch.float16)
    ops.attention(dirty[:, :, 0], dirty[:, :, 1], dirty[:, :, 2], out=out, windows=((0, L, 1), (Lt - 1, Li + 1, Lt)))
    assert torch.equal(out[0], full[0]) and torch.equal(out[1, Lt - 1:], full[1, Lt - 1:])
    assert (out[1, :Lt - 1] == 7.0).all()                                   # rows outside the window are not written
    assert torch.equal(dirty[1, :, 1:], qkv[1, :, 1:])                      # k and v were filled, q was not
    assert not torch.equal(dirty[1, :Lt - 1, 0], qkv[1, :Lt - 1, 0])
    from r3g._abi import R3GError
    with pytest.raises(R3GError):                                           # not enough rows before the window
        ops.attention(qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2], windows=((0, L, 1), (Lt - 1, Li + 1, Lt + 1)))


@pytest.fixture(scope="module")
def full_dit():
    from r3g.dit import Hunyuan3DDiT
    return Hunyuan3DDiT().init_random(seed=21)


def test_full_depth_forward_collapsed_against_full(full_dit):
    m = full_dit
    torch.manual_seed(0)
    x = torch.randn(2, 3072, 64, device="cuda").half()
    c = torch.cat([torch.randn(1, 1370, 1536, device="cuda"), torch.zeros(1, 1370, 1536, device="cuda")]).half()
    t = torch.tensor([0.3469, 0.3469], device="cuda").half()
    full = m(x, t, {"main": c}).clone()
    coll = m(x, t, {"main": c}, uncond_txt_shared=True).clone()
    assert torch.equal(coll, full)


class _FullPathOnly:
    """The model with the collapsed branch switched off, to run _denoise on the full path as a reference."""

    def __init__(self, m):
        self.m, self.taps = m, None

    def __call__(self, x, t, contexts, uncond_txt_shared=False):
        return self.m(x, t, contexts)


def _pipe(model):
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline, ImageProcessorV2
    from r3g.scheduler import FlowMatchEulerDiscreteScheduler
    return Hunyuan3DDiTFlowMatchingPipeline(
        vae=types.SimpleNamespace(latent_shape=(3072, 64)), model=model,
        scheduler=FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000), conditioner=None,
        image_processor=ImageProcessorV2(size=512, border_ratio=0.15))


def _latents(pipe, un, steps):
    torch.manual_seed(1)
    cond = {"main": torch.cat([torch.randn(1, 1370, 1536).cuda().half(), un])}
    lat0 = torch.randn((1, 3072, 64), generator=torch.manual_seed(1234567), dtype=torch.float16)
    out = pipe(cond=cond, latents=lat0, num_inference_steps=steps, guidance_scale=5.0, output_type="latent")
    return out.clone(), [k[-1] for k in pipe._graphs.entries]


def test_denoise_selects_the_path_from_the_input(full_dit):
    steps = 3
    rnd = torch.randn(1, 1370, 1536, generator=torch.manual_seed(5)).cuda().half()
    got, keys = _latents(_pipe(full_dit), rnd, steps)
    ref, _ = _latents(_pipe(_FullPathOnly(full_dit)), rnd, steps)
    assert keys == [False] and torch.equal(got, ref)
    const = torch.randn(1, 1, 1536, generator=torch.manual_seed(6)).expand(1, 1370, 1536).cuda().half()
    _, keys = _latents(_pipe(full_dit), const, steps)
    assert keys == [True]


def test_fifty_steps_collapsed_against_full(full_dit):
    zeros = torch.zeros(1, 1370, 1536, device="cuda", dtype=torch.float16)
    got, keys = _latents(_pipe(full_dit), zeros, 50)
    ref, _ = _latents(_pipe(_FullPathOnly(full_dit)), zeros, 50)
    assert keys == [True] and torch.equal(got, ref)
