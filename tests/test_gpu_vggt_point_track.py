"""GPU: VGGT's point head and track head on libr3g against tests/golden/vggt_point_track_mini.npz (the reference's own
modules, oracle/make_golden_vggt_heads.py) and, at full width, against the float32 torch mirrors; VGGT.forward.

Bounds.  The point head is held to the depth head's rel-L2 <= 1e-2 (fp16 operands, float32 accumulation).  The track
head's fp16 rounding enters at the GEMM operands (track features and LayerNormed pixel rows of the correlation, every
block input of the update former), at each branch output before it joins a float32 stream, and at the MLP hidden
activations; four iterations feed each other's coordinates back through the correlation lookup, so the coordinate
error grows per iteration.  Measured on an H100 80GB HBM3 (700 W): per-iteration coordinate error 0.0003, 0.003, 0.012,
0.043 px on the fixture and 0.0003, 0.002, 0.017, 0.054 px at 518 x 518, S = 4, N = 256; vis / conf error 0.029 / 0.018
and 0.014 / 0.036.  vis / conf are sigmoids of a linear of the track features after four updates, each of which
LayerNorms (GroupNorm) the fp16-rounded flow-head output: their error is the largest.  The bounds below leave about
4x (coordinates) and 2x (vis / conf) over the worst measured value; fp16 operands keep the last iteration far inside
1 px of the float32 mirror, so no GEMM of the tracker needs float32 operands."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "3d-re-gen_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

# per-iteration track coordinates (pixels, max over points and frames) and vis / conf (absolute), r3g vs float32
TRACK_PX = 0.25
VIS_ABS = 8e-2


def rel_l2(a, b):
    a, b = a.double().flatten().cpu(), torch.as_tensor(b).double().flatten().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


@pytest.fixture(scope="module")
def fx(golden_dir):
    import make_golden_vggt_heads as G
    from r3g.vggt_heads import random_state_dict
    z = np.load(os.path.join(golden_dir, "vggt_point_track_mini.npz"))
    toks, images, qp = G.inputs()
    return G, z, random_state_dict(**G.WEIGHTS), [t.cuda() for t in toks], images.cuda(), qp.cuda()


def _track_errors(a, b):
    (la, va, ca), (lb, vb, cb) = a, b
    d = lambda x, y: (x.cpu() - torch.as_tensor(y).cpu()).abs().max().item()  # noqa: E731
    return [d(x, y) for x, y in zip(la, lb)], d(va, vb), d(ca, cb)


def test_point_head_against_fixture_and_mirror(fx):
    from r3g.vggt_heads import DPTHead, DPTHeadR3G, random_state_dict
    G, z, sd, toks, images, _ = fx
    pts, conf = DPTHeadR3G(sd, "point_head.", activation="inv_log")(toks, images, 5)
    k = G.SUB["heads"]
    assert pts.shape == (1, G.S, G.H, G.W, 3) and conf.shape == (1, G.S, G.H, G.W) and pts.dtype == torch.float32
    e = rel_l2(pts[:, :, ::k, ::k], z["heads_points"]), rel_l2(conf[:, :, ::k, ::k], z["heads_points_conf"])
    print(f"point head vs reference fixture: points rel-L2 {e[0]:.2e}, confidence {e[1]:.2e}")
    assert max(e) < 1e-2
    # full width: dim_in 2048, features 256, out_channels (256, 512, 1024, 1024), 518 x 518, two frames
    full = random_state_dict(5, embed_dim=1024, depth=1, vit_depth=1, trunk_depth=1, full=True)
    full = {k: v.half().float() for k, v in full.items() if k.startswith("point_head.")}
    torch.manual_seed(1)
    P = 37 * 37
    toks = [torch.randn(1, 2, 5 + P, 2048, device="cuda") for _ in range(2)]
    imgs = torch.rand(1, 2, 3, 518, 518, device="cuda")
    kw = dict(activation="inv_log", intermediate_layer_idx=(0, 1, 0, 1))
    p1, c1 = DPTHeadR3G(full, "point_head.", **kw)(toks, imgs, 5)
    p2, c2 = DPTHead(full, "point_head.", device="cuda", **kw)(toks, imgs, 5)
    e = rel_l2(p1, p2), rel_l2(c1, c2)
    print(f"point head at full width vs float32 mirror: points rel-L2 {e[0]:.2e}, confidence {e[1]:.2e}")
    assert max(e) < 1e-2


def test_track_head_against_fixture(fx):
    from r3g.vggt_track import TrackHeadR3G
    G, z, sd, toks, images, qp = fx
    head = TrackHeadR3G(sd)
    track_list, vis, conf = head(toks, images, 5, qp)
    assert len(track_list) == G.ITERS and all(t.shape == (1, G.S, G.NQ, 2) for t in track_list)
    assert vis.shape == conf.shape == (1, G.S, G.NQ) and vis.dtype == conf.dtype == torch.float32
    px, ev, ec = _track_errors((track_list, vis, conf), (list(z["heads_track"]), z["heads_vis"], z["heads_conf"]))
    print(f"track head vs reference fixture: per-iteration px {['%.3g' % p for p in px]}, vis {ev:.2e}, conf {ec:.2e}")
    assert max(px) < TRACK_PX and max(ev, ec) < VIS_ABS


def test_track_head_full_size_against_mirror():
    """518 x 518, S = 4, N = 256 query points, VGGT-1B widths (dim_in 2048)."""
    from r3g.vggt_heads import random_state_dict
    from r3g.vggt_track import TrackHead, TrackHeadR3G
    sd = random_state_dict(6, embed_dim=1024, depth=1, vit_depth=1, trunk_depth=1, full=True)
    sd = {k: (v.half().float() if v.dim() >= 2 else v) for k, v in sd.items() if k.startswith("track_head.")}
    torch.manual_seed(2)
    S, N = 4, 256
    toks = [torch.randn(1, S, 5 + 37 * 37, 2048, device="cuda") for _ in range(2)]
    imgs = torch.rand(1, S, 3, 518, 518, device="cuda")
    qp = torch.rand(1, N, 2, device="cuda") * 517
    kw = dict(intermediate_layer_idx=(0, 1, 0, 1))
    mine = TrackHeadR3G(sd, **kw)(toks, imgs, 5, qp)
    ref = TrackHead(sd, device="cuda", **kw)(toks, imgs, 5, qp)
    px, ev, ec = _track_errors(mine, ref)
    print(f"track head at 518x518 S=4 N=256 vs float32 mirror: per-iteration px {['%.3g' % p for p in px]}, "
          f"vis {ev:.2e}, conf {ec:.2e}")
    assert max(px) < TRACK_PX and max(ev, ec) < VIS_ABS


def test_attention_over_zero_padded_48_wide_heads():
    """The tracker's attention: 8 heads of 48 zero-padded to 64 through ops.attention, scale 48^-0.5, against float32."""
    from r3g import ops
    torch.manual_seed(3)
    for B, Lq, Lk in ((320, 4, 4), (4, 64, 256), (4, 256, 64)):
        q, k, v = (torch.randn(B, L, 8, 48, device="cuda").half() for L in (Lq, Lk, Lk))
        pad = lambda t: torch.nn.functional.pad(t, (0, 16))  # noqa: E731
        o = ops.attention(pad(q), pad(k), pad(v), scale=48 ** -0.5)
        ref = torch.nn.functional.scaled_dot_product_attention(q.float().transpose(1, 2), k.float().transpose(1, 2),
                                                               v.float().transpose(1, 2)).transpose(1, 2)
        assert (o[..., :48].float() - ref).abs().max().item() < 2e-2
        assert torch.count_nonzero(o[..., 48:]) == 0


def test_correlation_gemm_against_float32():
    """x = fp16 query features [N, 128] (a strided view of the [N, S, 128] track rows), w = pixel rows [H*W padded to
    32, 128]: float32 out equals the float64 product of the fp16 operands to float32 accumulation error."""
    from r3g import ops
    torch.manual_seed(4)
    t = torch.randn(256, 4, 128, device="cuda").half()
    rows = torch.zeros(67104, 128, device="cuda", dtype=torch.float16)
    rows[:67081] = torch.randn(67081, 128, device="cuda").half()
    out = torch.empty(256, 67104, device="cuda")
    ops.linear(t[:, 2], rows, out=out)
    ref = t[:, 2].double() @ rows.double().t()
    assert (out.double() - ref).abs().max().item() < 1e-3
    assert torch.count_nonzero(out[:, 67081:]) == 0


def test_forward_with_and_without_query_points():
    from r3g.vggt_heads import VGGT, random_state_dict
    sd = random_state_dict(3, embed_dim=128, depth=2, vit_depth=0, trunk_depth=1, features=32,
                           out_channels=(32, 64, 128, 128), img_size=140, full=True, patch_embed="conv")
    idx = dict(intermediate_layer_idx=(0, 1, 0, 1))
    model = VGGT(img_size=140, embed_dim=128, depth=2, num_heads=2, patch_embed="conv",
                 camera_head_kwargs=dict(trunk_depth=1, num_heads=2), depth_head_kwargs=idx, point_head_kwargs=idx,
                 track_head_kwargs=idx).load_state_dict(sd)
    torch.manual_seed(5)
    images = torch.rand(3, 3, 140, 154, device="cuda")
    qp = torch.rand(24, 2, device="cuda") * 139
    pred = model(images, qp)
    shapes = {"pose_enc": (1, 3, 9), "depth": (1, 3, 140, 154, 1), "depth_conf": (1, 3, 140, 154),
              "world_points": (1, 3, 140, 154, 3), "world_points_conf": (1, 3, 140, 154), "track": (1, 3, 24, 2),
              "vis": (1, 3, 24), "conf": (1, 3, 24), "images": (1, 3, 3, 140, 154)}
    assert set(pred) == set(shapes) | {"pose_enc_list"} and len(pred["pose_enc_list"]) == 4
    for k, s in shapes.items():
        assert tuple(pred[k].shape) == s and pred[k].dtype == torch.float32 and torch.isfinite(pred[k]).all(), k
    # the heads one by one, as the stage script calls them, give the same tensors bit for bit
    tokens, psi = model.aggregator(images[None])
    assert torch.equal(model.camera_head(tokens)[-1], pred["pose_enc"])
    d, c = model.depth_head(tokens, images[None], psi)
    assert torch.equal(d, pred["depth"]) and torch.equal(c, pred["depth_conf"])
    track_list, vis, conf = model.track_head(tokens, images[None], psi, qp[None])
    assert torch.equal(track_list[-1], pred["track"]) and torch.equal(vis, pred["vis"])
    pred2 = model(images)
    assert not {"track", "vis", "conf"} & set(pred2)
    assert torch.equal(pred2["world_points"], pred["world_points"])
