"""CPU: the float32 torch mirrors of VGGT's point head and track head, and VGGT.forward composed of them, against
tests/golden/vggt_point_track_mini.npz, which oracle/make_golden_vggt_heads.py generates from the reference's own
DPTHead / TrackHead / VGGT modules on r3g.vggt_heads.random_state_dict weights; the state-dict surface of VGGT."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "oracle"), os.path.join(ROOT, "3d-re-gen_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import make_golden_vggt_heads as G  # noqa: E402
from r3g import vggt_heads as M  # noqa: E402
from r3g.vggt_track import TrackHead  # noqa: E402


@pytest.fixture(scope="module")
def fx(golden_dir):
    z = np.load(os.path.join(golden_dir, "vggt_point_track_mini.npz"))
    toks, images, qp = G.inputs()
    for name, t in (("sum_tokens", torch.stack(toks)), ("sum_images", images), ("sum_query", qp)):
        # the float64 sum's order follows torch's thread count: equal to reassociation, not bit for bit
        assert np.isclose(G.checksum(t), z[name], rtol=1e-10, atol=0), f"{name}: the seeded inputs differ from the fixture's"
    return z, M.random_state_dict(**G.WEIGHTS), toks, images, qp


def _close(a, ref, tol=1e-4):
    a, ref = np.asarray(a, np.float64), np.asarray(ref, np.float64)
    assert a.shape == ref.shape
    err = np.abs(a - ref).max() / max(1.0, np.abs(ref).max())
    assert err < tol, f"max error {err:.2e} (relative to max(1, |ref|))"


def test_point_head_mirror_matches_reference(fx):
    z, sd, toks, images, _ = fx
    head = M.DPTHead(sd, "point_head.", activation="inv_log", device="cpu")
    pts, conf = head(toks, images, 5)
    k = G.SUB["heads"]
    assert pts.shape == (1, G.S, G.H, G.W, 3) and conf.shape == (1, G.S, G.H, G.W)
    _close(pts[:, :, ::k, ::k], z["heads_points"])
    _close(conf[:, :, ::k, ::k], z["heads_points_conf"])


# vis / conf read the track features after four updates, each of which feeds the previous one's float32 rounding
# (reassociated sums in the correlation GEMMs and attention) back through the correlation lookup: after one iteration
# mirror and reference agree to 3e-7, after four to 3e-4, so they are held to 1e-3.
VIS_TOL = 1e-3


def test_track_head_mirror_matches_reference(fx):
    z, sd, toks, images, qp = fx
    track_list, vis, conf = TrackHead(sd, device="cpu")(toks, images, 5, qp, iters=G.ITERS)
    assert len(track_list) == G.ITERS
    for i, t in enumerate(track_list):
        assert t.shape == (1, G.S, G.NQ, 2) and t.dtype == torch.float32
        _close(t, z["heads_track"][i])
    _close(vis, z["heads_vis"], VIS_TOL)
    _close(conf, z["heads_conf"], VIS_TOL)


def _mini_model(sd, **kw):
    """VGGT on the CPU mirrors with the oracle's float32 aggregator standing in for the libr3g one (CUDA only)."""
    import vggt_ref as V
    model = M.VGGT(img_size=G.H, embed_dim=G.EMBED, depth=G.LAYERS, num_heads=1, patch_embed="conv", device="cpu",
                   camera_head_kwargs=dict(num_heads=16), **kw).load_state_dict(sd)
    asd = {k[len("aggregator."):]: v for k, v in sd.items() if k.startswith("aggregator.")}
    model.aggregator = lambda images: (V.aggregator(asd, images, G.LAYERS, 1), 5)
    return model


def test_forward_matches_reference_model(fx):
    z, sd, _, images, qp = fx
    pred = _mini_model(sd)(images[0], qp[0])
    assert sorted(pred) == sorted(z["model_keys"].tolist())
    for k, v in pred.items():
        if k == "pose_enc_list":
            assert len(v) == len(z["model_pose_enc_list"])
            for a, b in zip(v, z["model_pose_enc_list"]):
                _close(a, b)
            continue
        assert tuple(v.shape) == tuple(z["model_shape_" + k]) and v.dtype == torch.float32, k
        if k in ("depth", "depth_conf", "world_points", "world_points_conf"):
            n = G.SUB["model"]
            _close(v[:, :, ::n, ::n], z["model_" + k])
        elif k != "images":
            _close(v, z["model_" + k], VIS_TOL if k in ("vis", "conf") else 1e-4)
    assert torch.equal(pred["images"], images)


def test_forward_without_query_points_or_disabled_heads(fx):
    _, sd, _, images, qp = fx
    pred = _mini_model(sd)(images)
    assert not {"track", "vis", "conf"} & set(pred)
    pred = _mini_model(sd, enable_point=False, enable_track=False)(images, qp)
    assert set(pred) == {"pose_enc", "pose_enc_list", "depth", "depth_conf", "images"}


def test_generator_reproduces_fixture(golden_dir, tmp_path, monkeypatch):
    import ref_import
    if not os.path.isdir(os.path.join(ref_import.VGGT, "vggt")):
        pytest.skip("the reference checkout is not on this machine")
    monkeypatch.setattr(G, "OUT", str(tmp_path / "f.npz"))
    G.main()
    a, b = np.load(G.OUT), np.load(os.path.join(golden_dir, "vggt_point_track_mini.npz"))
    assert sorted(a.files) == sorted(b.files)
    for k in a.files:
        if a[k].dtype.kind in "fc":      # the reference's own float32 rounding varies with torch's thread count
            _close(a[k], b[k], VIS_TOL if k.endswith(("_vis", "_conf")) and "points" not in k else 1e-4)
        else:
            assert np.array_equal(a[k], b[k]), k


def test_full_state_dict_loads_strictly_and_names_bad_keys():
    sd = M.random_state_dict(3, embed_dim=64, depth=2, vit_depth=0, trunk_depth=1, features=32,
                             out_channels=(32, 64, 128, 128), img_size=56, full=True, patch_embed="conv")
    kw = dict(img_size=56, embed_dim=64, depth=2, num_heads=1, patch_embed="conv", device="cpu",
              camera_head_kwargs=dict(trunk_depth=1), depth_head_kwargs=dict(intermediate_layer_idx=(0, 1, 0, 1)),
              point_head_kwargs=dict(intermediate_layer_idx=(0, 1, 0, 1)),
              track_head_kwargs=dict(intermediate_layer_idx=(0, 1, 0, 1)))
    model = M.VGGT(**kw).load_state_dict(sd)
    assert isinstance(model.track_head, TrackHead) and model.point_head.activation == "inv_log"
    # the camera + depth state dict builds exactly the stage-4 heads
    base = {k: v for k, v in sd.items() if not k.startswith(("point_head.", "track_head."))}
    model = M.VGGT(**kw).load_state_dict(base)
    assert model.point_head is None and model.track_head is None and model.depth_head is not None
    with pytest.raises(KeyError, match="enable_track=True"):
        M.VGGT(enable_track=True, **kw).load_state_dict(base)
    broken = dict(sd)
    del broken["track_head.tracker.updateformer.time_blocks.3.mlp.fc1.weight"], broken["point_head.norm.bias"]
    with pytest.raises(KeyError, match=r"point_head\.norm\.bias.*time_blocks\.3\.mlp\.fc1\.weight"):
        M.VGGT(**kw).load_state_dict(broken)
    extra = dict(sd, **{"track_head.tracker.bogus": torch.zeros(1)})
    with pytest.raises(KeyError, match=r"unexpected keys \['track_head\.tracker\.bogus'\]"):
        M.VGGT(**kw).load_state_dict(extra)
    M.VGGT(**kw).load_state_dict(extra, strict=False)
    assert M.VGGT(enable_track=False, **kw).load_state_dict(extra).track_head is None     # a head left out: keys ignored
    with pytest.raises(KeyError, match=r"unexpected keys \['decoder\.w'\]"):
        M.VGGT(**kw).load_state_dict(dict(sd, **{"decoder.w": torch.zeros(1)}))


def test_tracker_padding_388_to_392_is_exact():
    """TrackHeadR3G's load-time layout: input_transform zero-padded from K = 388 to 392, corr_mlp.fc1 from 567 to 568,
    attention heads from 48 to 64 columns, flow_head reordered and padded to 160 rows.  Evaluated in float32 on the CPU,
    each padded form gives the unpadded product."""
    sd = M.random_state_dict(3, embed_dim=64, depth=1, vit_depth=0, trunk_depth=1, features=32,
                             out_channels=(32, 64, 128, 128), img_size=56, full=True, patch_embed="conv")
    from r3g import vggt_track as T
    raw = {k[len("track_head.tracker."):]: v for k, v in sd.items() if k.startswith("track_head.tracker.")}
    w = T.pad_tracker_weights(raw, torch.device("cpu"), 7, 4)
    u = "updateformer."
    g = torch.Generator().manual_seed(0)
    x = torch.randn(10, T.TDIM, generator=g)
    xp = torch.cat([x, torch.zeros(10, T.TDIM_PAD - T.TDIM)], 1)
    ref = torch.nn.functional.linear(x, raw[u + "input_transform.weight"], raw[u + "input_transform.bias"])
    got = torch.nn.functional.linear(xp, w[u + "input_transform"][0].float(), w[u + "input_transform"][1].float())
    assert torch.allclose(got, torch.nn.functional.linear(x, raw[u + "input_transform.weight"].half().float(),
                                                          raw[u + "input_transform.bias"].half().float()), atol=1e-6)
    assert (got - ref).abs().max() < 1e-2
    c = torch.randn(10, 567, generator=g)
    cp = torch.cat([c, torch.zeros(10, 1)], 1)
    assert torch.allclose(torch.nn.functional.linear(cp, w["corr_mlp.fc1"][0].float()),
                          torch.nn.functional.linear(c, raw["corr_mlp.fc1.weight"].half().float()), atol=1e-5)
    # attention over 8 heads of 48 == over the same heads zero-padded to 64 (scale 48^-0.5)
    p = u + "time_blocks.0.attn."
    h = torch.randn(2, 5, T.HIDDEN, generator=g)
    ref = T._mha({k[len(p):]: v.half().float() for k, v in raw.items() if k.startswith(p)}, "", h, h)
    wqkv, bqkv = (t.float() for t in w[p + "qkv"])
    qkv = torch.nn.functional.linear(h, wqkv, bqkv).view(2, 5, 3, T.HEADS, 64).permute(2, 0, 3, 1, 4)
    o = torch.nn.functional.scaled_dot_product_attention(qkv[0], qkv[1], qkv[2], scale=48 ** -0.5)
    o = torch.nn.functional.linear(o.transpose(1, 2).reshape(2, 5, -1), *(t.float() for t in w[p + "out"]))
    assert torch.allclose(o, ref, atol=1e-5)
    fw = torch.nn.functional.linear(h, w[u + "flow_head"][0].float(), w[u + "flow_head"][1].float())
    fr = torch.nn.functional.linear(h, raw[u + "flow_head.weight"].half().float(), raw[u + "flow_head.bias"].half().float())
    assert torch.allclose(fw[..., :128], fr[..., 2:], atol=1e-6) and torch.allclose(fw[..., 128:130], fr[..., :2], atol=1e-6)
    assert torch.count_nonzero(fw[..., 130:]) == 0
