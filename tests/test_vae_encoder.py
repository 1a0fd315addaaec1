"""CPU: the ShapeVAE encoder's fixture (tests/golden/vae_encoder_mini.npz, from the reference's own
PointCrossAttentionEncoder by oracle/make_golden_encoder.py), the oracle FPS against a brute-force restatement, r3g's
sampling on the fixture's draws, and checkpoint / config loading."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
FIXTURE = os.path.join(ROOT, "tests", "golden", "vae_encoder_mini.npz")
CASES = ["split", "nosharp", "full"]


def case(z, name):
    """(ShapeVAE kwargs, encoder + pre_kl state dict, surface, draws, fixture arrays) of one fixture geometry."""
    from hy3d_mini_ref import mini_state_dict
    i = lambda k: int(z[f"{name}_{k}"])  # noqa: E731
    kw = dict(num_latents=i("num_latents"), embed_dim=16, width=128, heads=2, num_decoder_layers=1,
              num_encoder_layers=i("layers"), pc_size=i("pc_size"), pc_sharpedge_size=i("pc_sharpedge_size"),
              point_feats=3, downsample_ratio=20, num_freqs=8, include_pi=bool(i("include_pi")),
              qkv_bias=bool(i("qkv_bias")), qk_norm=bool(i("qk_norm")), use_ln_post=True)
    sd = mini_state_dict(z[f"{name}_w_keys"], z[f"{name}_w_shapes"], i("seed"))
    t = lambda k: torch.from_numpy(z[f"{name}_{k}"])  # noqa: E731
    draws = (t("perm_r"), t("start_r"), t("perm_s"), t("start_s"))
    return kw, sd, t("surface"), draws


def ref_cfg(kw):
    return dict(num_freqs=kw["num_freqs"], include_pi=kw["include_pi"], heads=kw["heads"],
                layers=kw["num_encoder_layers"], qk_norm=kw["qk_norm"], use_ln_post=kw["use_ln_post"])


def cpu_vae(kw, sd):
    from r3g.vae import ShapeVAE
    vae = ShapeVAE(device="cpu", **kw)
    full = dict(ShapeVAE(device="cpu", **kw).init_random(5).reference_state_dict())
    full.update(sd)
    return vae.load_state_dict(full, strict=True), full


def brute_fps(pts, start, count):
    """Every pick from scratch: the minimum over the picks so far of the float32 squared distance, the first maximum."""
    pts = np.asarray(pts, dtype=np.float32)
    picks = [start]
    while len(picks) < count:
        best = None
        for j in range(len(pts)):
            dmin = np.float32(np.inf)
            for p in picks:
                dx, dy, dz = pts[j] - pts[p]
                dmin = min(dmin, np.float32(np.float32(dx * dx + dy * dy) + dz * dz))
            if best is None or dmin > best[0]:
                best = (dmin, j)
        picks.append(best[1])
    return np.array(picks)


def test_generator_reproduces_the_fixture(tmp_path):
    import ref_import
    if not ref_import.available():
        pytest.skip("the reference checkout is not present")
    import make_golden_encoder
    d = make_golden_encoder.generate(str(tmp_path / "enc.npz"))
    z = np.load(FIXTURE)
    assert sorted(d) == sorted(z.files)
    for k in z.files:
        assert np.array_equal(d[k], z[k]), k


@pytest.mark.parametrize("kind", ["ties", "duplicates", "random"])
def test_oracle_fps_matches_brute_force(kind):
    import vae_encoder_ref as V
    rng = np.random.default_rng(3)
    if kind == "ties":        # a lattice: many points at equal distances from the picks
        ax = np.arange(4, dtype=np.float32)
        pts = np.stack(np.meshgrid(ax, ax, ax[:2], indexing="ij"), -1).reshape(-1, 3)
    elif kind == "duplicates":  # every point twice, and an exact copy of the start
        base = rng.standard_normal((20, 3)).astype(np.float32)
        pts = np.concatenate([base, base])
    else:
        pts = rng.standard_normal((40, 3)).astype(np.float16).astype(np.float32)
    for start in (0, 7):
        assert np.array_equal(V.fps_segment(pts, start, 15), brute_fps(pts, start, 15)), (kind, start)


def test_oracle_fps_stub_segments_and_r3g_fps():
    """Three batch segments through the torch_cluster stand-in, each against the brute force; r3g's device FPS (run
    on the CPU here) picks the same points."""
    import vae_encoder_ref as V
    from r3g.vae import farthest_point_sample
    rng = np.random.default_rng(4)
    pts = rng.standard_normal((3, 30, 3)).astype(np.float16).astype(np.float32)
    pts[1, 10:20] = pts[1, :10]                       # duplicates in one segment
    src = torch.from_numpy(pts.reshape(-1, 3))
    batch = torch.arange(3).repeat_interleave(30)
    stub = V.FpsStub()
    torch.manual_seed(0)
    picks = stub(src, batch, ratio=0.3).numpy()
    starts = stub.calls[0][0]
    assert len(picks) == 3 * V.fps_count(30, 0.3) == 27
    for b in range(3):
        assert np.array_equal(picks[9 * b:9 * b + 9] - 30 * b, brute_fps(pts[b], int(starts[b]), 9))
    mine = farthest_point_sample(torch.from_numpy(pts), starts, 9)
    assert np.array_equal((mine + torch.arange(3)[:, None] * 30).reshape(-1).numpy(), picks)


@pytest.mark.parametrize("name", CASES)
def test_sampling_on_the_fixture_draws_and_the_float32_restatement(name):
    """r3g's sampling core picks the fixture's FPS points; the float32 restatement of the network on its rows gives
    the reference's moments."""
    import vae_encoder_ref as V
    z = np.load(FIXTURE)
    kw, sd, surface, draws = case(z, name)
    vae, _ = cpu_vae(kw, sd)
    q, d, (pick_r, pick_s) = vae.encoder.sample(surface, *draws)
    assert np.array_equal(pick_r.numpy(), z[f"{name}_fps_r"])
    assert np.array_equal(pick_s.numpy(), z[f"{name}_fps_s"])
    assert q.shape[1] == vae.encoder.queries() == z[f"{name}_mean"].shape[1]
    m = V.encoder_forward(sd, ref_cfg(kw), q, d)
    mean, logvar = m.chunk(2, -1)
    for got, key in ((mean, "mean"), (logvar.clamp(-30, 20), "logvar")):
        ref = torch.from_numpy(z[f"{name}_{key}"])
        assert (got - ref).abs().max() <= 1e-4 * ref.abs().max(), key


def test_query_counts_follow_the_reference():
    from r3g.vae import PointCrossAttentionEncoder
    e = lambda **k: PointCrossAttentionEncoder(  # noqa: E731
        **dict(dict(num_latents=16, downsample_ratio=20, pc_size=300, pc_sharpedge_size=200, point_feats=3, width=128,
                    heads=2, layers=1, device="cpu"), **k))
    assert e().plan() == ((192, 9.6 / 192, 10), (128, 6.4 / 128, 7))
    assert e().queries() == 17                               # ceil on both parts: one more than num_latents
    assert e(pc_size=5120, pc_sharpedge_size=5120, num_latents=512).queries() == 512
    assert e(pc_size=400, pc_sharpedge_size=0).plan() == ((320, 0.05, 16), (0, None, 0))
    with pytest.raises(ValueError, match="pc_size"):        # a 200-point subset of 100 points
        e(pc_size=100, pc_sharpedge_size=60).plan()
    with pytest.raises(NotImplementedError, match="normal_pe"):
        e(normal_pe=True)


def test_reference_refuses_a_subset_larger_than_its_part():
    """The reference views the subset of a too-small part as the nominal size and fails; r3g's plan() refuses it."""
    import ref_import
    if not ref_import.available():
        pytest.skip("the reference checkout is not present")
    import make_golden_encoder as M
    cfg = dict(M.BASE, pc_size=100, pc_sharpedge_size=60, num_latents=16, layers=1, qk_norm=False, qkv_bias=True,
               include_pi=False, seed=1)
    _, enc, _, _, _ = M.reference_encoder(cfg)
    with pytest.raises(RuntimeError, match="invalid for input"):
        enc(torch.zeros(1, 160, 3), torch.zeros(1, 160, 3))


def test_encoder_checkpoint_loads_strictly_and_decoder_only_still_loads():
    from r3g.vae import ShapeVAE
    z = np.load(FIXTURE)
    kw, sd, surface, _ = case(z, "split")
    vae, full = cpu_vae(kw, sd)
    assert vae.has_encoder and vae.w["pre_kl.weight"].shape == (32, 128)
    assert vae.encoder.w["input_proj.weight"].shape == (128, 64)       # K = 51 + 3 padded to 64
    # r3g's own seeded encoder weights have the reference's keys and shapes
    mine = ShapeVAE(device="cpu", **kw).init_random(1, encoder=True).reference_state_dict()
    assert {k: tuple(v.shape) for k, v in mine.items() if k.startswith(("encoder.", "pre_kl."))} == \
        {k: tuple(v.shape) for k, v in sd.items()}
    with pytest.raises(RuntimeError, match="unexpected"):
        ShapeVAE(device="cpu", **kw).load_state_dict(dict(full, **{"encoder.extra.weight": torch.zeros(1)}),
                                                      strict=True)
    with pytest.raises(KeyError):
        ShapeVAE(device="cpu", **kw).load_state_dict({k: v for k, v in full.items() if k != "pre_kl.bias"})
    dec_only = {k: v for k, v in full.items() if not k.startswith(("encoder.", "pre_kl."))}
    vae2 = ShapeVAE(device="cpu", **kw).load_state_dict(dec_only)
    assert not vae2.has_encoder and "pre_kl.weight" not in vae2.w
    with pytest.raises(RuntimeError, match="encoder"):
        ShapeVAE(device="cpu", **kw).load_state_dict(dec_only, strict=True)
    with pytest.raises(RuntimeError, match="withencoder"):
        vae2.encode(surface.half())
    with pytest.raises(TypeError, match="float16"):
        vae.encode(surface.float())


def test_from_pretrained_resolves_the_withencoder_subfolder(tmp_path, monkeypatch):
    import yaml
    from r3g.pipelines import HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG as CFG
    from r3g.vae import ShapeVAE
    kw = dict(CFG, width=128, heads=2, num_decoder_layers=1, num_encoder_layers=1, num_latents=16, pc_size=160,
              pc_sharpedge_size=160)
    sd = ShapeVAE(device="cpu", **kw).init_random(3, encoder=True).reference_state_dict()
    d = tmp_path / "tencent" / "Hunyuan3D-2mini" / "hunyuan3d-vae-v2-mini-withencoder"
    d.mkdir(parents=True)
    torch.save(sd, d / "model.fp16.ckpt")
    (d / "config.yaml").write_text(yaml.safe_dump(
        {"target": "hy3dgen.shapegen.models.ShapeVAE", "params": dict(kw, num_decoder_layers=4)}))
    monkeypatch.setenv("HY3DGEN_MODELS", str(tmp_path))
    vae = ShapeVAE.from_pretrained("tencent/Hunyuan3D-2mini", subfolder="hunyuan3d-vae-v2-mini-withencoder",
                                   use_safetensors=False, device="cpu", num_decoder_layers=1)   # kwargs win
    assert vae.has_encoder and vae.layers == 1 and vae.encoder.queries() == 16
    assert torch.equal(vae.w["pre_kl.weight"], sd["pre_kl.weight"])
    with pytest.raises(FileNotFoundError):
        ShapeVAE.from_pretrained("tencent/Hunyuan3D-2mini", subfolder="missing", device="cpu")


def test_withencoder_config_builds():
    from r3g.pipelines import HUNYUAN3D_2MINI_CONFIG, HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG as CFG
    from r3g.vae import ShapeVAE
    vae = ShapeVAE(device="cpu", **CFG)
    assert vae.encoder.plan() == ((5120, 0.05, 256), (5120, 0.05, 256))
    assert vae.encoder.layers == 8 and vae.latent_shape == (512, 64)
    assert {k: v for k, v in CFG.items() if k in HUNYUAN3D_2MINI_CONFIG["vae"]} == HUNYUAN3D_2MINI_CONFIG["vae"]
