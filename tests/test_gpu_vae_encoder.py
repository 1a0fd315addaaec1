"""GPU: ShapeVAE.encode on the r3g kernels -- the fixture of the reference's own encoder (tests/golden/vae_encoder_mini.npz)
on its recorded draws, the 2mini width against a float32 torch restatement, FPS at the 2.0 encoder's size against the
oracle, graph replay against eager, and minimal_vae_demo.py's call sequence on a seeded checkpoint."""
import os
import sys

import numpy as np
import pytest
import torch

from test_vae_encoder import case, ref_cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
FIXTURE = os.path.join(ROOT, "tests", "golden", "vae_encoder_mini.npz")

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm())


def gpu_vae(kw, sd):
    from r3g.vae import ShapeVAE
    full = dict(ShapeVAE(device="cpu", **kw).init_random(5).reference_state_dict())
    full.update(sd)
    return ShapeVAE(device="cuda", **kw).load_state_dict(full, strict=True)


def sphere_surface(B, n_random, n_sharp, seed=0, r=0.6):
    """Points on a sphere of radius r (uniform, then the equator for the sharp-edge part) with their outward normals,
    fp16 [B, n_random + n_sharp, 6] on cuda."""
    g = torch.Generator().manual_seed(seed)
    d = torch.nn.functional.normalize(torch.randn(B, n_random, 3, generator=g), dim=-1)
    t = torch.rand(B, n_sharp, generator=g) * 2 * torch.pi
    e = torch.stack([t.cos(), t.sin(), torch.zeros_like(t)], -1)
    n = torch.cat([d, e], 1)
    return torch.cat([n * r, n], -1).half().cuda()


@pytest.mark.parametrize("name", ["split", "nosharp", "full"])
def test_encode_core_on_the_fixture_draws(name):
    z = np.load(FIXTURE)
    kw, sd, surface, draws = case(z, name)
    vae = gpu_vae(kw, sd)
    noise = torch.from_numpy(z[f"{name}_noise"]).cuda()
    lat, mean, logvar, pick_r, pick_s = vae.encode_core(surface.half().cuda(), *(t.cuda() for t in draws), noise=noise)
    assert np.array_equal(pick_r.cpu().numpy(), z[f"{name}_fps_r"])
    assert np.array_equal(pick_s.cpu().numpy(), z[f"{name}_fps_s"])
    errs = {k: rel_l2(t, torch.from_numpy(z[f"{name}_{k}"])) for k, t in
            (("mean", mean), ("logvar", logvar), ("sample", lat))}
    print(name, errs)
    assert all(e <= 5e-3 for e in errs.values()), errs
    assert lat.dtype == torch.float16 and lat.shape == z[f"{name}_mean"].shape


def test_graph_replay_equals_eager_bit_for_bit():
    z = np.load(FIXTURE)
    kw, sd, surface, _ = case(z, "split")
    vae = gpu_vae(kw, sd)
    s = surface.half().cuda()
    for sample in (True, False):
        torch.manual_seed(7)
        draws = vae.encoder.draw(s)
        noise = torch.randn(2, vae.encoder.queries(), 16, device="cuda", dtype=torch.float16) if sample else None
        vae.use_cuda_graph = False
        eager = vae.encode_core(s, *draws, noise=noise)
        vae.use_cuda_graph = True
        for _ in range(2):      # capture, then a replay
            graph = vae.encode_core(s, *draws, noise=noise)
            assert all(torch.equal(a, b) for a, b in zip(eager, graph))
    assert vae._enc_graphs.captures == 2
    # encode() draws in the reference's order: the same seed gives the same latents, the mean without sampling
    torch.manual_seed(3)
    a = vae.encode(s)
    torch.manual_seed(3)
    assert torch.equal(a, vae.encode(s))
    torch.manual_seed(5)
    m = vae.encode(s, sample_posterior=False)
    torch.manual_seed(5)
    assert torch.equal(m, vae.encode_core(s, *vae.encoder.draw(s))[1])


def test_2mini_width_against_the_float32_restatement():
    import vae_encoder_ref as V
    from r3g.pipelines import HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG as CFG
    from r3g.vae import ShapeVAE
    kw = dict(CFG, num_decoder_layers=1)
    vae = ShapeVAE(device="cuda", **kw).init_random(11, encoder=True)
    sd = {k: v.cuda() for k, v in vae.reference_state_dict().items() if k.startswith(("encoder.", "pre_kl."))}
    s = sphere_surface(1, 5120, 5120, seed=1)
    torch.manual_seed(0)
    draws = vae.encoder.draw(s)
    _, mean, logvar, _, _ = vae.encode_core(s, *draws)
    assert mean.shape == (1, 512, 64)
    q, d, _ = vae.encoder.sample(s, *draws)
    ref = V.encoder_forward(sd, ref_cfg(kw), q, d)
    rm, rl = ref.chunk(2, -1)
    errs = rel_l2(mean, rm), rel_l2(logvar, rl.clamp(-30, 20))
    print("2mini width rel-L2 mean, logvar:", errs)
    assert max(errs) <= 1e-2, errs


def test_fps_at_the_2_0_encoder_size_matches_the_oracle():
    import vae_encoder_ref as V
    from r3g.vae import farthest_point_sample
    pts = sphere_surface(2, 30720, 0, seed=2)[..., :3].float()
    start = torch.tensor([12345, 0], device="cuda")
    got = farthest_point_sample(pts, start, 1536).cpu().numpy()
    for b in range(2):
        assert np.array_equal(got[b], V.fps_segment(pts[b].cpu().numpy(), int(start[b]), 1536)), b


def test_minimal_vae_demo_flow(tmp_path):
    """from_single_file -> encode -> decode -> latents2mesh, as minimal_vae_demo.py calls them, on a seeded checkpoint
    and a surface sampled from a sphere."""
    import yaml
    from r3g.pipelines import HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG as CFG, export_to_trimesh
    from r3g.vae import ShapeVAE
    kw = dict(CFG, width=256, heads=4, num_latents=64, num_decoder_layers=2, num_encoder_layers=2, pc_size=640,
              pc_sharpedge_size=640)
    sd = ShapeVAE(device="cpu", **kw).init_random(4, encoder=True).reference_state_dict()
    torch.save(sd, tmp_path / "model.fp16.ckpt")
    (tmp_path / "config.yaml").write_text(yaml.safe_dump({"target": "hy3dgen.shapegen.models.ShapeVAE",
                                                          "params": kw}))
    vae = ShapeVAE.from_single_file(str(tmp_path / "model.fp16.ckpt"), str(tmp_path / "config.yaml"),
                                    use_safetensors=False)
    surface = sphere_surface(1, 640, 640, seed=3)
    latents = vae.encode(surface)
    assert latents.shape == (1, 64, 64) and torch.isfinite(latents).all()
    latents = vae.decode(latents)
    assert latents.shape == (1, 64, 256) and torch.isfinite(latents).all()
    mesh = vae.latents2mesh(latents, output_type="trimesh", bounds=1.01, mc_level=0.0, num_chunks=20000,
                            octree_resolution=64, mc_algo="mc", enable_pbar=True)
    assert len(mesh) == 1
    grid = vae.volume_decoder(latents, vae.geo_decoder, bounds=1.01, octree_resolution=64)
    assert torch.isfinite(grid).all()
    if grid.min() < 0 < grid.max():     # random weights: a surface exists only where the logits change sign
        m = export_to_trimesh(mesh)[0]
        assert m is not None and len(m.faces) > 0 and m.faces.max() < len(m.vertices)
