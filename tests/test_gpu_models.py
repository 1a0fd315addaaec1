"""GPU: the DiT / ShapeVAE / geo-decoder mirrors (fp16 storage, fp32 accumulate on wgmma) against
 (a) the fixtures produced by the REFERENCE's own modules (fp32, fp16-rounded weights), and
 (b) the fp32 oracle restatement run on the same device at the reference's full widths.
Tolerances (stated, not bit-exact -- fp16 activations): relative L2 of hidden states <= 3e-3 per block tap,
<= 1e-2 for the DiT output / SDF grid; SDF sign agreement reported separately."""
import gc
import os
import weakref

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def load(golden_dir, name):
    z = np.load(os.path.join(golden_dir, name))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    return z, sd


def test_dit_mini_against_reference_fixture(golden_dir):
    from r3g.dit import Hunyuan3DDiT
    z, sd = load(golden_dir, "dit_mini.npz")
    m = Hunyuan3DDiT(in_channels=64, context_in_dim=96, hidden_size=128, num_heads=2, depth=2, depth_single_blocks=2)
    m.load_state_dict(sd)
    m.taps = []
    x = torch.from_numpy(z["x"]).cuda().half()
    t = torch.from_numpy(z["t"]).cuda().half()
    c = torch.from_numpy(z["cond"]).cuda().half()
    y = m(x, t, {"main": c}).float().cpu()
    for i, tp in enumerate(m.taps):
        e = rel_l2(tp.cpu(), torch.from_numpy(z[f"tap{i}"]))
        assert e < 3e-3, f"tap {i}: rel L2 {e}"
    e = rel_l2(y, torch.from_numpy(z["y"]))
    assert e < 1e-2, f"output rel L2 {e}"


def test_dit_full_width_blocks_against_oracle():
    """hidden 1024 / 16 heads / L = 1370 + 3072 (the real geometry), 1 double + 2 single blocks, B = 2."""
    import hy3d_ref as R
    from r3g.dit import Hunyuan3DDiT
    m = Hunyuan3DDiT(depth=1, depth_single_blocks=2).init_random(seed=3)
    m.taps = []
    torch.manual_seed(0)
    x = torch.randn(2, 3072, 64, device="cuda").half()
    c = torch.randn(2, 1370, 1536, device="cuda").half()
    t = torch.tensor([0.5102, 0.5102], device="cuda").half()
    y = m(x, t, {"main": c})
    sd = {k: v.float().cuda() for k, v in m.reference_state_dict().items()}
    taps = []
    ref = R.dit_forward(sd, x.float(), t.float(), c.float(), 16, 1, 2, taps=taps)
    for i, (a, b) in enumerate(zip(m.taps, taps)):
        e = rel_l2(a, b)
        assert e < 3e-3, f"tap {i}: rel L2 {e}"
    assert rel_l2(y, ref) < 1e-2


def test_vae_and_sdf_grid_against_reference_fixture(golden_dir):
    from r3g.vae import ShapeVAE
    z, sd = load(golden_dir, "vae_mini.npz")
    heads, layers, Rr = int(z["cfg_heads"]), int(z["cfg_layers"]), int(z["cfg_R"])
    vae = ShapeVAE(num_latents=48, embed_dim=64, width=128, heads=heads, num_decoder_layers=layers, num_freqs=8,
                   include_pi=False, qkv_bias=False, qk_norm=True)
    vae.load_state_dict(sd)
    vae.taps = []
    lat = vae(torch.from_numpy(z["z"]).cuda().half())
    for i, tp in enumerate(vae.taps):
        assert rel_l2(tp.cpu(), torch.from_numpy(z[f"tap{i}"])[0]) < 3e-3
    assert rel_l2(lat.cpu(), torch.from_numpy(z["latents"])) < 3e-3
    # decode from the fixture's latents so the grid comparison isolates the geo-decoder
    lat_ref = torch.from_numpy(z["latents"]).cuda().half()
    grid = vae.volume_decoder(lat_ref, vae.geo_decoder, bounds=1.01, num_chunks=100, octree_resolution=Rr)
    g, gr = grid.cpu(), torch.from_numpy(z["grid"])
    assert g.shape == gr.shape and g.dtype == torch.float32
    assert (g - gr).abs().max().item() < 1e-2 * gr.abs().max().item()
    confident = gr.abs() > 1e-2 * gr.abs().max()
    assert (torch.sign(g[confident]) == torch.sign(gr[confident])).all()
    # explicit-query call form of the plug point
    q = torch.from_numpy(z["xyz"]).cuda().half()[None]
    geo = vae.geo_decoder
    captured = [weakref.ref(t) for t in next(iter(geo._ws.values())).values()]
    lg = geo(queries=q, latents=lat_ref)
    assert lg.shape == (1, q.shape[1], 1)
    assert torch.equal(lg.view(-1).float().cpu(), g.view(-1))
    # fewer queries size a smaller workspace, which replaces the one the grid's graph was captured with
    geo(queries=q[:, :100], latents=lat_ref)
    gc.collect()
    assert all(r() is not None for r in captured), "the graph must keep its captured workspace alive"
    again = vae.volume_decoder(lat_ref, geo, bounds=1.01, num_chunks=100, octree_resolution=Rr)
    geo.use_cuda_graph = False
    eager = vae.volume_decoder(lat_ref, geo, bounds=1.01, num_chunks=100, octree_resolution=Rr)
    assert torch.equal(again, grid) and torch.equal(eager, grid), "graph replay must equal the eager launches"


def test_sdf_decode_full_width_against_oracle():
    """width 1024 / 16 heads / 3072 latents, 33^3 grid: logits vs the fp32 oracle, and the meshes they give."""
    import hy3d_ref as R
    from r3g.vae import ShapeVAE
    vae = ShapeVAE(num_latents=3072, embed_dim=64, width=1024, heads=16, num_decoder_layers=1, num_freqs=8,
                   include_pi=False, qkv_bias=False, qk_norm=True).init_random(seed=5)
    torch.manual_seed(1)
    lat = (torch.randn(1, 3072, 1024, device="cuda") * 0.5).half()
    Rr = 32
    grid = vae.volume_decoder(lat, vae.geo_decoder, bounds=1.01, octree_resolution=Rr)
    sd = {k: v.float().cuda() for k, v in vae.reference_state_dict().items()}
    ref = R.vanilla_volume_decode(sd, lat.float(), 16, Rr, num_chunks=8192)
    scale = ref.abs().max().item()
    err = (grid - ref).abs().max().item()
    assert err < 1e-2 * scale, f"SDF abs err {err} vs scale {scale}"
    confident = ref.abs() > 2e-2 * scale
    agree = (torch.sign(grid[confident]) == torch.sign(ref[confident])).float().mean().item()
    assert agree == 1.0
    outs = vae.surface_extractor(grid, mc_level=0.0, bounds=1.01, octree_resolution=Rr)
    assert outs[0] is not None and outs[0].mesh_v.dtype == np.float32 and outs[0].mesh_f.shape[1] == 3


def test_vae_full_width_layer_against_oracle():
    import hy3d_ref as R
    from r3g.vae import ShapeVAE
    vae = ShapeVAE(num_latents=3072, embed_dim=64, width=1024, heads=16, num_decoder_layers=2, num_freqs=8,
                   include_pi=False, qkv_bias=False, qk_norm=True).init_random(seed=6)
    torch.manual_seed(2)
    zl = torch.randn(1, 3072, 64, device="cuda").half()
    out = vae(zl)
    sd = {k: v.float().cuda() for k, v in vae.reference_state_dict().items()}
    ref = R.vae_forward(sd, zl.float(), 16, 2)
    assert rel_l2(out, ref) < 3e-3


def test_conditioner_on_r3g_kernels_against_the_hf_module():
    """rows a2 / f4: the DINOv2 forward of the conditioner on the r3g kernels vs transformers' Dinov2Model (the module
    the reference runs, conditioner.py:125-131) in fp32 on the same weights; incl. a SwiGLU width that needs padding."""
    from r3g.conditioner import DinoImageEncoder
    for hidden, heads, mlp in ((192, 3, 4), (128, 2, 4)):          # SwiGLU widths 512 and 344 (padded to 352)
        cfg = dict(hidden_size=hidden, num_hidden_layers=3, num_attention_heads=heads, mlp_ratio=mlp, patch_size=14,
                   image_size=70, use_swiglu_ffn=True, layerscale_value=1.0, qkv_bias=True, hidden_act="gelu",
                   layer_norm_eps=1e-6)
        torch.manual_seed(0)
        enc = DinoImageEncoder(config=cfg, image_size=70, device="cuda", dtype=torch.float16)
        assert enc.backend == "r3g"
        with torch.no_grad():
            for n, p_ in enc.model.named_parameters():
                if "lambda1" in n:
                    p_.copy_(0.3 + 0.2 * torch.rand_like(p_))
                elif "norm" in n and n.endswith("weight"):
                    p_.copy_(1 + 0.2 * torch.randn_like(p_))
        img = torch.rand(2, 3, 90, 90) * 2 - 1
        got = enc(img)
        ref_model = type(enc.model)(enc.model.config).to("cuda").float()
        ref_model.load_state_dict({k: v.float() for k, v in enc.model.state_dict().items()})
        with torch.no_grad():
            px = enc._transform(((img + 1) / 2).cuda().half()).float()
            ref = ref_model(px).last_hidden_state
        assert got.shape == ref.shape == (2, 26, hidden) and got.dtype == torch.float16
        assert rel_l2(got, ref) < 5e-3, rel_l2(got, ref)
        enc.backend = "hf"
        assert rel_l2(enc(img), ref) < 5e-3
