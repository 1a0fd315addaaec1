"""GPU: FlashVDMVolumeDecoding on the r3g kernels against the fixture produced by the REFERENCE class
(volume_decoders.py:280-435 + attention_processors.py:35-79, run in fp32 by oracle/make_golden.py::golden_flashvdm).
The decoder is adaptive -- which points are evaluated at the fine level depends on the coarse logits, and which keys a
bucket attends to depends on a top-k over similarities -- so fp16 storage can flip a few decisions at band / top-k
boundaries.  Stated tolerances: >= 98 % of the grid agrees on evaluated-vs-NaN, and on the points both evaluate the
logits agree to 3e-2 of the largest |logit| at the 99.5th percentile (a flipped top-k choice moves single points more),
with sign agreement >= 99.5 % on confident points."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _load(golden_dir):
    z = np.load(os.path.join(golden_dir, "flashvdm_mini.npz"))
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    return z, sd


def _vae(sd, heads):
    from r3g.vae import ShapeVAE
    vae = ShapeVAE(num_latents=48, embed_dim=64, width=128, heads=heads, num_decoder_layers=0, num_freqs=8,
                   include_pi=False, qkv_bias=False, qk_norm=True)
    vae.geo_decoder.load(sd)
    return vae


def _report(name, got, ref):
    fin_g, fin_r = torch.isfinite(got), torch.isfinite(ref)
    mask_agree = (fin_g == fin_r).float().mean().item()
    both = fin_g & fin_r
    scale = ref[fin_r].abs().max().item()
    d = (got[both] - ref[both]).abs()
    p995 = torch.quantile(d.float(), 0.995).item()
    conf = both & (ref.abs() > 2e-2 * scale)
    sign = (torch.sign(got[conf]) == torch.sign(ref[conf])).float().mean().item()
    print(f"{name}: evaluated {fin_g.float().mean().item():.4f} (reference {fin_r.float().mean().item():.4f}), mask agreement "
          f"{mask_agree:.4f}; |d| p99.5 {p995:.3e}, max {d.max().item():.3e} of scale {scale:.3e}; sign agreement {sign:.5f}")
    return mask_agree, p995 / scale, sign


def test_flashvdm_two_levels_against_reference_fixture(golden_dir):
    from r3g.vae import FlashVDMVolumeDecoding
    z, sd = _load(golden_dir)
    vae = _vae(sd, int(z["cfg_heads"]))
    lat = torch.from_numpy(z["latents"]).cuda().half()
    dec = FlashVDMVolumeDecoding("mean")
    grid = dec(lat, vae.geo_decoder, bounds=1.01, num_chunks=int(z["cfg_num_chunks"]), mc_level=0.0,
               octree_resolution=int(z["cfg_octree"]), min_resolution=int(z["cfg_min_resolution"]), enable_pbar=False)
    ref = torch.from_numpy(z["grid"])
    assert grid.shape == ref.shape and grid.dtype == torch.float16
    assert dec.stats["resolutions"] == [31, 62]
    m, e, s = _report("two levels", grid.float().cpu(), ref)
    assert m >= 0.98 and e <= 3e-2 and s >= 0.995
    # the refinement level decoded in several groups of whole buckets gives the same grid bit for bit
    assert dec.stats["groups"] == [1]
    split = FlashVDMVolumeDecoding("mean")
    split.max_group_queries = max(dec.stats["queries"][1] // 5, 1)
    grid_split = split(lat, vae.geo_decoder, bounds=1.01, num_chunks=int(z["cfg_num_chunks"]), mc_level=0.0,
                       octree_resolution=int(z["cfg_octree"]), min_resolution=int(z["cfg_min_resolution"]),
                       enable_pbar=False)
    assert split.stats["groups"][0] > 1
    assert torch.equal(grid_split.isnan(), grid.isnan()) and torch.equal(grid_split.nan_to_num(), grid.nan_to_num())
    # single dense level (every point evaluated, top-k attention per mini-grid)
    g0 = dec(lat, vae.geo_decoder, bounds=1.01, num_chunks=3000, octree_resolution=31, min_resolution=31, enable_pbar=False)
    m0, e0, s0 = _report("dense level", g0.float().cpu(), torch.from_numpy(z["grid_level0"]))
    assert m0 == 1.0 and e0 <= 3e-2 and s0 >= 0.995


def test_flashvdm_through_the_vae_plug_point_and_marching_cubes(golden_dir):
    """enable_flashvdm_decoder -> latents2mesh: NaN outside the band, marching cubes on the fp16 / NaN grid."""
    z, sd = _load(golden_dir)
    vae = _vae(sd, int(z["cfg_heads"]))
    vae.enable_flashvdm_decoder(True, adaptive_kv_selection=True, topk_mode="mean", mc_algo="mc")
    with pytest.raises(NotImplementedError):
        vae.enable_flashvdm_decoder(True, adaptive_kv_selection=False)
    lat = torch.from_numpy(z["latents"]).cuda().half()
    outs = vae.latents2mesh(lat, bounds=1.01, num_chunks=3000, mc_level=0.0, octree_resolution=64, min_resolution=31,
                            enable_pbar=False)
    assert len(outs) == 1 and outs[0] is not None and outs[0].mesh_f.shape[1] == 3
    vae.enable_flashvdm_decoder(False)
    from r3g.vae import VanillaVolumeDecoder
    assert isinstance(vae.volume_decoder, VanillaVolumeDecoder)


def test_flashvdm_full_width_evaluates_a_fraction_of_the_grid():
    """Real geometry (3072 latents, 1024 wide, top-k 1024): resolutions [63, 126, 252] for octree_resolution 256."""
    from r3g.pipelines import HUNYUAN3D_2_CONFIG
    from r3g.vae import FlashVDMVolumeDecoding, ShapeVAE
    vae = ShapeVAE(**HUNYUAN3D_2_CONFIG["vae"]).init_random(seed=5)
    torch.manual_seed(4)
    lat = (torch.randn(1, 3072, 1024, device="cuda") * 0.5).half()
    dec = FlashVDMVolumeDecoding()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    grid = dec(lat, vae.geo_decoder, bounds=1.01, octree_resolution=256, num_chunks=16000, enable_pbar=False)
    e1.record()
    torch.cuda.synchronize()
    assert dec.stats["resolutions"] == [63, 126, 252] and grid.shape == (1, 253, 253, 253)
    per_level = list(dec.stats["queries"])
    dense = vae.volume_decoder(lat, vae.geo_decoder, bounds=1.01, octree_resolution=63)
    lvl0 = dec(lat, vae.geo_decoder, bounds=1.01, octree_resolution=63, enable_pbar=False)
    scale = dense.abs().max().item()
    conf = dense.abs() > 5e-2 * scale
    agree = (torch.sign(lvl0.float()[conf]) == torch.sign(dense[conf])).float().mean().item()
    print(f"FlashVDM 252^3: {e0.elapsed_time(e1):.0f} ms, queries per level {per_level} of {253 ** 3} (a noise-like field of random weights keeps most of the volume inside the |logit| < 0.95 band); "
          f"top-1024-of-3072 attention vs full attention at 64^3: sign agreement {agree:.4f} on confident points")
    assert agree > 0.9
