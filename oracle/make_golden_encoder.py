#!/usr/bin/env python
"""ORACLE -- test infrastructure only.

Generates tests/golden/vae_encoder_mini.npz by running the REFERENCE's own PointCrossAttentionEncoder
(Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/attention_blocks.py) and a pre_kl Linear in float32 on the CPU.
Run in the build container only:
    python oracle/make_golden_encoder.py

torch_cluster is not installed: its fps is the FpsStub of vae_encoder_ref.py, which records the start index of every
batch segment and its picks.  torch.randperm is wrapped to record the two permutations.  DiagonalGaussianDistribution
lives in model.py, whose imports (skimage, the package's utils) are not available here; its arithmetic (chunk,
clamp(-30, 20), mean + exp(0.5 logvar) * noise) is restated below, with the fp16-valued noise recorded.

Geometries (width 128, 2 heads, 8 Fourier frequencies, 3 point features):
  split    a 300 / 200 random / sharp-edge split, 16 latents -> 10 + 7 = 17 queries (the reference's ceil), B = 2,
           2 self-attention layers, qk_norm, qkv_bias
  nosharp  pc_sharpedge_size = 0, 8 latents, B = 1, 1 layer, no qk_norm, no qkv_bias
  full     a 160 / 160 split, 16 latents: each subset is its whole part, B = 2, 1 layer, qk_norm
Weights are regenerated from the key names, shapes and a seed (hy3d_mini_ref.mini_state_dict).
"""
import os
import sys
import types

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_import  # noqa: E402
import vae_encoder_ref as V  # noqa: E402
from hy3d_mini_ref import mini_state_dict  # noqa: E402

OUT = os.path.join(os.path.dirname(HERE), "tests", "golden", "vae_encoder_mini.npz")
BASE = dict(width=128, heads=2, num_freqs=8, point_feats=3, downsample_ratio=20, use_ln_post=True, embed_dim=16)
GEOMETRIES = {
    "split": dict(pc_size=300, pc_sharpedge_size=200, num_latents=16, B=2, layers=2, qk_norm=True, qkv_bias=True,
                  include_pi=False, seed=21),
    "nosharp": dict(pc_size=200, pc_sharpedge_size=0, num_latents=8, B=1, layers=1, qk_norm=False, qkv_bias=False,
                    include_pi=False, seed=22),
    "full": dict(pc_size=160, pc_sharpedge_size=160, num_latents=16, B=2, layers=1, qk_norm=True, qkv_bias=True,
                 include_pi=False, seed=23),
}
INT_KEYS = ("pc_size", "pc_sharpedge_size", "num_latents", "B", "layers", "qk_norm", "qkv_bias", "include_pi", "seed")


def reference_encoder(cfg):
    """(reference PointCrossAttentionEncoder, pre_kl) with the fixture's weights, and its state-dict keys / shapes
    as a ShapeVAE holds them (encoder.* and pre_kl.*)."""
    ab, _, _ = ref_import.hunyuan_autoencoders()
    fe = ab.FourierEmbedder(num_freqs=cfg["num_freqs"], include_pi=cfg["include_pi"])
    enc = ab.PointCrossAttentionEncoder(
        fourier_embedder=fe, num_latents=cfg["num_latents"], downsample_ratio=cfg["downsample_ratio"],
        pc_size=cfg["pc_size"], pc_sharpedge_size=cfg["pc_sharpedge_size"], point_feats=cfg["point_feats"],
        width=cfg["width"], heads=cfg["heads"], layers=cfg["layers"], qkv_bias=cfg["qkv_bias"],
        use_ln_post=cfg["use_ln_post"], qk_norm=cfg["qk_norm"]).eval()
    pre_kl = nn.Linear(cfg["width"], 2 * cfg["embed_dim"])
    sd = {"encoder." + k: v for k, v in enc.state_dict().items()}
    sd.update({"pre_kl." + k: v for k, v in pre_kl.state_dict().items()})
    keys = list(sd)
    shapes = [tuple(sd[k].shape) for k in keys]
    w = mini_state_dict(keys, shapes, cfg["seed"])
    enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items() if k.startswith("encoder.")}, strict=True)
    pre_kl.load_state_dict({k[len("pre_kl."):]: v for k, v in w.items() if k.startswith("pre_kl.")}, strict=True)
    return ab, enc, pre_kl, keys, shapes


def golden(name, geo):
    cfg = dict(BASE, **geo)
    ab, enc, pre_kl, keys, shapes = reference_encoder(cfg)
    g = torch.Generator().manual_seed(cfg["seed"])
    B, N = cfg["B"], cfg["pc_size"] + cfg["pc_sharpedge_size"]
    xyz = torch.rand(B, N, 3, generator=g) * 2 - 1
    nrm = torch.nn.functional.normalize(torch.randn(B, N, 3, generator=g), dim=-1)
    surface = torch.cat([xyz, nrm], -1).half().float()
    stub = V.FpsStub()
    perms = []
    randperm = torch.randperm

    def recording_randperm(*a, **k):
        perms.append(randperm(*a, **k))
        return perms[-1]
    tc = types.ModuleType("torch_cluster")
    tc.fps = stub
    saved = sys.modules.get("torch_cluster")
    sys.modules["torch_cluster"] = tc
    torch.randperm = recording_randperm
    try:
        torch.manual_seed(cfg["seed"])
        with torch.no_grad():
            latents, _ = enc(surface[..., :3], surface[..., 3:])
            moments = pre_kl(latents)
    finally:
        torch.randperm = randperm
        if saved is None:
            del sys.modules["torch_cluster"]
        else:
            sys.modules["torch_cluster"] = saved
    mean, logvar = torch.chunk(moments, 2, dim=-1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    noise = torch.randn(mean.shape, generator=g).half().float()
    sample = mean + torch.exp(0.5 * logvar) * noise
    width = max(len(s) for s in shapes)
    d = {f"{name}_w_keys": np.array(keys),
         f"{name}_w_shapes": np.array([list(s) + [0] * (width - len(s)) for s in shapes]),
         f"{name}_surface": surface.half().numpy(), f"{name}_noise": noise.half().numpy(),
         f"{name}_mean": mean.numpy(), f"{name}_logvar": logvar.numpy(), f"{name}_sample": sample.numpy()}
    for k in INT_KEYS:
        d[f"{name}_{k}"] = np.int64(cfg[k])
    parts = ("r", "s")
    empty = np.zeros(0, dtype=np.int64)
    for i, part in enumerate(parts):
        d[f"{name}_perm_{part}"] = perms[i].numpy() if i < len(perms) else empty
        d[f"{name}_start_{part}"] = stub.calls[i][0].numpy() if i < len(stub.calls) else np.zeros(B, np.int64)
        d[f"{name}_fps_{part}"] = stub.calls[i][1].numpy() if i < len(stub.calls) else empty
    return d


def generate(path=OUT):
    torch.set_num_threads(4)
    d = {}
    for name, geo in GEOMETRIES.items():
        d.update(golden(name, geo))
    np.savez_compressed(path, **d)
    return d


if __name__ == "__main__":
    assert ref_import.available(), "reference checkout not found"
    d = generate()
    print("vae_encoder_mini:", {k: v.shape for k, v in d.items() if k.endswith(("_mean", "_fps_r", "_fps_s"))})
