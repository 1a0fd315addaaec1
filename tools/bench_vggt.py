#!/usr/bin/env python
"""BASELINE.json config 4: VGGT aggregator forward (S=2 frames at 518x518, the resolution the stage runs the model
at) + point-cloud back-projection, 1 x H100.  Random weights of the VGGT-1B aggregator geometry (no checkpoint
is reachable).  Prints one JSON object; the back-projection number is HBM GB/s on the [64,1022,1022] stress shape."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from r3g import ops  # noqa: E402
from r3g.vggt import Aggregator  # noqa: E402


def rand_block(sd, p, C, g, qk):
    for n, shp in (("attn.qkv", (3 * C, C)), ("attn.proj", (C, C)), ("mlp.fc1", (4 * C, C)), ("mlp.fc2", (C, 4 * C))):
        sd[p + n + ".weight"] = torch.randn(*shp, generator=g) * 0.02
        sd[p + n + ".bias"] = torch.randn(shp[0], generator=g) * 0.02
    for n in ("norm1", "norm2"):
        sd[p + n + ".weight"], sd[p + n + ".bias"] = torch.ones(C), torch.zeros(C)
    if qk:
        for n in ("attn.q_norm", "attn.k_norm"):
            sd[p + n + ".weight"], sd[p + n + ".bias"] = torch.ones(64), torch.zeros(64)
    sd[p + "ls1.gamma"], sd[p + "ls2.gamma"] = torch.full((C,), 0.1), torch.full((C,), 0.1)


def main():
    g = torch.Generator().manual_seed(0)
    C, depth = 1024, 24
    sd = {"camera_token": torch.randn(1, 2, 1, C, generator=g) * 0.02,
          "register_token": torch.randn(1, 2, 4, C, generator=g) * 0.02,
          "patch_embed.patch_embed.proj.weight": torch.randn(C, 3, 14, 14, generator=g) * 0.02,
          "patch_embed.patch_embed.proj.bias": torch.zeros(C),
          "patch_embed.cls_token": torch.randn(1, 1, C, generator=g) * 0.02,
          "patch_embed.pos_embed": torch.randn(1, 1370, C, generator=g) * 0.02,
          "patch_embed.register_tokens": torch.randn(1, 4, C, generator=g) * 0.02,
          "patch_embed.norm.weight": torch.ones(C), "patch_embed.norm.bias": torch.zeros(C)}
    for i in range(24):
        rand_block(sd, f"patch_embed.blocks.{i}.", C, g, False)
    for i in range(depth):
        rand_block(sd, f"frame_blocks.{i}.", C, g, True)
        rand_block(sd, f"global_blocks.{i}.", C, g, True)
    agg = Aggregator().load_state_dict(sd)
    S = 2
    imgs = torch.rand(1, S, 3, 518, 518, device="cuda")

    def timed(fn, iters=5, warm=2):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / iters

    ms_agg = timed(lambda: agg(imgs))
    P = 1374
    blocks = 24 + 2 * depth
    fl = S * P * 24 * C * C * blocks + 4 * C * (24 * S * P * P + depth * S * P * P + depth * (S * P) ** 2)
    rng = np.random.default_rng(0)
    Sx, H, W = 64, 1022, 1022
    depth_map = torch.rand(Sx, H, W, device="cuda") + 0.5
    q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
    E = np.tile(np.concatenate([q, rng.normal(size=(3, 1))], 1).astype(np.float32), (Sx, 1, 1))
    K = np.tile(np.array([[800, 0, 511], [0, 800, 511], [0, 0, 1]], np.float32), (Sx, 1, 1))
    ms64 = timed(lambda: ops.unproject(depth_map, E, K, torch.float64))
    ms32 = timed(lambda: ops.unproject(depth_map, E, K, torch.float32))
    d2 = torch.rand(2, 518, 518, device="cuda") + 0.5
    ms_small = timed(lambda: ops.unproject(d2, E[:2], K[:2], torch.float64), iters=20)
    px = Sx * H * W
    pk = bench.peaks()
    print(json.dumps({
        "config": "VGGT aggregator (DINOv2-L patch embed + 24 frame + 24 global blocks) S=2 @518^2, fp16 operands / fp32 residual",
        "aggregator_ms": ms_agg, "aggregator_algorithmic_tflop": fl / 1e12, "aggregator_tflops": fl / ms_agg / 1e9,
        "published_h100_fa3_aggregator_ms_2_frames": 50.0,
        "unproject_f64_stress_ms": ms64, "unproject_f64_GBps": px * 28 / ms64 / 1e6,
        "unproject_f32_stress_ms": ms32, "unproject_f32_GBps": px * 16 / ms32 / 1e6,
        "unproject_2x518x518_f64_ms": ms_small, "hbm_peak_GBps": pk["hbm"], "peak_source": pk["source"]}))


if __name__ == "__main__":
    main()
