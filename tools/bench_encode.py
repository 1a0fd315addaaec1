#!/usr/bin/env python
"""ShapeVAE.encode timing on the GPU: the whole encode graph, and the sampling (randperm subsets + FPS) alone in a graph
of its own; the network is the difference.  Two geometries with seeded weights: the 2mini encoder (5120 + 5120 points
-> 512 latents, HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG) and the 2.0 demo's (30720 + 30720 points -> 3072 latents).
CUDA events over `--iters` replays after a warm-up; prints one JSON line with the card's name and power limit.

    python tools/bench_encode.py [--iters 20]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))

from r3g.graphs import GraphCache  # noqa: E402
from r3g.pipelines import HUNYUAN3D_2MINI_VAE_WITHENCODER_CONFIG as MINI  # noqa: E402
from r3g.vae import ShapeVAE  # noqa: E402

GEOMETRIES = {
    "2mini_10240_to_512": dict(MINI, num_decoder_layers=1),
    "2.0_61440_to_3072": dict(MINI, num_decoder_layers=1, num_latents=3072, pc_size=30720, pc_sharpedge_size=30720),
}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def bench(kw, iters):
    vae = ShapeVAE(device="cuda", **kw).init_random(0, encoder=True)
    n = kw["pc_size"] + kw["pc_sharpedge_size"]
    g = torch.Generator().manual_seed(0)
    d = torch.nn.functional.normalize(torch.randn(1, n, 3, generator=g), dim=-1)
    surface = torch.cat([d * 0.6, d], -1).half().cuda()
    torch.manual_seed(0)
    draws = vae.encoder.draw(surface)
    noise = torch.randn(1, vae.encoder.queries(), kw["embed_dim"], device="cuda", dtype=torch.float16)
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    vae.encode_core(surface, *draws, noise=noise)           # warm-up and capture
    t1.record()
    torch.cuda.synchronize()
    entry = next(iter(vae._enc_graphs.entries.values()))
    fps = GraphCache().get("sample", (surface,) + draws, lambda s, *dr: vae.encoder.sample(s, *dr)[2])
    total_ms = timed(entry.replay, iters)
    fps_ms = timed(fps.replay, iters)
    return dict(latents=vae.encoder.queries(), points=n, encode_ms=round(total_ms, 3), fps_ms=round(fps_ms, 3),
                network_ms=round(total_ms - fps_ms, 3), first_call_ms=round(t0.elapsed_time(t1), 1),
                graph_nodes_r3g=entry.launches,
                encode_call_ms=round(timed(lambda: vae.encode_core(surface, *draws, noise=noise), iters), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_encode.py needs a CUDA device")
    out = {"card": card(), "iters": args.iters}
    for name, kw in GEOMETRIES.items():
        out[name] = bench(kw, args.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
