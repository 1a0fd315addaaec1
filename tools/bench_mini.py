#!/usr/bin/env python
"""Objects/s and per-phase times of Hunyuan3D-2mini and 2mini-turbo next to the 2.0 base, on seeded random weights with
a precomputed (random) conditioner output, so that the three rows time the same phases: denoise (CFG, graph replays),
VAE forward, dense SDF decode, marching cubes.  Prints one JSON line per model with the card's name and power limit.

    python tools/bench_mini.py [--steps 50] [--turbo-steps 5] [--octree 256] [--repeat 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--turbo-steps", type=int, default=5)
    ap.add_argument("--octree", type=int, default=256)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mini needs a CUDA device")
    from r3g.pipelines import (HUNYUAN3D_2_CONFIG, HUNYUAN3D_2MINI_CONFIG, HUNYUAN3D_2MINI_TURBO_CONFIG,
                               Hunyuan3DDiTFlowMatchingPipeline)
    where = card()
    rows = (("2.0", HUNYUAN3D_2_CONFIG, 1370, 1536, a.steps), ("2mini", HUNYUAN3D_2MINI_CONFIG, 1370, 1024, a.steps),
            ("2mini-turbo", HUNYUAN3D_2MINI_TURBO_CONFIG, 1370, 1024, a.turbo_steps))
    for name, cfg, Lt, C, steps in rows:
        pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=cfg, conditioner=None)
        g = torch.Generator().manual_seed(0)
        main_cond = torch.randn(1, Lt, C, generator=g)
        cond = {"main": torch.cat([main_cond, torch.zeros_like(main_cond)]).cuda().half()}
        kw = dict(cond=cond, num_inference_steps=steps, octree_resolution=a.octree, num_chunks=20000, output_type="mesh",
                  enable_pbar=False)
        pipe(generator=torch.manual_seed(1), **kw)          # warm-up: graphs, workspaces
        times, phases = [], []
        for r in range(a.repeat):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe(generator=torch.manual_seed(1), **kw)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            phases.append({k: round(v, 2) for k, v in pipe.timings.items()})
        med = sorted(times)[len(times) // 2]
        print(json.dumps(dict(model=name, objects_per_s=round(1.0 / med, 4), seconds=[round(t, 3) for t in times],
                              steps=steps, octree=a.octree, phases_ms=phases[len(phases) // 2], card=where,
                              note="random weights, precomputed conditioner output (encoder not timed)")), flush=True)
        del pipe
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
