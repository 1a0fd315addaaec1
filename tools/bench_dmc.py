#!/usr/bin/env python
"""Device-event time of the two surface extractors on the same grids, in one process: ops.marching_cubes (Lewiner, with
the bounds rescale MCSurfaceExtractor applies) against ops.dual_marching_cubes, called alternately after warm-up.
Grids: a torus at 257^3 and 513^3, and the 257^3 dense decode (octree_resolution 256) of a from_random pipeline with
the Hunyuan3D-2 geometry.  Each call includes the count pass, its one host synchronisation and the output allocation.
Prints one JSON line with V / F and the median and spread per extractor and grid, and the card's name and power limit
read in the same run.

    python tools/bench_dmc.py [--reps 10]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "3d-re-gen_b200"), os.path.dirname(os.path.abspath(__file__))):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_decimate import card  # noqa: E402


def torus_grid(n, device):
    ax = torch.linspace(-1.01, 1.01, n, device=device)
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    return (0.25 - torch.sqrt((torch.sqrt(x * x + y * y) - 0.6) ** 2 + z * z)).contiguous()


def decoded_grid(device):
    """The dense 257^3 logit grid of a random-weight Hunyuan3D-2 pipeline (3 denoising steps, random conditioning)."""
    from r3g.pipelines import Hunyuan3DDiTFlowMatchingPipeline
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, conditioner=None, device=device)
    gen = torch.Generator().manual_seed(1)
    cond = torch.randn(1, 1370, 1536, generator=gen)
    cond = {"main": torch.cat([cond, torch.zeros_like(cond)]).to(device).half()}
    pipe(cond=cond, generator=torch.manual_seed(2), num_inference_steps=3, octree_resolution=256, output_type="mesh",
         num_chunks=16000, enable_pbar=False)
    return pipe.last_grid[0].float().contiguous()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_dmc needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from r3g import ops
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = card()
    bounds = [-1.01] * 3 + [1.01] * 3
    extractors = {"mc": lambda grid: ops.marching_cubes(grid, 0.0, bounds=bounds),
                  "dmc": lambda grid: ops.dual_marching_cubes(grid)}
    result = {"metric": "surface_extraction_ms", "gpu": name, "power_limit": power, "grids": []}
    grids = [("torus257", lambda: torus_grid(257, dev)), ("torus513", lambda: torus_grid(513, dev)),
             ("decode257", lambda: decoded_grid(dev))]
    for gname, make in grids:
        grid = make()
        row = {"grid": gname, "shape": list(grid.shape)}
        for key, fn in extractors.items():         # warm-up: module load, workspace, allocator blocks
            for _ in range(2):
                v, f = fn(grid)
            row[key] = {"V": int(v.shape[0]), "F": int(f.shape[0])}
        times = {key: [] for key in extractors}
        for _ in range(args.reps):
            for key, fn in extractors.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn(grid)
                b.record()
                torch.cuda.synchronize()
                times[key].append(a.elapsed_time(b))
        for key, ts in times.items():
            row[key].update(ms_median=round(float(np.median(ts)), 3), ms_min=round(min(ts), 3),
                            ms_max=round(max(ts), 3))
        result["grids"].append(row)
        del grid
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
