"""Whole-call marching-cubes timings on the GPU, on a sparse surface (torus) and on a dense, noise-like one, at the
metric's 257^3 and at 513^3.  Prints one JSON line; tools/mc_launch_summary.py splits a call by kernel from an ncu run.

    python tools/mc_probe.py > gpurun_out/mc_probe.json
"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))


def volumes(n):
    ax = torch.linspace(-1.01, 1.01, n, device="cuda")
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    yield "torus", (0.25 - torch.sqrt((torch.sqrt(x * x + y * y) - 0.6) ** 2 + z * z)).contiguous()
    k = 0.16 * n          # ~ n/12 periods per axis: a dense sheet structure, millions of vertices
    yield "dense", (torch.sin(k * x) * torch.sin(k * y) + torch.sin(k * y) * torch.sin(k * z)
                    + torch.sin(k * z) * torch.sin(k * x) + 0.1).contiguous()


def main():
    from r3g import ops
    out = []
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for n in (257, 513):
        for name, vol in volumes(n):
            v, f = ops.marching_cubes(vol, 0.0)         # warm-up: workspace, output blocks in the caching allocator
            ts = []
            for _ in range(7):
                flush.zero_()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                v, f = ops.marching_cubes(vol, 0.0)
                torch.cuda.synchronize()
                ts.append(1e3 * (time.perf_counter() - t0))
            ts.sort()
            nbytes = n ** 3 * 4 + v.numel() * 4 + f.numel() * 4      # algorithmic: grid once + outputs once
            out.append(dict(n=n, volume=name, ms_median=ts[len(ts) // 2], ms_min=ts[0], verts=len(v), faces=len(f),
                            algorithmic_mb=nbytes / 1e6, gbs=nbytes / ts[len(ts) // 2] / 1e6))
            print(out[-1], file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
