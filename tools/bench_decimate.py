#!/usr/bin/env python
"""Device-event time of FaceReducerR3G (r3g_mesh_decimate) to 40 000 faces on the marching-cubes meshes of an analytic
scene (a sphere, a torus around it and a small sphere) at 257^3 and 385^3 grids, after warm-up.  Prints one JSON line with
faces in / out, rounds, the median and spread of the timed calls, and the card's name and power limit read in the same
run.  The decimator synchronises its stream once or twice per round, so the time includes those host round trips.

    python tools/bench_decimate.py [--reps 5] [--target 40000]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "3d-re-gen_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def scene_grid(n, device):
    """The field of tests/test_decimate_oracle.py::sdf_scene3 on an n^3 grid over [-1, 1]^3, built on the device."""
    ax = torch.linspace(-1, 1, n, device=device, dtype=torch.float32)
    x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
    sphere = 0.45 - torch.sqrt(x * x + y * y + (z - 0.05) ** 2)
    q = torch.sqrt(x * x + y * y) - 0.7
    torus = 0.15 - torch.sqrt(q * q + z * z)
    small = 0.12 - torch.sqrt((x - 0.75) ** 2 + (y - 0.75) ** 2 + (z - 0.6) ** 2)
    return torch.maximum(torch.maximum(sphere, torus), small).contiguous()


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:          # the time is still reported; the card line says why it is missing
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--target", type=int, default=40000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decimate needs a CUDA device")
    import __graft_entry__ as g
    g.build()
    from r3g import ops
    from r3g.postprocessors import FaceReducerR3G
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    name, power = card()
    result = {"metric": "face_reducer_r3g_ms", "target": args.target, "gpu": name, "power_limit": power, "grids": []}
    red = FaceReducerR3G()
    for n in (257, 385):
        v, f = ops.marching_cubes(scene_grid(n, dev), 0.0, bounds=[-1.0] * 3 + [1.0] * 3)
        for _ in range(2):                                      # warm-up: module load, workspace, allocator
            red((v, f), max_facenum=args.target)
        _, _, rounds = ops.mesh_decimate(v, f, args.target)
        times = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            v2, f2 = red((v, f), max_facenum=args.target)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        result["grids"].append({"grid": n, "faces_in": int(f.shape[0]), "verts_in": int(v.shape[0]),
                                "faces_out": int(f2.shape[0]), "verts_out": int(v2.shape[0]), "rounds": int(rounds),
                                "ms_median": round(float(np.median(times)), 3),
                                "ms_min": round(min(times), 3), "ms_max": round(max(times), 3)})
    print(json.dumps(result))


if __name__ == "__main__":
    main()
