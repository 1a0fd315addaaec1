#!/usr/bin/env python
"""Per-phase latency of the multi-view shape model (Hunyuan3D-2mv architecture, random weights) for V = 1 .. 4 views,
in one process with the view counts alternated object by object (so that clock and neighbour drift hit all alike).

Each object is `pipe(image={tag: crop, ...}, num_inference_steps=50, octree_resolution=256, num_chunks=16000)`: 50
classifier-free-guidance steps on a context of V * 1370 rows (the unconditional sample collapsed to one text row), the
257^3 dense decode and marching cubes.  pipe.timings gives cond / denoise / vae / decode / mc in device events.  The
executed DiT FLOP/s counts what the kernels run: the conditional sample's full forward plus the collapsed unconditional
one (Li + 1 query rows over all L keys), per step.  The card's name and power limit are read in the same run.

    python tools/bench_multiview.py [--objects 3] [--out <dir>]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))

KEYS = ("cond_ms", "denoise_ms", "vae_ms", "decode_ms", "mc_ms")
TAGS = ("front", "left", "back", "right")


def card():
    import torch
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as e:          # the times are still reported; the card line says why it is missing
        return torch.cuda.get_device_name(0), f"unknown ({e})"


def executed_dit_flops(m, Li, Lt):
    """One CFG step: the conditional forward in full, the unconditional one on Li + 1 query rows (its GEMMs and
    attention queries) with attention over all Li + Lt keys; both embed all Lt context rows."""
    H, Mh = m.hidden_size, m.mlp_hidden
    L, Lq = Li + Lt, Li + 1
    per_tok = 2 * (3 * H * H + H * H + 2 * H * Mh)
    blocks = m.depth + m.depth_single_blocks
    uncond = blocks * (per_tok * Lq + 4 * Lq * L * H) + 2 * Li * m.in_channels * H * 2 + 2 * Lt * m.context_in_dim * H
    return m.flops_per_sample(Li, Lt) + uncond


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--objects", type=int, default=3, help="timed objects per view count (after one warm-up each)")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for bench_multiview.json")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiview needs a CUDA device")
    import bench
    import __graft_entry__ as g
    g.build()
    from r3g.pipelines import HUNYUAN3D_2MV_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    name, power = card()
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2MV_CONFIG)
    kw = dict(num_inference_steps=args.steps, octree_resolution=256, num_chunks=16000, guidance_scale=5.0)
    rec = {V: [] for V in (1, 2, 3, 4)}
    for i in range(args.objects + 1):
        for V in rec:
            views = {tag: bench.synthetic_crop(1000 * i + 10 * V + j) for j, tag in enumerate(TAGS[:V])}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mesh = pipe(image=views, generator=torch.manual_seed(1234567 + i), output_type="mesh", enable_pbar=False,
                        **kw)[0]
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if i:              # object 0 of each view count is the warm-up (graph capture, workspaces)
                rec[V].append(dict(seconds=dt, faces=0 if mesh is None else int(len(mesh.mesh_f)),
                                   **{k: pipe.timings[k] for k in KEYS}))
    result = {"metric": "multiview_object_ms", "gpu": name, "power_limit": power, "steps": args.steps,
              "objects_per_view_count": args.objects, "views": {}}
    Li = pipe.vae.latent_shape[0]
    for V, rows in rec.items():
        med = {k: statistics.median(r[k] for r in rows) for k in KEYS}
        fl = args.steps * executed_dit_flops(pipe.model, Li, V * 1370)
        result["views"][V] = dict(context_rows=V * 1370, median_seconds=statistics.median(r["seconds"] for r in rows),
                                  median_timings_ms=med, dit_executed_tflop=fl / 1e12,
                                  dit_executed_tflops_per_s=fl / (med["denoise_ms"] * 1e-3) / 1e12,
                                  faces=[r["faces"] for r in rows])
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_multiview.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
