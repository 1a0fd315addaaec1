#!/usr/bin/env python
"""Objects per second of the base Hunyuan3D-2 shape model against the guidance-distilled one, in one process with the
configurations alternated object by object (so that clock and neighbour drift hit all of them alike):

  base       hunyuan3d-dit-v2-0: 50 classifier-free-guidance steps (two samples per DiT step), 257^3 dense decode
  distilled  the -turbo architecture (guidance_in + consistency scheduler) at the stage's settings: 5 steps, one
             sample per step, 257^3 dense decode, num_chunks 16000
  turbo      the same model at examples/fast_shape_gen_with_flashvdm.py's settings: 5 steps, FlashVDM, octree 380

Each object is `pipe(image=<512x512 RGBA crop>, ..., output_type="mesh")` timed from the call to the mesh on the host;
pipe.timings splits it into cond / denoise / vae / decode / mc (device events).  Weights are random: FlashVDM's work
depends on the near-surface band of the SDF, so the turbo row's decode time says little about real objects.

    python tools/bench_distilled.py --out <dir> [--objects 5]
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


def gpu_details():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(zip(q.split(","), [s.strip() for s in out.stdout.splitlines()[0].split(",")])) if out.stdout else {}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True, help="directory for bench_distilled.json")
    ap.add_argument("--objects", type=int, default=5, help="timed objects per configuration (after one warm-up each)")
    args = ap.parse_args()
    import torch
    import bench
    import __graft_entry__ as g
    g.build()
    from r3g.pipelines import HUNYUAN3D_2_TURBO_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    if not torch.cuda.is_available():
        raise SystemExit("bench_distilled needs a CUDA device")
    base = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0)
    dist = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2_TURBO_CONFIG)
    configs = {
        "base": (base, False, dict(num_inference_steps=50, octree_resolution=256, num_chunks=16000)),
        "distilled": (dist, False, dict(num_inference_steps=5, octree_resolution=256, num_chunks=16000)),
        "turbo": (dist, True, dict(num_inference_steps=5, octree_resolution=380, num_chunks=16000)),
    }
    crops = [bench.synthetic_crop(1234567 + i) for i in range(args.objects + 1)]
    rec = {name: [] for name in configs}
    for i, crop in enumerate(crops):
        for name, (pipe, flashvdm, kw) in configs.items():
            if flashvdm:
                pipe.enable_flashvdm()
            else:
                pipe.disable_flashvdm()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            mesh = pipe(image=crop, generator=torch.manual_seed(1234567 + i), output_type="mesh", enable_pbar=False,
                        **kw)[0]
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            faces = 0 if mesh is None else int(len(mesh.mesh_f))
            if i:              # object 0 of each configuration is the warm-up (graph capture, workspaces)
                rec[name].append(dict(seconds=dt, faces=faces, **{k: pipe.timings[k] for k in KEYS}))
    result = {"gpu": gpu_details(), "objects_per_config": args.objects, "configs": {}}
    for name, (_, flashvdm, kw) in configs.items():
        rows = rec[name]
        med = {k: statistics.median(r[k] for r in rows) for k in KEYS}
        sec = statistics.median(r["seconds"] for r in rows)
        result["configs"][name] = dict(settings=dict(kw, flashvdm=flashvdm), objects_per_s=1.0 / sec,
                                       median_seconds=sec, median_timings_ms=med, faces=[r["faces"] for r in rows],
                                       per_object=rows)
        print(f"{name:9s} {1.0 / sec:6.3f} objects/s  " + "  ".join(f"{k} {med[k]:8.1f}" for k in KEYS))
    b, d = result["configs"]["base"], result["configs"]["distilled"]
    result["denoise_ratio_base_over_distilled"] = b["median_timings_ms"]["denoise_ms"] / d["median_timings_ms"]["denoise_ms"]
    print("gpu:", result["gpu"], " denoise base / distilled:", round(result["denoise_ratio_base_over_distilled"], 2))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bench_distilled.json"), "w") as fh:
        json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
