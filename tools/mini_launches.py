#!/usr/bin/env python
"""Latents and kernel launches of seeded Hunyuan3D-2mini pipeline calls with CUDA graphs on: three calls with
output_type="latent" on a precomputed (random) conditioner output -- the first captures the step graph, the second
replays it on the same context, the third on another context.  Per call it records the r3g kernels launched outside
graph replays (`_abi.get_context(dev).launches`), the kernels run by replays (`replayed_launches`), the graphs captured
and a SHA-256 of the latents, and prints one JSON line with the card's name and power limit.  --out DIR also writes
each call's latents as DIR/latents_<call>.npy.  --tree runs another tree's pipeline (e.g. the parent commit extracted
into ab_parent/ and built there), so two arms can be compared bit for bit in one session:
  python tools/mini_launches.py --tree ab_parent --out a; python tools/mini_launches.py --out b"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=ROOT, help="repository tree whose pipeline runs")
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--out", default=None, help="directory for the latents of each call")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mini_launches needs a CUDA device")
    sys.path.insert(0, os.path.join(os.path.abspath(a.tree), "3d-re-gen_b200"))
    from r3g import _abi
    from r3g.pipelines import HUNYUAN3D_2MINI_CONFIG, Hunyuan3DDiTFlowMatchingPipeline
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    pipe = Hunyuan3DDiTFlowMatchingPipeline.from_random(seed=0, config=HUNYUAN3D_2MINI_CONFIG, conditioner=None)
    ctx = _abi.get_context(torch.cuda.current_device())
    calls = []
    for call, seed in enumerate((0, 0, 1)):
        main_cond = torch.randn(1, 1370, 1024, generator=torch.Generator().manual_seed(seed))
        cond = {"main": torch.cat([main_cond, torch.zeros_like(main_cond)]).cuda().half()}
        torch.cuda.synchronize()
        n0, r0, c0 = ctx.launches, pipe.replayed_launches, pipe._graphs.captures
        lat = pipe(cond=cond, num_inference_steps=a.steps, generator=torch.manual_seed(1), output_type="latent")
        torch.cuda.synchronize()
        host = lat.cpu().numpy()
        calls.append(dict(context_seed=seed, launches=ctx.launches - n0, replayed=pipe.replayed_launches - r0,
                          captures=pipe._graphs.captures - c0, latents_sha256=hashlib.sha256(host.tobytes()).hexdigest()))
        if a.out:
            import numpy as np
            os.makedirs(a.out, exist_ok=True)
            np.save(os.path.join(a.out, f"latents_{call}.npy"), host)
    print(json.dumps(dict(tree=os.path.relpath(os.path.abspath(a.tree), ROOT), steps=a.steps, calls=calls,
                          card=card[torch.cuda.current_device()] if card else "unknown")), flush=True)


if __name__ == "__main__":
    main()
