#!/usr/bin/env python
"""A/B of the DiT forward with and without the collapsed unconditional text (Hunyuan3DDiT.forward, uncond_txt_shared) at
the bench shape: B = 2 (cond, zeros), 1370 + 3072 tokens, 16 + 32 blocks, seeded random weights.

Both forwards are captured as CUDA graphs and replayed alternately, `--rounds` x `--reps` replays each, timed with CUDA
events; prints one JSON line with the per-forward mean, spread (min / max over rounds) and the ratio, and the output
check (the two outputs are bit-identical).  --profile DIR also writes a torch.profiler kernel table of one eager
forward per mode to DIR/prof_<mode>.txt."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
from r3g.dit import Hunyuan3DDiT  # noqa: E402
from r3g.graphs import GraphCache  # noqa: E402
from r3g.pipelines import HUNYUAN3D_2_CONFIG  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--profile", metavar="DIR", default=None)
    args = ap.parse_args()
    model = Hunyuan3DDiT(device="cuda", **HUNYUAN3D_2_CONFIG["model"]).init_random(0)
    torch.manual_seed(0)
    x = torch.randn(2, 3072, 64, device="cuda").half()
    t = torch.full((2,), 0.5, device="cuda", dtype=torch.float16)
    c = torch.cat([torch.randn(1, 1370, 1536, device="cuda"), torch.zeros(1, 1370, 1536, device="cuda")]).half()
    cache = GraphCache(keep_all=True)
    modes = {"full": False, "collapsed": True}
    graphs = {name: cache.get(flag, (x, t, c), lambda xs, ts, cs, f=flag: model(xs, ts, {"main": cs}, uncond_txt_shared=f))
              for name, flag in modes.items()}
    outs = {}
    for name, g in graphs.items():
        g.replay()
        outs[name] = g.outputs.clone()
    for _ in range(2):
        for g in graphs.values():
            g.replay()
    ms = {name: [] for name in modes}
    for _ in range(args.rounds):
        for name, g in graphs.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                g.replay()
            b.record()
            torch.cuda.synchronize()
            ms[name].append(a.elapsed_time(b) / args.reps)
    mean = {k: sum(v) / len(v) for k, v in ms.items()}
    line = {"gpu": torch.cuda.get_device_name(), "forward_ms_mean": mean,
            "forward_ms_min": {k: min(v) for k, v in ms.items()}, "forward_ms_max": {k: max(v) for k, v in ms.items()},
            "ratio_collapsed_over_full": mean["collapsed"] / mean["full"], "launches": {k: g.launches for k, g in graphs.items()},
            "outputs_equal": bool(torch.equal(outs["collapsed"], outs["full"]))}
    print(json.dumps(line))
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        os.makedirs(args.profile, exist_ok=True)
        for name, flag in modes.items():
            model(x, t, {"main": c}, uncond_txt_shared=flag)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                model(x, t, {"main": c}, uncond_txt_shared=flag)
                torch.cuda.synchronize()
            table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30)
            with open(os.path.join(args.profile, f"prof_{name}.txt"), "w") as fh:
                fh.write(table)


if __name__ == "__main__":
    main()
