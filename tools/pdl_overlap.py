"""Does a chain of tests/test_gpu_pdl_chains.py really overlap its two launches?  Runs each named chain back to back
under torch.profiler (CUDA activity) and reports, per run, how far the consumer kernel started before the producer
kernel ended (overlap > 0: the consumer's CTAs were running under the producer's tail).  With --both it runs itself
again with R3G_PDL=0, where the overlap must be <= 0.

    python tools/pdl_overlap.py --both [--runs 5] [--chains name ...] [--json out.json]
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "3d-re-gen_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import test_gpu_pdl_chains as chains  # noqa: E402

DEFAULT = ["chain_layernorm_f32_to_gemv_f32_over_its_input", "chain_layernorm_f32_then_lnpost_dot_over_its_input",
           "chain_layernorm_to_lnpost_dot", "chain_layernorm_to_linear128_residual", "chain_swiglu_to_layernorm_affine",
           "chain_swiglu_to_linear256_gated_residual", "chain_gemv_to_gemv_b2_silu_in", "chain_lnpost_dot_to_gemv_f32_b8",
           "chain_bilinear_to_im2col_stride1", "chain_im2col_to_bilinear_up", "chain_layernorm_to_bilinear_down_over_its_input",
           "chain_gemv_f32_to_small_attention_f32_d128", "chain_layernorm_to_windowed_attention"]


def measure(names, runs):
    specs = {s.name: s for s in chains.CHAINS}
    r3g = re.compile(r"\b(" + "|".join(chains.ENTRY) + r")\b")
    result = {}
    for name in names:
        c = specs[name].build()
        chains.run_back_to_back(c)                  # warm-up: module load, function attributes
        gaps = []
        for _ in range(runs):
            c.reset()
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                torch.cuda._sleep(20_000_000)         # both launches are queued before the producer starts
                c.producer()
                c.consumer()
                torch.cuda.synchronize()
            ks = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and r3g.search(e.name)),
                        key=lambda e: e.time_range.start)
            p, q = ks[0], ks[1]                       # the producer and the launch right after it
            gaps.append({"producer": r3g.search(p.name).group(1), "consumer": r3g.search(q.name).group(1),
                         "producer_us": p.time_range.end - p.time_range.start,
                         "overlap_us": p.time_range.end - q.time_range.start})
        result[name] = gaps
    return result


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chains", nargs="*", default=DEFAULT)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--both", action="store_true", help="also run with R3G_PDL=0 (a subprocess) and print both")
    ap.add_argument("--json")
    a = ap.parse_args()
    res = {"pdl": os.environ.get("R3G_PDL", "1")[:1] != "0", "gpu": torch.cuda.get_device_name(0),
           "chains": measure(a.chains, a.runs)}
    if not a.both:
        print(json.dumps(res))
        return
    env = dict(os.environ, R3G_PDL="0")
    r = subprocess.run([sys.executable, "-s", os.path.abspath(__file__), "--runs", str(a.runs), "--chains", *a.chains],
                       env=env, capture_output=True, text=True, check=True)
    off = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"{res['gpu']}: consumer start before producer end, microseconds (min / max over {a.runs} runs)")
    print(f"{'chain':58s} {'producer us':>11s} {'PDL on':>17s} {'R3G_PDL=0':>17s}")
    for name in a.chains:
        on, of = res["chains"][name], off["chains"][name]
        f = lambda g: f"{min(x['overlap_us'] for x in g):7.1f} / {max(x['overlap_us'] for x in g):7.1f}"  # noqa: E731
        print(f"{name[len('chain_'):]:58s} {on[0]['producer_us']:11.1f} {f(on):>17s} {f(of):>17s}")
    if a.json:
        with open(a.json, "w") as fh:
            json.dump({"on": res, "off": off}, fh, indent=1)


if __name__ == "__main__":
    main()
