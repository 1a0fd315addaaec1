#!/usr/bin/env python
"""Time r3g_linear at every GEMM shape of one DiT forward and one decode chunk, with its real epilogue: CUDA events
around replays of a CUDA graph of `--reps` launches, after a warm-up.  Prints one JSON line per shape (ms per launch,
executed TFLOP/s = 2 M N K / time).  --tree times the library of another tree (e.g. the parent commit extracted into
ab_parent/ and built there), so two arms can be compared in one session:
  python tools/ab_gemm.py --tree ab_parent; python tools/ab_gemm.py"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, MH = 1024, 4096          # DiT hidden width and MLP width


def shapes(ops):
    """(name, M, N, K, kwargs) of the launches; M of the DiT = 2 x (4096 latents + 346 text tokens) (CFG pairs)."""
    g64 = (1 + 0.1 * torch.randn(64, device="cuda")).half()
    gate = torch.randn(2, H, device="cuda").half()
    rms = lambda k0, cols: dict(mode=ops.QKN_RMS, q_col0=0, k_col0=k0, cols=cols, eps=1e-6, q_w=g64, k_w=g64)
    ln = dict(mode=ops.QKN_LAYERNORM, q_col0=0, k_col0=None, cols=H, eps=1e-6, q_w=g64, q_b=g64)
    return [
        ("dit.single.linear1", 8884, 3 * H + MH, H, dict(act=ops.ACT_GELU_TANH, act_cols=(3 * H, 3 * H + MH),
                                                          qk_norm=rms(H, H))),
        ("dit.single.linear2", 8884, H, 5120, dict(gate=gate, gate_rows=4442, residual=True)),
        ("dit.double.img_qkv", 8192, 3 * H, H, dict(qk_norm=rms(H, H))),
        ("dit.double.txt_qkv", 2740, 3 * H, H, dict(qk_norm=rms(H, H))),
        ("dit.double.img_proj", 8192, H, H, dict(gate=gate, gate_rows=4096, residual=True)),
        ("dit.double.img_fc1", 8192, MH, H, dict(act=ops.ACT_GELU_TANH)),
        ("dit.double.img_fc2", 8192, H, MH, dict(gate=gate, gate_rows=4096, residual=True)),
        ("decode.c_q", 65536, H, H, dict(qk_norm=ln)),
        ("decode.c_proj", 65536, H, H, dict(residual=True)),
        ("decode.c_fc", 65536, MH, H, dict(act=ops.ACT_GELU_ERF)),
        ("decode.mlp_proj", 65536, H, MH, dict(residual=True)),
    ]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=ROOT, help="repository tree whose built libr3g is timed")
    ap.add_argument("--reps", type=int, default=20, help="launches per graph")
    ap.add_argument("--replays", type=int, default=10)
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(os.path.abspath(args.tree), "3d-re-gen_b200"))
    from r3g import ops
    torch.manual_seed(0)
    arm = os.path.relpath(os.path.abspath(args.tree), ROOT)
    for name, M, N, K, kw in shapes(ops):
        x = torch.randn(M, K, device="cuda").half()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
        b = torch.randn(N, device="cuda").half()
        y = torch.randn(M, N, device="cuda").half()
        if kw.pop("residual", False):
            kw["residual"] = y
        for _ in range(3):
            ops.linear(x, w, b, out=y, **kw)
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
            for _ in range(args.reps):
                ops.linear(x, w, b, out=y, **kw)
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.replays):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / (args.replays * args.reps)
        print(json.dumps({"arm": arm, "shape": name, "M": M, "N": N, "K": K, "ms": round(ms, 4),
                          "tflops": round(2.0 * M * N * K / ms * 1e-9, 1)}), flush=True)


if __name__ == "__main__":
    main()
