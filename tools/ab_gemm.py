#!/usr/bin/env python
"""Time r3g_linear at every GEMM shape of one DiT forward and one decode chunk, with its real epilogue, and the grouped
fc1, grouped fc2 and combine launches of one Hunyuan3D-2mini MoE layer: CUDA events around replays of a CUDA graph of
`--reps` launches, after a warm-up.  Prints one JSON line per shape (ms per launch, executed TFLOP/s = 2 M N K / time,
M = the rows computed).  --tree times the library of another tree (e.g. the parent commit extracted into ab_parent/ and
built there), so two arms can be compared in one session:
  python tools/ab_gemm.py --tree ab_parent; python tools/ab_gemm.py"""
import argparse
import itertools
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


def linear_launches(ops):
    """(name, M, N, K, launch) of shapes(), each on fresh random operands."""
    for name, M, N, K, kw in shapes(ops):
        x = torch.randn(M, K, device="cuda").half()
        w = (torch.randn(N, K, device="cuda") * K ** -0.5).half()
        b = torch.randn(N, device="cuda").half()
        y = torch.randn(M, N, device="cuda").half()
        if kw.pop("residual", False):
            kw["residual"] = y
        yield name, M, N, K, lambda: ops.linear(x, w, b, out=y, **kw)


def moe_launches(ops):
    """(name, rows, N, K, launch) of the three GEMMs of one 2mini MoE layer (HunYuanDiTPlain._moe) on a CFG pair: M = 2 x
    (512 latents + 1) rows routed top-2 over 8 experts by a random gate; fc1 computes the experts' 2 M rows and the shared
    expert's M, fc2 the experts' 2 M, combine the shared expert's M."""
    from r3g.pipelines import HUNYUAN3D_2MINI_CONFIG
    cfg = HUNYUAN3D_2MINI_CONFIG["model"]
    H, E, k = cfg["hidden_size"], cfg["num_experts"], cfg["moe_top_k"]
    M = 2 * (HUNYUAN3D_2MINI_CONFIG["vae"]["num_latents"] + 1)
    f16 = lambda *s, std=1.0: (torch.randn(*s, device="cuda") * std).half()  # noqa: E731
    i32 = lambda *s: torch.empty(*s, device="cuda", dtype=torch.int32)  # noqa: E731
    SX, SH, SY = f16((E + 1) * M, H), f16((E + 1) * M, 4 * H), f16(E * M, H)
    r = dict(slot_scale=f16(E * M), counts=i32(E), ids=i32(M, k), weights=f16(M, k), slots=i32(M, k))
    ops.moe_route(SX[E * M:], f16(E, H, std=H ** -0.5), top_k=k, cap=M, slot_x=SX, **r)
    w1, b1 = f16(E + 1, 4 * H, H, std=H ** -0.5), f16(E + 1, 4 * H)
    w2, b2 = f16(E, H, 4 * H, std=(4 * H) ** -0.5), f16(E, H)
    wc, bc, s = f16(H, 4 * H, std=(4 * H) ** -0.5), f16(H), f16(M, H)
    yield "mini.moe.fc1", (k + 1) * M, 4 * H, H, lambda: ops.moe_grouped(
        SX, w1, b1, counts=r["counts"], experts=E, out=SH, act=ops.ACT_GELU_ERF)
    yield "mini.moe.fc2", k * M, H, 4 * H, lambda: ops.moe_grouped(
        SH[:E * M], w2, b2, counts=r["counts"], experts=E, out=SY, row_scale=r["slot_scale"])
    yield "mini.moe.combine", M, H, 4 * H, lambda: ops.moe_combine(
        SH[E * M:], wc, bc, slot_y=SY, ids=r["ids"], slots=r["slots"], residual=s, out=s)


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
    for name, M, N, K, launch in itertools.chain(linear_launches(ops), moe_launches(ops)):
        for _ in range(3):
            launch()
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(g, stream=s):
            for _ in range(args.reps):
                launch()
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
