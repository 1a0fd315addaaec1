"""Times VGGT's point head and track head on libr3g (device events) at VGGT-1B widths, 518 x 518, on seeded random
weights and tokens, and writes a torch.profiler trace of one track-head call under --out.

  python tools/bench_vggt_heads.py --frames 4 --queries 256 --reps 10 --out OUT_DIR

Prints one JSON line: milliseconds per head call, the tracker's GEMM FLOPs (from shapes) over the track-head time and
over the time of the GEMM kernels in the trace, and the share of the traced GPU time spent in kernels that are not
libr3g's (torch glue: grid_sample, pooling, element-wise ops, copies)."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))


def tracker_gemm_flops(S, N, HH, WW, iters=4, levels=7, radius=4, hidden=384, latent=128, depth=6, virtual=64):
    """FLOPs of the tracker's GEMMs per call (2 * M * N * K each; attention QK^T and PV at the padded head width 64)."""
    f, H, W = 0, HH, WW
    for _ in range(levels):
        f += 2 * S * N * (H * W) * latent                     # correlation of every query with every pixel
        H, W = H // 2, W // 2
    M = N * S
    f += 2 * M * hidden * (levels * (2 * radius + 1) ** 2) + 2 * M * latent * hidden        # corr_mlp
    f += 2 * M * hidden * 392 + 2 * M * 160 * hidden + 2 * M * latent * latent               # in / flow / ffeat
    Nt = N + virtual
    blk = lambda rows, ctx, Lq, Lk, nb: (2 * rows * 512 * 384 + 2 * ctx * 1024 * 384 + 2 * rows * 384 * 512  # noqa: E731
                                         + 4 * nb * 8 * Lq * Lk * 64 + 2 * 2 * rows * 1536 * 384)
    per = depth * blk(Nt * S, Nt * S, S, S, Nt)                                              # time blocks
    per += depth * (blk(virtual * S, N * S, virtual, N, S) + blk(virtual * S, virtual * S, virtual, virtual, S)
                    + blk(N * S, virtual * S, N, virtual, S))                                # space blocks
    return iters * (f + per) + 2 * M * 32 * latent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=4)
    ap.add_argument("--queries", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", required=True, help="directory for the profiler trace")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vggt_heads needs a CUDA device")
    from r3g.vggt_heads import DPTHeadR3G, random_state_dict
    from r3g.vggt_track import TrackHeadR3G
    os.makedirs(args.out, exist_ok=True)
    S, N = args.frames, args.queries
    sd = random_state_dict(0, depth=1, vit_depth=1, trunk_depth=1, full=True)
    sd = {k: v for k, v in sd.items() if k.startswith(("point_head.", "track_head."))}
    idx = dict(intermediate_layer_idx=(0, 1, 2, 3))
    point = DPTHeadR3G(sd, "point_head.", activation="inv_log", **idx)
    track = TrackHeadR3G(sd, **idx)
    g = torch.Generator(device="cuda").manual_seed(0)
    toks = [torch.randn(1, S, 5 + 37 * 37, 2048, device="cuda", generator=g) for _ in range(4)]
    imgs = torch.rand(1, S, 3, 518, 518, device="cuda", generator=g)
    qp = torch.rand(1, N, 2, device="cuda", generator=g) * 517

    def timed(fn):
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / args.reps

    ms_point = timed(lambda: point(toks, imgs, 5))
    ms_track = timed(lambda: track(toks, imgs, 5, qp))
    flops = tracker_gemm_flops(S, N, 259, 259)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        track(toks, imgs, 5, qp)
        torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(args.out, "track_head_trace.json"))
    total = gemm = glue = 0.0
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if e.key.startswith(("aten::", "cuda", "Memcpy", "Memset")) or t == 0:
            continue
        total += t
        torch_kernel = "at::" in e.key or "native" in e.key      # aten's kernels; libr3g's live in its own namespace
        if torch_kernel:
            glue += t
        elif "linear" in e.key:
            gemm += t
    props = torch.cuda.get_device_properties(0)
    line = {"device": props.name, "frames": S, "queries": N, "ms_point_head": round(ms_point, 3),
            "ms_track_head": round(ms_track, 3), "tracker_gemm_gflop": round(flops / 1e9, 2),
            "tracker_gemm_tflops_over_head_time": round(flops / (ms_track * 1e-3) / 1e12, 2),
            "tracker_gemm_tflops_over_gemm_kernel_time": round(flops / (gemm * 1e-6) / 1e12, 2) if gemm else None,
            "torch_glue_share_of_kernel_time": round(glue / total, 3) if total else None,
            "trace": os.path.join(args.out, "track_head_trace.json")}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
