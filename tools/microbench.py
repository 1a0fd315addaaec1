#!/usr/bin/env python
"""Kernel micro-benchmarks on one H100 (CUDA events, warm-up, L2 flush between timed launches)."""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3d-re-gen_b200"))
from r3g import ops  # noqa: E402

FLUSH = None


def flush_l2():
    global FLUSH
    if FLUSH is None:
        FLUSH = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    FLUSH.zero_()


def timeit(fn, iters=10, warm=3, flush=True):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush:
            flush_l2()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    out = []
    torch.manual_seed(0)
    only = os.environ.get("R3G_MB_ONLY", "")
    for (M, N, K) in [] if only and "linear" not in only else [(8884, 7168, 1024), (8884, 1024, 5120), (6144, 3072, 1024), (6144, 4096, 1024),
                      (6144, 1024, 4096), (2740, 3072, 1024), (32768, 4096, 1024), (32768, 1024, 4096),
                      (32768, 1024, 1024)]:
        x = torch.randn(M, K, device="cuda").half()
        w = torch.randn(N, K, device="cuda").half()
        b = torch.randn(N, device="cuda").half()
        y = torch.empty(M, N, device="cuda", dtype=torch.float16)
        ms = timeit(lambda: ops.linear(x, w, b, out=y))
        ms_t = timeit(lambda: torch.nn.functional.linear(x, w, b))
        fl = 2.0 * M * N * K
        out.append(dict(op="linear", M=M, N=N, K=K, ms=ms, tflops=fl / ms / 1e9, torch_ms=ms_t,
                        torch_tflops=fl / ms_t / 1e9))
        print(out[-1], flush=True)
    for (B, H, Lq, Lk) in [] if only and "attention" not in only else [(2, 16, 4442, 4442), (1, 16, 3072, 3072), (1, 16, 65536, 3072)]:
        q = torch.randn(B, Lq, H, 64, device="cuda").half()
        k = torch.randn(B, Lk, H, 64, device="cuda").half()
        v = torch.randn(B, Lk, H, 64, device="cuda").half()
        o = torch.empty_like(q)
        ms = timeit(lambda: ops.attention(q, k, v, out=o))
        qt, kt, vt = (t.transpose(1, 2).contiguous() for t in (q, k, v))
        ms_t = timeit(lambda: torch.nn.functional.scaled_dot_product_attention(qt, kt, vt))
        fl = 4.0 * B * H * Lq * Lk * 64
        out.append(dict(op="attention", B=B, H=H, Lq=Lq, Lk=Lk, ms=ms, tflops=fl / ms / 1e9, torch_ms=ms_t,
                        torch_tflops=fl / ms_t / 1e9))
        print(out[-1], flush=True)
    for n in [] if only and "mc" not in only else (257, 513):
        ax = torch.linspace(-1.01, 1.01, n, device="cuda")
        x, y, z = torch.meshgrid(ax, ax, ax, indexing="ij")
        vol = (0.25 - torch.sqrt((torch.sqrt(x * x + y * y) - 0.6) ** 2 + z * z)).contiguous()
        del x, y, z
        ms = timeit(lambda: ops.marching_cubes(vol, 0.0), iters=5)
        v, f = ops.marching_cubes(vol, 0.0)
        out.append(dict(op="marching_cubes", n=n, ms=ms, verts=len(v), faces=len(f),
                        grid_gbs=n ** 3 * 4 * 3 / ms / 1e6))
        print(out[-1], flush=True)
    if not only or "rowops" in only:
        def rec(name, fn, nbytes, **kw):
            for fl in (True, False):
                ms = timeit(fn, iters=20, flush=fl)
                out.append(dict(op=name, l2="flushed" if fl else "warm", us=ms * 1e3, gbs=nbytes / ms / 1e6, **kw))
                print(out[-1], flush=True)
        W = 1024
        for rows, B in ((6144, 2), (8884, 2)):   # DiT: modulated LayerNorm of the img stream / the joint stream
            x = torch.randn(rows, W, device="cuda").half()
            sc, sh = torch.randn(B, W, device="cuda").half(), torch.randn(B, W, device="cuda").half()
            y = torch.empty_like(x)
            rec("layernorm_mod", lambda: ops.layernorm(x, eps=1e-6, scale=sc, shift=sh, rows_per_batch=rows // B, out=y),
                rows * W * 4, rows=rows)
        for rows in (65536,):                     # decode: affine LayerNorm, q LayerNorm per head, ln_post + dot
            x = torch.randn(rows, W, device="cuda").half()
            g, b_ = torch.randn(W, device="cuda").half(), torch.randn(W, device="cuda").half()
            y = torch.empty_like(x)
            rec("layernorm_affine", lambda: ops.layernorm(x, g, b_, eps=1e-6, out=y), rows * W * 4, rows=rows)
            g64, b64 = torch.randn(64, device="cuda").half(), torch.randn(64, device="cuda").half()
            rec("qk_norm_ln_q", lambda: ops.qk_norm_(x, 16, 0, 0, 64, 1, 1e-6, g64, b64), rows * W * 4, rows=rows)
            wo, bo = torch.randn(W, device="cuda").half(), torch.randn(1, device="cuda").half()
            o32 = torch.empty(rows, device="cuda", dtype=torch.float32)
            rec("lnpost_dot", lambda: ops.lnpost_dot(x, g, b_, wo, bo, o32, eps=1e-5), rows * W * 2, rows=rows)
            emb = torch.empty(rows, 64, device="cuda", dtype=torch.float16)
            rec("grid_fourier", lambda: ops.grid_fourier(emb, 0, rows, 256, [-1.01] * 3 + [1.01] * 3, 8, False),
                rows * 128, rows=rows)
        for rows, ld, koff in ((6144, 3072, 1024), (8884, 7168, 5120)):   # DiT: RMS norm of q and k inside the packed qkv
            qkv = torch.randn(rows, ld, device="cuda").half()
            g64 = torch.randn(64, device="cuda").half()
            rec("qk_norm_rms_qk", lambda: ops.qk_norm_(qkv, 16, 0, koff, 64, 0, 1e-6, g64, None, g64, None),
                rows * 2048 * 4, rows=rows, ld=ld)
        wm = torch.randn(290 * 1024, W, device="cuda").half()
        bm = torch.randn(290 * 1024, device="cuda").half()
        vec = torch.randn(2, W, device="cuda").half()
        om = torch.empty(2, 290 * 1024, device="cuda", dtype=torch.float16)
        rec("gemv_modulation", lambda: ops.gemv(wm, bm, vec, silu_in=True, out=om), wm.numel() * 2, rows=290 * 1024)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(out, open(os.path.join(ROOT, "gpurun_out", os.environ.get("R3G_MB_OUT", "microbench.json")), "w"), indent=1)


if __name__ == "__main__":
    main()
