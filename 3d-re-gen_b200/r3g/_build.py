"""In-tree build of libr3g.so (nvcc, sm_90a only).

The object files and the .so are build products (git-ignored); build_cuda() rebuilds them when a source is newer.
"""
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(PKG_DIR))
CSRC = os.path.join(os.path.dirname(PKG_DIR), "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libr3g.so")

CU_SOURCES = ["ctx.cu", "mc.cu", "mesh.cu", "decimate.cu", "rowops.cu", "heads.cu", "conv.cu", "gemm.cu", "attn.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "-cudart", "static",
]


def _newer(target, sources):
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(s) <= t for s in sources)


def _nvcc():
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: cannot build libr3g.so")
    return exe


def build_cuda(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in CU_SOURCES]
    deps = srcs + [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith((".h", ".cuh"))]
    deps += [os.path.join(ROOT, "include", h) for h in ("r3g.h", "r3g_mc_tables.h")]
    if not force and _newer(LIB_PATH, deps):
        return LIB_PATH
    objs = []
    obj_dir = os.path.join(os.path.dirname(PKG_DIR), "build")
    os.makedirs(obj_dir, exist_ok=True)
    procs = []
    for s in srcs:
        o = os.path.join(obj_dir, os.path.basename(s).replace(".cu", ".o"))
        objs.append(o)
        cmd = [_nvcc()] + NVCC_FLAGS + ["-c", s, "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for s, pr in procs:
        out, _ = pr.communicate()
        if verbose and out:
            print(out)
        if pr.returncode != 0:
            raise RuntimeError(f"nvcc failed on {s}:\n{out}")
    link = [_nvcc(), "-shared", "-cudart", "static", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB_PATH] + objs
    r = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}")
    return LIB_PATH


if __name__ == "__main__":
    print(build_cuda(force="--force" in sys.argv, verbose="-v" in sys.argv))
