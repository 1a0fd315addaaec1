"""CPU: what the built library's machine code must contain (cuobjdump on the in-tree libr3g.so).  These are the SASS
mnemonics that prove the Hopper paths are the ones compiled in -- warpgroup MMAs (HGMMA), TMA loads (UTMALDG), the
register-operand P V product of the attention kernel -- and guards against two regressions: a GPU-scope membar in the
GEMM pipeline (a `.release` arrive compiles to MEMBAR.ALL.GPU) and register spills in the hot kernels."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "3d-re-gen_b200", "r3g", "libr3g.so")


@pytest.fixture(scope="module")
def sass():
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    import sys
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge
    ge.build()
    txt = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for blk in re.split(r"\n\s*Function : ", txt)[1:]:
        name, _, body = blk.partition("\n")
        funcs[name.strip()] = body
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    usage = {m.group(1): (int(m.group(2)), int(m.group(3)))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+)", res)}
    return funcs, usage


def _one(funcs, *needles):
    hits = [n for n in funcs if all(s in n for s in needles)]
    assert hits, f"no kernel matching {needles}"
    return hits


def test_gemm_is_wgmma_tma_and_has_no_gpu_scope_membar(sass):
    funcs, usage = sass
    for name, shape in ((_one(funcs, "linear_kernelILi128E")[0], "64x128x16"),
                        (_one(funcs, "linear_kernelILi256E")[0], "64x256x16")):
        body = funcs[name]
        assert "HGMMA." + shape + ".F32" in body and "UTMALDG" in body, name
        assert "MEMBAR.ALL.GPU" not in body, name + ": a GPU-scope membar in the pipeline"
    name = _one(funcs, "linear_kernelILi256E")[0]
    assert usage[name][1] == 0, f"{name}: {usage[name][1]} bytes of stack (spills)"


def test_attention_uses_register_operand_wgmma(sass):
    funcs, usage = sass
    name = _one(funcs, "attention_kernel")[0]
    body = funcs[name]
    assert re.search(r"HGMMA\.64x128x16\.F32\S* R\d+, gdesc\[", body), "Q K^T is the shared-memory form"
    assert re.search(r"HGMMA\.64x64x16\.F32\S* R\d+, R\d+, gdesc\[UR\d+\]\.tnspB", body), \
        "P V must take its A operand from registers and V MN-major"
    for op in ("UTMALDG", "MUFU.EX2"):
        assert op in body, op
    assert usage[name][1] == 0, "register spills in the softmax loop"
    assert "NANOSLEEP.SYNCS" in body           # mbarrier.try_wait carries the suspend-time hint


def test_row_kernels_move_rows_as_16_byte_accesses(sass):
    funcs, _ = sass
    # every fp16 row moves as 16-byte accesses (a `__half2 v[4]` payload is copied member-wise: four 32-bit LDG/STG)
    for needle in ("layernorm_kernelILi4E", "lnpost_dot_kernelILi4E", "qk_norm_kernel", "gemv_kernel"):
        body = funcs[_one(funcs, needle)[0]]
        assert "LDG.E.128" in body or "LDG.E.CONSTANT.128" in body or "LD.E.128" in body, needle
    for needle in ("layernorm_kernelILi4E", "grid_fourier_kernel"):
        assert "STG.E.128" in funcs[_one(funcs, needle)[0]], needle


def test_no_spills_in_row_kernels(sass):
    funcs, usage = sass
    # (grid_fourier_kernel keeps 32 bytes of stack: sinf/cosf's Payne-Hanek branch, unreachable for fp16 arguments)
    for needle in ("layernorm_kernelILi4E", "lnpost_dot_kernelILi4E", "qk_norm_kernel", "cfg_euler_kernel"):
        name = _one(funcs, needle)[0]
        assert usage[name][1] == 0, f"{name}: {usage[name][1]} bytes of stack"


def test_marching_cubes_emit_has_no_output_atomics(sass):
    funcs, _ = sass
    for needle in ("mc_vertex_kernel", "mc_face_kernel"):
        body = funcs[_one(funcs, needle)[0]]
        assert "ATOMG" not in body and "RED." not in body, needle + ": output order must come from the scans"
