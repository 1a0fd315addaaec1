"""CPU: libr3g.so loads without a GPU, exports exactly what include/r3g.h declares, and refuses to compute
without a CUDA device (no CPU fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as g
    g.build()
    from r3g import _abi
    return _abi.load_library()


def header_symbols():
    text = open(os.path.join(ROOT, "include", "r3g.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(r3g_[a-z0-9_]+)\s*\(", text)))


def test_header_and_binding_agree(lib):
    from r3g import _abi
    syms = header_symbols()
    assert syms, "no symbols parsed from r3g.h"
    assert sorted(_abi.SIGNATURES.keys()) == syms
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in r3g.h but not exported by libr3g.so"


def test_no_torch_or_oracle_linkage():
    so = os.path.join(ROOT, "3d-re-gen_b200", "r3g", "libr3g.so")
    import subprocess
    out = subprocess.run(["ldd", so], capture_output=True, text=True).stdout
    assert "torch" not in out and "oracle" not in out and "libcuda.so" not in out


def test_compute_fails_loudly_without_gpu(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from r3g import _abi
    with pytest.raises(_abi.R3GError):
        _abi.Context(0)
    assert lib.r3g_mc_workspace_bytes(9, 9, 9) > 0
    assert lib.r3g_version() >= 100


def test_every_compute_call_refuses_a_context_without_device(lib):
    """r3g_create(-1) returns R3G_E_CUDA but still hands back a (device-less) context, on any machine.  Every compute
    entry point given that context, or a NULL one, returns R3G_E_CUDA before it reads an argument (all are zero / NULL
    here), names itself in the error, and launches nothing."""
    from r3g import _abi
    not_compute = {"r3g_version", "r3g_create", "r3g_destroy", "r3g_last_error", "r3g_launch_count",
                   "r3g_mc_workspace_bytes", "r3g_decimate_workspace_bytes"}
    calls = [(name, [t() for t in argtypes[1:]]) for name, (_, argtypes) in sorted(_abi.SIGNATURES.items())
             if name not in not_compute]
    assert len(calls) == 26
    handle = ctypes.c_void_p()
    assert lib.r3g_create(-1, ctypes.byref(handle)) == _abi.R3G_E_CUDA and handle
    try:
        for name, zeros in calls:
            assert getattr(lib, name)(handle, *zeros) == _abi.R3G_E_CUDA, name
            assert lib.r3g_last_error(handle).decode().startswith(name[len("r3g_"):] + ": no CUDA device"), name
            assert getattr(lib, name)(None, *zeros) == _abi.R3G_E_CUDA, name
        assert lib.r3g_launch_count(handle) == 0
    finally:
        lib.r3g_destroy(handle)


def test_marching_cubes_workspace_size(lib):
    """r3g_mc_workspace_bytes is pure arithmetic (no device): it covers 16 B of vertex-id slots per grid point plus the
    sign bits, the crossed-cell list and the info words sized for every cell; degenerate grids give 0."""
    assert lib.r3g_mc_workspace_bytes(1, 9, 9) == 0
    prev = 0
    for n in (2, 9, 33, 65, 257, 513):
        b = lib.r3g_mc_workspace_bytes(n, n, n)
        assert b % 256 == 0 and b > prev
        assert b >= 16 * n ** 3 + n ** 3 // 8 + 6 * (n - 1) ** 3
        assert b <= 1.05 * (16 * n ** 3 + n ** 3 // 8 + 6 * (n - 1) ** 3) + (1 << 20)      # + masks, scan arrays, alignment
        prev = b
    assert lib.r3g_mc_workspace_bytes(7, 12, 9) > 0


def test_decimate_workspace_size(lib):
    """Pure arithmetic: grows with both sizes, 256-byte granular, 0 where the int32 limits are exceeded."""
    b = lib.r3g_decimate_workspace_bytes
    assert b(100, 200) > 0 and b(100, 200) % 256 == 0
    assert b(1000, 200) > b(100, 200) and b(100, 2000) > b(100, 200)
    n = 1 << 20
    assert 150 * n <= b(n, 0) - b(0, 0) <= 200 * n and 280 * n <= b(0, n) - b(0, 0) <= 330 * n
    assert b(1 << 31, 10) == 0 and b(10, 1 << 30) == 0 and b(-1, 10) == 0


def test_product_package_does_not_import_oracle():
    pkg = os.path.join(ROOT, "3d-re-gen_b200")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dp, f)).read()
                assert "oracle" not in src.replace("no oracle", ""), f"{f} mentions the oracle"
