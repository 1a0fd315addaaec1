"""ORACLE -- test infrastructure only.  ctypes front end of oracle/dmc_oracle.c (CPU dual marching cubes, the
specification of r3g's R3G_MC_DUAL).  Importable only from tests/."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "_build", "libr3g_dmc_oracle.so")
_lib = None


def build(force=False):
    src = os.path.join(_HERE, "dmc_oracle.c")
    deps = [src, os.path.join(_HERE, "mc_oracle.c"), os.path.join(_HERE, "..", "include", "r3g_mc_tables.h")]
    if not force and os.path.exists(_LIB) and all(os.path.getmtime(_LIB) >= os.path.getmtime(p) for p in deps):
        return _LIB
    os.makedirs(os.path.dirname(_LIB), exist_ok=True)
    subprocess.run(["gcc", "-O2", "-std=c11", "-ffp-contract=off", "-shared", "-fPIC", src, "-lm", "-o", _LIB],
                   check=True)
    return _LIB


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB):
            build()
        _lib = C.CDLL(_LIB)
        _lib.r3g_oracle_dual_marching_cubes.restype = C.c_int
        _lib.r3g_oracle_dual_marching_cubes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float,
                                                        C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                                        C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                                        C.POINTER(C.c_void_p)]
        _lib.r3g_oracle_free.argtypes = [C.c_void_p]
    return _lib


def dual_marching_cubes(volume, level=0.0, return_cells=False):
    """(verts float32 [V,3] in [0, 1]^3, array-axis order; faces int32 [F,3], normals towards increasing values), and
    with return_cells the flat index of the cell each vertex belongs to.  Raises RuntimeError when no cell is crossed,
    like ops.dual_marching_cubes."""
    lib = _load()
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    n0, n1, n2 = vol.shape
    vp, fp, cp = C.c_void_p(), C.c_void_p(), C.c_void_p()
    nv, nf = C.c_int64(), C.c_int64()
    rc = lib.r3g_oracle_dual_marching_cubes(vol.ctypes.data, n0, n1, n2, float(level), C.byref(vp), C.byref(nv),
                                            C.byref(fp), C.byref(nf), C.byref(cp) if return_cells else None)
    if rc == 2:
        raise RuntimeError("No surface found at the given iso value.")
    verts = _take(lib, vp, C.c_float, np.float32, (nv.value, 3))
    faces = _take(lib, fp, C.c_int32, np.int32, (nf.value, 3))      # a grid with no interior edge has no face
    if not return_cells:
        return verts, faces
    return verts, faces, _take(lib, cp, C.c_int64, np.int64, (nv.value,))


def _take(lib, p, ctype, dtype, shape):
    """Copy a malloc'd C array into numpy and free it (NULL: the array is empty)."""
    if not p.value:
        return np.zeros(shape, dtype)
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(ctype)), shape=shape).copy()
    lib.r3g_oracle_free(p)
    return out
