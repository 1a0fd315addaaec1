"""CPU: the numpy mirror of the GPU decimator (oracle/decimate.py) on marching-cubes meshes of analytic fields -- the
reduced meshes are closed (or open where the input is), consistently oriented 2-manifolds with the input's topology, stay
on the surface, and land on the target face count.  tests/test_gpu_decimate.py pins the CUDA kernels to this mirror bit
for bit."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- meshes -----------------------------------------------------------------------------------------------------------
def sdf_sphere(p, r=0.6):
    return r - np.sqrt((p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1]) + p[..., 2] * p[..., 2])


def sdf_torus(p, R=0.55, r=0.2):
    q = np.sqrt(p[..., 0] * p[..., 0] + p[..., 1] * p[..., 1]) - R
    return r - np.sqrt(q * q + p[..., 2] * p[..., 2])


def sdf_scene(p):
    """test_gpu_postprocess's scene: a big sphere and three small ones (one of them under FloaterRemover's 0.5 % rule)."""
    d = sdf_sphere(p)
    for cx, cy, cz, r in ((0.8, 0.8, 0.8, 0.15), (-0.85, 0.8, -0.8, 0.035), (0.85, -0.85, 0.2, 0.03)):
        d = np.maximum(d, sdf_sphere(p - np.array([cx, cy, cz], p.dtype), r))
    return d


def sdf_scene3(p):
    """The benchmark's analytic scene: a sphere, a torus around it and a small sphere."""
    d = np.maximum(sdf_sphere(p - np.array([0.0, 0.0, 0.05], p.dtype), 0.45), sdf_torus(p, 0.7, 0.15))
    return np.maximum(d, sdf_sphere(p - np.array([0.75, 0.75, 0.6], p.dtype), 0.12))


def sdf_open(p):
    """A sphere larger than the grid box: marching cubes cuts it open at the six faces of the box."""
    return sdf_sphere(p, 1.1)


FIELDS = {"sphere": sdf_sphere, "torus": sdf_torus, "scene": sdf_scene, "scene3": sdf_scene3, "open": sdf_open}


def mc_mesh(kind, n):
    """Marching cubes (oracle/mc.py, skimage's conventions) of FIELDS[kind] on an n^3 grid over [-1, 1]^3; vertices in
    float32 world coordinates, faces in descent winding."""
    import mc as omc
    ax = np.linspace(-1, 1, n, dtype=np.float32)
    g = np.stack(np.meshgrid(ax, ax, ax, indexing="ij"), -1)
    v, f = omc.marching_cubes(FIELDS[kind](g).astype(np.float32), 0.0)
    return (v * np.float32(2.0 / (n - 1)) - np.float32(1.0)).astype(np.float32), f


# ---- properties -------------------------------------------------------------------------------------------------------
def _edges(f):
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)


def _components(n, e):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    if len(e) == 0:
        return 0
    used = np.unique(e)
    g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    return len(np.unique(lab[used]))


def topology(v, f):
    """(Euler characteristic, components, boundary loops, boundary edges, directed edges seen twice, edges in > 2
    faces)."""
    d = _edges(f)
    n = np.int64(len(v))
    ukey, cnt = np.unique(d.min(1) * n + d.max(1), return_counts=True)
    _, dcnt = np.unique(d[:, 0] * n + d[:, 1], return_counts=True)
    bk = ukey[cnt == 1]
    bnd = np.stack([bk // n, bk % n], 1)
    chi = len(np.unique(f)) - len(ukey) + len(f)
    return chi, _components(len(v), d), _components(len(v), bnd), len(bnd), int((dcnt > 1).sum()), int((cnt > 2).sum())


def _normal_signs(v, f, sdf):
    """sign of (face normal . field gradient at the centroid) per face."""
    p = v.astype(np.float64)
    n = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
    c = (p[f[:, 0]] + p[f[:, 1]] + p[f[:, 2]]) / 3
    h = 1e-5
    grad = np.stack([(sdf(c + h * np.eye(3)[i]) - sdf(c - h * np.eye(3)[i])) / (2 * h) for i in range(3)], 1)
    return np.sign((n * grad).sum(1))


def check_reduced(v_in, f_in, v, f, target, sdf, err_bound, exact=True):
    """The properties every reduced mesh must have; returns the largest |sdf| over the output vertices.  sdf None: the
    topology checks only (a mesh reduced to a few faces per component no longer follows the surface)."""
    assert v.dtype == np.float32 and f.dtype == np.int32 and v.ndim == 2 and f.ndim == 2
    if exact:
        assert len(f) in (target - 1, target), (len(f), target)
    else:
        assert len(f) <= len(f_in)
    assert ((f[:, 0] != f[:, 1]) & (f[:, 1] != f[:, 2]) & (f[:, 0] != f[:, 2])).all(), "a face repeats an index"
    assert f.min() >= 0 and f.max() < len(v) and len(np.unique(f)) == len(v), "unreferenced vertices"
    chi0, comp0, loops0, _, _, _ = topology(v_in, f_in)
    chi, comp, loops, nbnd, twice, over = topology(v, f)
    assert over == 0 and twice == 0, "not a consistently oriented 2-manifold"
    assert (chi, comp, loops) == (chi0, comp0, loops0)
    if loops0 == 0:
        assert nbnd == 0
    if sdf is None:
        return None
    # winding: every face normal points up the field (skimage's descent winding), as the input's non-degenerate faces do
    s_in = _normal_signs(v_in, f_in, sdf)
    assert (s_in[s_in != 0] > 0).all()
    s = _normal_signs(v, f, sdf)
    assert (s > 0).all(), f"{(s <= 0).sum()} of {len(f)} faces do not point up the field"
    err = np.abs(sdf(v.astype(np.float64))).max()
    assert err <= err_bound, err
    return err


# (mesh, grid, targets, bound on |sdf| of the reduced vertices, in units of the input grid spacing 2 / (n - 1))
CASES = [("sphere", 41, (2000, 501), 0.25), ("torus", 41, (2000, 601), 0.5), ("scene", 65, (3000, 1001), 0.5),
         ("open", 41, (4000, 2000), 0.5)]


@pytest.mark.parametrize("kind, n, targets, bound", CASES, ids=[c[0] for c in CASES])
def test_mirror_reduces_to_the_target_and_keeps_the_surface(kind, n, targets, bound):
    import decimate as odec
    v0, f0 = mc_mesh(kind, n)
    for target in targets:
        assert len(f0) > target
        v, f, rounds = odec.decimate(v0, f0, target)
        assert rounds > 0
        check_reduced(v0, f0, v, f, target, FIELDS[kind], bound * 2 / (n - 1))


def test_mirror_stops_at_the_smallest_mesh_the_rules_allow():
    """An unreachable target: every component keeps at least a tetrahedron, the rounds end when no edge is valid."""
    import decimate as odec
    v0, f0 = mc_mesh("scene3", 33)
    v, f, _ = odec.decimate(v0, f0, 0)
    chi, comp, _, _, _, _ = topology(v, f)
    assert comp == topology(v0, f0)[1] == 3 and len(f) >= 4 * comp
    check_reduced(v0, f0, v, f, 0, None, None, exact=False)


def test_mirror_is_deterministic_and_cleans():
    import decimate as odec
    v0, f0 = mc_mesh("torus", 33)
    a = odec.decimate(v0, f0, 700)
    b = odec.decimate(v0.copy(), f0.copy(), 700)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    # autoclean: a face with a repeated index and an unreferenced vertex are dropped, even at a target not below nf
    v1 = np.concatenate([v0, np.zeros((1, 3), np.float32)])
    f1 = np.concatenate([f0, [[0, 0, 1]]]).astype(np.int32)
    v, f, rounds = odec.decimate(v1, f1, len(f1))
    assert rounds == 0 and np.array_equal(f, f0) and np.array_equal(v, v0)
    with pytest.raises(ValueError):
        odec.decimate(v0, np.array([[0, 1, len(v0)]], np.int32), 0)


def test_no_spills_in_the_decimation_kernels():
    """Every kernel of decimate.cu runs without a stack frame (the float64 pricing kernel included)."""
    import shutil
    import subprocess
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not on PATH")
    import __graft_entry__ as g
    g.build()
    res = subprocess.run(["cuobjdump", "-res-usage", os.path.join(ROOT, "3d-re-gen_b200", "r3g", "libr3g.so")],
                         capture_output=True, text=True, check=True).stdout
    usage = {m.group(1): int(m.group(2)) for m in re.finditer(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", res)}
    ours = {name: stack for name, stack in usage.items() if "decimate_cu" in name}
    assert len(ours) >= 15 and any("cost_kernel" in n for n in ours), sorted(ours)
    assert not {n: s for n, s in ours.items() if s}, "stack frames (spills) in the decimation kernels"
