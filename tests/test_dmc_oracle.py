"""CPU: r3g's dual marching cubes oracle (oracle/dmc_oracle.c, table driven) against
  * a SECOND, independent implementation (oracle/dmc_tracer.py: tilings traced from the rules, patches by union-find,
    quads from a dict keyed by grid edge) -- bit for bit, order included,
  * counts and invariants computed directly from the volume with numpy,
  * the topology and orientation of closed test surfaces, and the open mesh of a surface that reaches the grid's faces.
Non-manifold edges are a property of plain dual marching cubes (one patch can hold both segments of an ambiguous face):
they may occur on noise, and the smooth closed surfaces here have none."""
import numpy as np
import pytest
import torch

import dmc as odmc
from test_mc_oracle import check_closed_manifold, edge_stats, noise, random_field, signed_volume, sphere, torus


def _atlas():
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location(
        "dump_goldens", os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools",
                                     "dump_skimage_goldens.py"))
    dg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dg)
    return dg.case_atlas(0)


def with_nans(vol, seed, frac=0.05):
    vol = vol.copy()
    vol[np.random.default_rng(seed).random(vol.shape) < frac] = np.nan
    return vol


def _volumes():
    yield "noise_12x13x14", noise((12, 13, 14), 0)
    yield "noise_14x12x13", noise((14, 12, 13), 1)
    yield "noise_9", noise((9, 9, 9), 2)
    yield "noise_ragged_open", np.random.default_rng(7).standard_normal((7, 12, 9)).astype(np.float32)
    yield "random_field_15", random_field(15, 3)
    yield "random_field_17", random_field(17, 5)
    yield "torus_17", torus(17)
    yield "nan_noise", with_nans(noise((11, 10, 12), 4), 4)
    yield "case_atlas", _atlas()


@pytest.mark.parametrize("name,vol", list(_volumes()), ids=[n for n, _ in _volumes()])
def test_oracle_equals_independent_tracer(name, vol):
    import dmc_tracer
    v, f = odmc.dual_marching_cubes(vol)
    tv, tf = dmc_tracer.dual_marching_cubes(vol)
    assert v.dtype == np.float32 and f.dtype == np.int32
    assert np.array_equal(v, tv, equal_nan=True) and np.array_equal(f, tf), name
    assert f.min() >= 0 and f.max() < len(v)


def interior_crossings(vol):
    """Sign-changing grid edges whose four incident cells lie in the grid, counted per array axis with numpy."""
    above = vol > 0
    n = 0
    for a in range(3):
        lo = np.take(above, range(vol.shape[a] - 1), axis=a)
        hi = np.take(above, range(1, vol.shape[a]), axis=a)
        ch = lo != hi
        for b in range(3):
            if b != a:
                ch = np.take(ch, range(1, vol.shape[b] - 1), axis=b)
        n += int(ch.sum())
    return n


@pytest.mark.parametrize("name,vol", [("noise", noise((12, 13, 14), 0)), ("ragged", random_field(15, 3)[:9, 2:, 4:]),
                                      ("nan", with_nans(random_field(13, 1), 1)), ("sphere", sphere(33))])
def test_two_triangles_per_interior_sign_changing_edge(name, vol):
    v, f = odmc.dual_marching_cubes(vol)
    assert len(f) == 2 * interior_crossings(vol), name


@pytest.mark.parametrize("vol,chi", [(sphere(65), 2), (torus(49), 0)], ids=["sphere65", "torus49"])
def test_closed_surfaces_topology_and_orientation(vol, chi):
    from r3g.pipelines import export_to_trimesh
    from r3g.vae import Latent2MeshOutput, center_vertices
    v, f = odmc.dual_marching_cubes(vol)
    assert check_closed_manifold(v, f) == chi          # every edge in exactly two faces, consistently oriented
    assert np.array_equal(np.unique(f), np.arange(len(v)))
    # run() orientation: normals towards increasing logits (into the object), like marching cubes: negative volume
    vc = center_vertices(torch.from_numpy(v)).numpy()
    assert signed_volume(vc, f) < 0
    mesh = export_to_trimesh(Latent2MeshOutput(mesh_v=vc, mesh_f=f))
    assert signed_volume(np.asarray(mesh.vertices), np.asarray(mesh.faces)) > 0
    # unit-sized and centred: the bounding box is symmetric about 0
    assert np.allclose(vc.min(0), -vc.max(0), atol=1e-6) and vc.max() < 0.5


def test_sphere_vertices_lie_near_the_surface():
    n = 65
    v, _ = odmc.dual_marching_cubes(sphere(n))
    w = v.astype(np.float64) * 2.02 - 1.01
    assert np.abs(np.linalg.norm(w, axis=1) - 0.6).max() < 1.5 * 2.02 / (n - 1)


@pytest.mark.parametrize("vol", [noise((12, 13, 14), 0), random_field(17, 5), with_nans(noise((9, 10, 11), 3), 3)],
                         ids=["noise", "random_field", "nan"])
def test_every_vertex_lies_in_its_cell_and_cells_follow_traversal_order(vol):
    v, f, cells = odmc.dual_marching_cubes(vol, return_cells=True)
    c = np.array(vol.shape) - 1
    ijk = np.stack(np.unravel_index(cells, tuple(c)), 1)
    above = vol > 0
    corners = [above[dz:dz + c[0], dy:dy + c[1], dx:dx + c[2]] for dz in (0, 1) for dy in (0, 1) for dx in (0, 1)]
    crossed = np.flatnonzero((np.logical_or.reduce(corners) & ~np.logical_and.reduce(corners)).ravel())
    assert (np.diff(cells) >= 0).all() and np.array_equal(np.unique(cells), crossed)
    fin = np.isfinite(v).all(1)
    p = v[fin].astype(np.float64) * c
    assert ((p >= ijk[fin] - 1e-5) & (p <= ijk[fin] + 1 + 1e-5)).all()
    assert fin.all() or np.isnan(vol).any()


def test_plane_through_the_grid_gives_an_open_mesh():
    """A surface that meets the grid's outer faces has no quads there: an open mesh, and vertices of boundary cells
    that no quad references are kept."""
    n = (9, 11, 10)
    z, y, x = np.meshgrid(*[np.arange(k, dtype=np.float32) for k in n], indexing="ij")
    vol = (4.3 - z + 0.31 * y - 0.17 * x).astype(np.float32)
    v, f, cells = odmc.dual_marching_cubes(vol, return_cells=True)
    _, counts, directed_unique = edge_stats(f)
    assert directed_unique and counts.max() == 2 and (counts == 1).any()
    unused = np.setdiff1d(np.arange(len(v)), np.unique(f))
    c = np.array(n) - 1
    ijk = np.stack(np.unravel_index(cells[unused], tuple(c)), 1)
    assert ((ijk == 0) | (ijk == c - 1)).any(1).all()
    # a plane is a disk: V - E + F = 1 over the referenced vertices
    used = len(v) - len(unused)
    assert used - len(counts) + len(f) == 1


def test_no_crossed_cell_raises():
    with pytest.raises(RuntimeError):
        odmc.dual_marching_cubes(np.zeros((5, 5, 5), np.float32))
    with pytest.raises(RuntimeError):
        odmc.dual_marching_cubes(np.full((4, 5, 6), np.nan, np.float32))
    v, f = odmc.dual_marching_cubes(np.array([[[1, -1], [-1, -1]], [[-1, -1], [-1, 1]]], np.float32))
    assert v.shape == (2, 3) and f.shape == (0, 3)       # one cell, two patches, no interior edge


def test_patch_table_is_additions_only_and_matches_the_generator():
    """The generated header gains the two dual arrays; the patch of every edge equals a union-find over the tiling."""
    import os
    import re
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    import gen_mc_tables as G
    text = open(os.path.join(root, "include", "r3g_mc_tables.h")).read()

    def arr(name):
        body = re.search(name + r"\[\d+\] = \{(.*?)\};", text, re.S).group(1)
        return [int(t) for t in body.replace("\n", "").split(",") if t.strip()]
    start, tri = arr("r3g_mc_tiling_start"), arr("r3g_mc_tri")
    patch, npatch = arr("r3g_mc_dual_patch"), arr("r3g_mc_dual_npatch")
    assert len(npatch) == len(start) - 1 and len(patch) == 12 * len(npatch)
    assert max(npatch) == 4 and text.index("r3g_mc_dual_patch") > text.index("r3g_mc_slice")
    for til in range(len(npatch)):
        tt = tri[start[til]:start[til + 1]]
        p, k = G.dual_patches([tt[i:i + 3] for i in range(0, len(tt), 3)])
        assert patch[12 * til:12 * til + 12] == p and npatch[til] == k
