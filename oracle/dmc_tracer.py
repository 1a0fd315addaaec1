"""ORACLE -- test infrastructure only (tests/ may import it; nothing under 3d-re-gen_b200/ may).

A SECOND, independent CPU dual marching cubes (r3g's R3G_MC_DUAL, include/r3g.h).  It does NOT read
include/r3g_mc_tables.h: the tiling of every crossed cell is traced from the rules by oracle/mc_tracer.py, its patches
are a union-find over the vertices of the traced triangles, and the quads are assembled from a dict keyed by grid edge
(array axis, lower grid point) that collects the (cell, vertex) pairs around each edge.  The four cells of a quad are
put in turn order by the angle of their centres about the edge, and the quad's owner and order are derived from the
cells themselves, not from an edge-ownership table.  tests/test_dmc_oracle.py checks oracle/dmc_oracle.c == this
tracer bit for bit (vertices, faces, order).  Pure Python over the crossed cells: use it on small volumes.
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mc_tracer  # noqa: E402
from mc_tracer import G  # noqa: E402  (rule code of tools/gen_mc_tables.py; the generated header is not used)


def _patches(tris):
    """Connected components of the triangles (shared vertices, centre 12 included): {cube edge: patch}, numbered by
    the smallest cube edge of each patch."""
    par = {}

    def find(a):
        par.setdefault(a, a)
        while par[a] != a:
            a = par[a]
        return a
    for t in tris:
        for v in t:
            ra, rb = find(t[0]), find(v)
            if ra != rb:
                par[rb] = ra
    edges = sorted({v for t in tris for v in t if v != 12})
    ids, out = {}, {}
    for e in edges:
        out[e] = ids.setdefault(find(e), len(ids))
    return out


def dual_marching_cubes(volume, level=0.0):
    vol = np.ascontiguousarray(volume, dtype=np.float32)
    n = vol.shape
    lvl = np.float64(np.float32(level))
    above = vol > np.float32(level)
    c0, c1, c2 = n[0] - 1, n[1] - 1, n[2] - 1
    corners = [above[o[2]:o[2] + c0, o[1]:o[1] + c1, o[0]:o[0] + c2] for o in G.CORNER]
    crossed = np.logical_or.reduce(corners) & ~np.logical_and.reduce(corners)
    verts, by_edge, vsign = [], {}, {}
    with np.errstate(divide="ignore", invalid="ignore"):
        for z, y, x in np.argwhere(crossed):          # traversal order: z, y, x with x fastest
            z, y, x = int(z), int(y), int(x)
            cv = [np.float64(vol[z + o[2], y + o[1], x + o[0]]) - lvl for o in G.CORNER]
            ci = sum((1 << i) for i in range(8) if cv[i] > 0)
            tris, _ = mc_tracer._cell_triangles(ci, cv)
            patch = _patches(tris)
            first = len(verts)
            for p in range(max(patch.values()) + 1):
                s = [np.float64(0.0)] * 3
                k = 0
                for e in sorted(patch):
                    if patch[e] != p:
                        continue
                    a, b = G.EDGE[e]
                    pa, pb = G.CORNER[a], G.CORNER[b]
                    t = cv[a] / (cv[a] - cv[b])
                    for d, (org, ax) in enumerate(((z, 2), (y, 1), (x, 0))):
                        qa, qb = np.float64(org + pa[ax]), np.float64(org + pb[ax])
                        s[d] = s[d] + (qa + t * (qb - qa))
                    k += 1
                verts.append([np.float32(s[d] / np.float64(k) / np.float64(n[d] - 1)) for d in range(3)])
            for e, p in patch.items():
                a, b = G.EDGE[e]
                pa, pb = G.CORNER[a], G.CORNER[b]
                axis = 2 - [i for i in range(3) if pa[i] != pb[i]][0]        # array axis of the edge
                lo = (z + min(pa[2], pb[2]), y + min(pa[1], pb[1]), x + min(pa[0], pb[0]))
                by_edge.setdefault((axis, lo), []).append(((z, y, x), first + p))
                hi = list(lo)
                hi[axis] += 1
                vsign[(axis, lo)] = bool(vol[tuple(hi)] > np.float32(level))
    if not verts:
        raise RuntimeError("No surface found at the given iso value.")
    v = np.array(verts, np.float32).reshape(-1, 3)
    quads = []
    for (axis, lo), cells in by_edge.items():
        if len(cells) != 4:                            # an edge on the grid's outer faces
            continue
        b, c = (axis + 1) % 3, (axis + 2) % 3          # right-handed (b, c, axis)
        # counter-clockwise about +axis: increasing angle of the cell centres around the edge, from the first cell
        ang = [math.atan2(cell[c] + 0.5 - lo[c], cell[b] + 0.5 - lo[b]) for cell, _ in cells]
        ring = [cells[i] for i in np.argsort(ang)]
        start = min(range(4), key=lambda i: ring[i][0])
        ring = ring[start:] + ring[:start]
        q = [vid for _, vid in ring]
        if not vsign[(axis, lo)]:                      # the normal must point to the upper end only if it is above
            q = [q[0], q[3], q[2], q[1]]
        quads.append((ring[0][0], axis, q))
    quads.sort(key=lambda r: (r[0], r[1]))
    faces = []
    for _, _, q in quads:
        def d2(i, j):
            dd = [np.float64(v[i, k]) - np.float64(v[j, k]) for k in range(3)]
            return dd[0] * dd[0] + dd[1] * dd[1] + dd[2] * dd[2]
        if d2(q[1], q[3]) < d2(q[0], q[2]):
            faces += [[q[0], q[1], q[3]], [q[1], q[2], q[3]]]
        else:
            faces += [[q[0], q[1], q[2]], [q[0], q[2], q[3]]]
    return v, np.array(faces, np.int32).reshape(-1, 3)
