#!/usr/bin/env python
"""Generate the marching-cubes tiling tables used by BOTH the CPU oracle (oracle/mc_oracle.c)
and the CUDA kernels (3d-re-gen_b200/csrc/mc.cu).

Why generated and not transcribed: the reference calls scikit-image's Lewiner marching cubes
(Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/surface_extractors.py:69-73); scikit-image and
its `_marching_cubes_lewiner_luts.py` are NOT in /root/reference nor in this image, and Lewiner's
LookUpTable.h cannot be reproduced from memory.  What CAN be restated from the published
algorithm (Lewiner et al. 2003, Chernyaev 1995, Nielson-Hamann 1991) is the structure:

  * Lewiner's cube numbering (corners v0..v7, edges e0..e11, centre vertex 12, faces 1..6),
  * cubeindex = sum((v_i - level) > 0) << i,
  * ambiguous faces resolved by the bilinear-saddle face test (Lewiner `test_face`),
  * every sign-changing cube edge carries exactly one vertex, polygons of >= 8 vertices
    are tiled around the centre vertex (as Lewiner's 7.3/10.2/12.2/13.3/13.4 tilings do).

The tables here are DERIVED from those rules: for every cubeindex and every outcome of the face
tests on its ambiguous faces we trace the iso-contour segments on the six faces, chain them into
closed loops and triangulate each loop.  Where Lewiner's big switch applies `test_interior` (sub-cases 4.1,
6.1, 7.4, 10.1, 12.1, 13.5) a second, "tunnel" tiling (4.1.2, 6.1.2, 7.4.2, 10.1.2, 12.1.2, 13.5.2: the two loops
joined by a tube instead of capped separately) is generated together with the descriptor of the interior test
(slice direction / reference edge and the sign whose connectivity is asked); the test itself (Lewiner's
`test_interior`, restated from the published routine) runs in the oracle and in the kernel.  What is still NOT
Lewiner's: the literal triangle order / diagonal choice of LookUpTable.h and the reference-edge column of his
TEST6/7/12 and TILING13_5_1 tables (chosen here by a stated rule) -- see DESIGN.md section 4.

Output: include/r3g_mc_tables.h (plain C arrays, included by the oracle and by the kernels).
"""
import itertools
import os
import sys

CORNER = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
EDGE = [(0, 1), (1, 2), (2, 3), (3, 0), (4, 5), (5, 6), (6, 7), (7, 4), (0, 4), (1, 5), (2, 6), (3, 7)]
# Lewiner's face list (test_face): corners A,B,C,D in cyclic order; A,C and B,D are the diagonals.
FACE = [(0, 4, 5, 1), (1, 5, 6, 2), (2, 6, 7, 3), (3, 7, 4, 0), (0, 3, 2, 1), (4, 7, 6, 5)]
EDGE_OF = {}
for ei, (a, b) in enumerate(EDGE):
    EDGE_OF[(a, b)] = ei
    EDGE_OF[(b, a)] = ei


def cross(u, v):
    return (u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0])


def sub(u, v):
    return tuple(a - b for a, b in zip(u, v))


def dot(u, v):
    return sum(a * b for a, b in zip(u, v))


def ccw_from_outside(face):
    """Return the face's corners ordered counter-clockwise when seen from outside the cube."""
    p = [CORNER[c] for c in face]
    n = cross(sub(p[1], p[0]), sub(p[2], p[1]))
    centre = tuple(sum(q[i] for q in p) / 4.0 for i in range(3))
    outward = sub(centre, (0.5, 0.5, 0.5))
    return list(face) if dot(n, outward) > 0 else list(face[::-1])


FACE_CCW = [ccw_from_outside(f) for f in FACE]


def face_segments(ci, face_ccw, pos_connected):
    """Oriented iso-segments (edge_from, edge_to) on one face, positive region on the LEFT when the
    face is seen from outside the cube."""
    s = [(ci >> c) & 1 for c in face_ccw]
    npos = sum(s)
    segs = []
    if npos == 0 or npos == 4:
        return segs
    ambiguous = npos == 2 and s[0] == s[2]
    if ambiguous and pos_connected:
        # positive band through the centre: cut off each NEGATIVE corner c_k,
        # segment runs edge(c_{k-1},c_k) -> edge(c_k,c_{k+1})
        for k in range(4):
            if s[k] == 0:
                e_in = EDGE_OF[(face_ccw[(k - 1) % 4], face_ccw[k])]
                e_out = EDGE_OF[(face_ccw[k], face_ccw[(k + 1) % 4])]
                segs.append((e_in, e_out))
        return segs
    # every maximal CCW arc of positive corners c_i..c_j is cut off by one segment running
    # edge(c_j,c_{j+1}) -> edge(c_{i-1},c_i)
    for i in range(4):
        if s[i] == 1 and s[(i - 1) % 4] == 0:
            j = i
            while s[(j + 1) % 4] == 1:
                j = (j + 1) % 4
            e_from = EDGE_OF[(face_ccw[j], face_ccw[(j + 1) % 4])]
            e_to = EDGE_OF[(face_ccw[(i - 1) % 4], face_ccw[i])]
            segs.append((e_from, e_to))
    return segs


def ambiguous_faces(ci):
    out = []
    for fi, f in enumerate(FACE):
        s = [(ci >> c) & 1 for c in f]
        if sum(s) == 2 and s[0] == s[2]:
            out.append(fi)
    return out


def loops_for(ci, decisions):
    """decisions: dict face_index -> pos_connected (only for ambiguous faces)."""
    nxt = {}
    for fi in range(6):
        for (a, b) in face_segments(ci, FACE_CCW[fi], decisions.get(fi, False)):
            assert a not in nxt, "edge starts two segments"
            nxt[a] = b
    # every crossing edge must start exactly one segment and end exactly one
    crossing = [ei for ei, (a, b) in enumerate(EDGE) if ((ci >> a) & 1) != ((ci >> b) & 1)]
    assert sorted(nxt.keys()) == crossing, (ci, decisions, nxt, crossing)
    assert sorted(nxt.values()) == crossing
    loops, seen = [], set()
    for e in crossing:  # increasing edge id => loops sorted by their smallest edge, started there
        if e in seen:
            continue
        lp, cur = [], e
        while cur not in seen:
            seen.add(cur)
            lp.append(cur)
            cur = nxt[cur]
        assert cur == e
        loops.append(lp)
    return loops


def edges_share_face(e1, e2):
    a, b = set(EDGE[e1]), set(EDGE[e2])
    return any(a <= set(f) and b <= set(f) for f in FACE)


def polygon_triangulations(P):
    """All triangulations of the polygon P (vertex list, orientation preserved), fan-like ones first."""
    if len(P) < 3:
        return [[]]
    if len(P) == 3:
        return [[tuple(P)]]
    out = []
    for k in range(len(P) - 2, 0, -1):
        for left in polygon_triangulations(P[:k + 1]):
            for right in polygon_triangulations(P[k:]):
                out.append([(P[0], P[k], P[-1])] + left + right)
    return out


def triangulate(loops):
    """Triangulate every loop.  A diagonal joining two polygon vertices that lie on a common cube face
    would be generated identically by the neighbouring cell (4 triangles on one edge, flat sliver pairs), so
    only triangulations without such diagonals are admissible -- the same constraint Lewiner's hand-built
    tilings satisfy.  Polygons with no admissible triangulation, and all polygons of >= 8 vertices, are
    tiled around the centre vertex (id 12)."""
    tris = []
    for lp in loops:
        n = len(lp)
        assert n >= 3
        # The loops are traced with the positive region on the left (normal towards increasing values in the
        # core's (x,y,z) frame).  scikit-image returns vertices in array-axis order (z,y,x) -- a reflection --
        # and its default gradient_direction='descent' output has right-hand normals pointing towards
        # INCREASING values (the reason export_to_trimesh flips the faces, pipelines.py:102).  So in the
        # core frame the stored winding is the reverse of the traced one.
        lp = [lp[0]] + lp[:0:-1]
        chosen = None
        if n < 8:
            for cand in polygon_triangulations(lp):
                ok = True
                for (a, b, c) in cand:
                    for (u, v) in ((a, b), (b, c), (c, a)):
                        iu, iv = lp.index(u), lp.index(v)
                        adjacent = (iu - iv) % n in (1, n - 1)
                        if not adjacent and edges_share_face(u, v):
                            ok = False
                if ok:
                    chosen = cand
                    break
        if chosen is None:
            chosen = [(lp[i], lp[(i + 1) % n], 12) for i in range(n)]
        tris.extend(chosen)
    return tris


ANTIPODE = [CORNER.index(tuple(1 - c for c in p)) for p in CORNER]


def surface_classes(ci, decisions):
    """Union-find over the 8 corners: same-sign corners joined by a cube edge, or across an ambiguous face by
    the face decision (pos_connected joins its two positive corners, otherwise its two negative ones)."""
    par = list(range(8))

    def find(a):
        while par[a] != a:
            par[a] = par[par[a]]
            a = par[a]
        return a

    def join(a, b):
        par[find(a)] = find(b)
    sg = [(ci >> i) & 1 for i in range(8)]
    for (a, b) in EDGE:
        if sg[a] == sg[b]:
            join(a, b)
    for fi, pc in decisions.items():
        f = FACE[fi]
        want = 1 if pc else 0
        pair = [c for c in f if sg[c] == want]
        assert len(pair) == 2
        join(pair[0], pair[1])
    return [find(i) for i in range(8)], sg


def loop_around(loops, ci, corners):
    """The loop made exactly of the cube edges leaving the corner set `corners` (edges with one end inside)."""
    want = sorted(ei for ei, (a, b) in enumerate(EDGE) if (a in corners) != (b in corners))
    for i, lp in enumerate(loops):
        if sorted(lp) == want:
            return i
    return None


def interior_test(ci, decisions, loops):
    """Where Lewiner's switch calls test_interior: returns (mode, ref_edge, sigma, loop_a, loop_b) or None.
    mode 1 = the closed-form slice height along z (cases 4 and 10), mode 2 = slice through the iso-crossing of a
    reference edge (cases 6, 7, 12, 13).  sigma = 1: the question is whether two POSITIVE corners are joined through
    the interior, 0: two negative ones.  loop_a / loop_b: the loops the tunnel tiling joins."""
    base = mc_case(ci)
    if base not in (4, 6, 7, 10, 12, 13):
        return None
    cls, sg = surface_classes(ci, decisions)
    if base == 13:
        # 13.5: three faces around a corner N decide for N's opposite sign; N and its antipode are each cut off by
        # a triangle, the rest is a hexagon (13.5.1).  The interior question is asked for the isolated corner of the
        # configuration's own sign convention: positive for cubeindex 165 (corners 0,2,5,7), negative for its inverse.
        if sum(1 for v in decisions.values() if v) != 3 or sorted(len(lp) for lp in loops) != [3, 3, 6]:
            return None
        sigma = 1 if ci == 165 else 0
        iso = [c for c in range(8) if sg[c] == sigma and sum(1 for d in range(8) if cls[d] == cls[c]) == 1]
        assert len(iso) == 1, (ci, decisions, iso)
        P = iso[0]
        la = loop_around(loops, ci, {P})
        lb = [i for i, lp in enumerate(loops) if len(lp) == 6][0]
        return (2, ref_edge_at(P, ci, None), sigma, la, lb)
    cands = []
    for P in range(8):
        Q = ANTIPODE[P]
        if P < Q and sg[P] == sg[Q] and cls[P] != cls[Q]:
            cands.append((P, Q))
    if base in (10, 12):
        cands = [(P, Q) for (P, Q) in cands if sg[P] == 1]   # Lewiner tests the positive polarity only (TEST10/12 > 0)
    if not cands:
        return None
    assert len(loops) == 2, (ci, decisions, loops)
    sigma = sg[cands[0][0]]
    assert all(sg[P] == sigma for P, _ in cands)
    if base in (4, 10):
        return (1, 15, sigma, 0, 1)
    # reference edge: at the corner of the pair that is alone in its class (all three cube edges there cross)
    P, Q = cands[0]
    size = lambda c: sum(1 for d in range(8) if cls[d] == cls[c])  # noqa: E731
    if size(P) != 1:
        P, Q = Q, P
    assert size(P) == 1, (ci, decisions)
    amb_with_P = [fi for fi in decisions if P in FACE[fi] and Q not in FACE[fi]]
    face = None
    if base in (6, 12):
        # the face whose test sent us here contains P and a corner of Q's class on its diagonal
        face = [fi for fi in decisions if P in FACE[fi]]
        assert len(face) >= 1
        face = face[0] if base == 6 else face
    return (2, ref_edge_at(P, ci, face), sigma, 0, 1)


def ref_edge_at(P, ci, faces):
    """Reference edge of the slice test: a crossing cube edge at corner P; among those lying on the tested
    ambiguous face(s) (if given) the one along the highest axis (z > y > x).  This reproduces the two rows of
    Lewiner's TEST6 that could be recalled ({2,7,10} for corners 0,1,6 and {4,7,11} for 0,1,7); the full column is
    not reconstructible without the table."""
    if faces is not None and not isinstance(faces, (list, tuple)):
        faces = [faces]
    best = None
    for ei, (a, b) in enumerate(EDGE):
        if P not in (a, b):
            continue
        if ((ci >> a) & 1) == ((ci >> b) & 1):
            continue
        if faces is not None and not any(a in FACE[f] and b in FACE[f] for f in faces):
            continue
        axis = [i for i in range(3) if CORNER[a][i] != CORNER[b][i]][0]
        if best is None or axis > best[0]:
            best = (axis, ei)
    assert best is not None, (P, ci, faces)
    return best[1]


def _mid(e):
    if e == 12:
        return (0.5, 0.5, 0.5)
    return tuple((CORNER[EDGE[e][0]][i] + CORNER[EDGE[e][1]][i]) / 2 for i in range(3))


def tunnel(loop_a, loop_b):
    """Triangulate the tube between two loops (the 4.1.2 / 6.1.2 / 7.4.2 / 10.1.2 / 12.1.2 / 13.5.2 tilings): a strip
    of len(a) + len(b) triangles that walks loop_a forwards and loop_b backwards.  Both loops are given in the STORED
    winding (see triangulate), which is the boundary orientation the tube needs: a strip triangle covers the boundary
    edge a_i -> a_{i+1} (or b_{j-1} -> b_j) in that direction.  Preference: fewest rungs lying in a cube face (7.4.2
    has no strip without one: each vertex of the triangle sees only two hexagon vertices off its faces), then least
    total rung length between edge midpoints; ties by enumeration order, so the table is deterministic."""
    A, B = loop_a, loop_b
    m, n = len(A), len(B)

    def cone_free(steps):
        # n retreats (or m advances) in a row, cyclically, would fan a whole loop around one vertex: a closed cone
        N = len(steps)
        for want, lim in ((True, m), (False, n)):
            run = best_run = 0
            for k in range(2 * N):
                run = run + 1 if steps[k % N] == want else 0
                best_run = max(best_run, run)
            if best_run >= lim:
                return False
        return True

    def d(u, v):
        return sum((a - b) ** 2 for a, b in zip(_mid(u), _mid(v))) ** 0.5
    best = None
    for j0 in range(n):
        # state (i, j): current rung A[i] -- B[j]; advance A: tri (A[i], A[i+1], B[j]); retreat B: tri (B[j-1], B[j], A[i])
        for mask in itertools.combinations(range(m + n), m):
            steps = [k in mask for k in range(m + n)]
            if not cone_free(steps):
                continue
            i, j, tris, cost, in_face = 0, j0, [], 0.0, 0
            for adv in steps:
                u, v = A[i % m], B[j % n]
                in_face += 1 if edges_share_face(u, v) else 0
                cost += d(u, v)
                if adv:
                    tris.append((u, A[(i + 1) % m], v))
                    i += 1
                else:
                    tris.append((B[(j - 1) % n], v, u))
                    j -= 1
            key = (in_face, round(cost, 9))
            if best is None or key < best[0]:
                best = (key, tris)
    assert best is not None, "no tunnel strip"
    return best[1]


def stored(lp):
    """Traced loop -> stored winding (see the comment in triangulate)."""
    return [lp[0]] + lp[:0:-1]


DUAL_NO_PATCH = 255


def dual_patches(tris):
    """Dual marching cubes: the connected components ("patches") of one tiling's triangles, joined through shared
    vertices (cube edges and the centre vertex 12).  Returns (patch of each of the 12 cube edges, DUAL_NO_PATCH for an
    edge the tiling does not use; number of patches), patches numbered in increasing order of their smallest edge."""
    par = list(range(13))

    def find(a):
        while par[a] != a:
            par[a] = par[par[a]]
            a = par[a]
        return a
    used = set()
    for t in tris:
        used.update(t)
        for v in t[1:]:
            par[find(v)] = find(t[0])
    patch, ids = [DUAL_NO_PATCH] * 12, {}
    for e in range(12):
        if e in used:
            patch[e] = ids.setdefault(find(e), len(ids))
    return patch, len(ids)


def mc_case(ci):
    """Lorensen/Chernyaev/Lewiner base-case number 0..14 of a cube index (shape invariant)."""
    def shape(bits):
        pts = [CORNER[i] for i in range(8) if (bits >> i) & 1]
        d = sorted(sum(abs(a - b) for a, b in zip(p, q)) for p, q in itertools.combinations(pts, 2))
        return len(pts), tuple(d)
    n, d = shape(ci)
    if n > 4:
        n, d = shape(ci ^ 0xFF)
    if n == 0:
        return 0
    if n == 1:
        return 1
    if n == 2:
        return {1: 2, 2: 3, 3: 4}[d[0]]
    if n == 3:
        return {(1, 1, 2): 5, (1, 2, 3): 6, (2, 2, 2): 7}[d]
    # n == 4
    table = {
        (1, 1, 1, 1, 2, 2): 8,    # four corners of a face
        (1, 1, 1, 2, 2, 2): 9,    # corner + its three neighbours
        (1, 1, 2, 2, 3, 3): 10,   # two opposite parallel edges
        (1, 1, 2, 2, 2, 3): 12,   # L on a face + the corner diagonal to the L's elbow
        (2, 2, 2, 2, 2, 2): 13,   # tetrahedral
        (1, 1, 1, 2, 2, 3): 11,   # zig-zag (11 and its mirror 14)
    }
    c = table[d]
    if c == 11:
        # chirality: 11 vs 14.  Path a-b-c-d of three unit steps; sign of the triple product.
        pts = [i for i in range(8) if (ci >> i) & 1]
        if len(pts) != 4:
            pts = [i for i in range(8) if not (ci >> i) & 1]
        adj = {p: [q for q in pts if q != p and sum(abs(a - b) for a, b in zip(CORNER[p], CORNER[q])) == 1]
               for p in pts}
        ends = [p for p in pts if len(adj[p]) == 1]
        a = min(ends)
        b = adj[a][0]
        cc = [q for q in adj[b] if q != a][0]
        dd = [q for q in adj[cc] if q != b][0]
        t = dot(cross(sub(CORNER[b], CORNER[a]), sub(CORNER[cc], CORNER[b])), sub(CORNER[dd], CORNER[cc]))
        # chirality convention anchored on Lewiner's table: cubeindex 23 (corners 0,1,2,4) is case 11
        c = 14 if t > 0 else 11
    return c


def main(out_path):
    amb_mask = [0] * 256
    offset = [0] * 256
    tiling_start = [0]
    tri = []
    ntil = 0
    case = [mc_case(ci) for ci in range(256)]
    interior = []      # per tiling: 0 = no interior test, else mode | ref_edge << 2 | sigma << 6
    tunnel_of = []     # per tiling: index of the tunnel tiling chosen when the interior test says "connected"
    pending = []       # (tiling index, loops, la, lb) whose tunnel tilings are appended after the face-test tilings
    for ci in range(256):
        amb = ambiguous_faces(ci)
        m = 0
        for f in amb:
            m |= 1 << f
        amb_mask[ci] = m
        offset[ci] = ntil
        for sub_id in range(1 << len(amb)):
            dec = {f: bool((sub_id >> j) & 1) for j, f in enumerate(amb)}
            loops = loops_for(ci, dec)
            t = triangulate(loops)
            for (a, b, c) in t:
                tri.extend((a, b, c))
            tiling_start.append(len(tri))
            it = interior_test(ci, dec, loops)
            if it is None:
                interior.append(0)
            else:
                mode, edge, sigma, la, lb = it
                interior.append(mode | (edge << 2) | (sigma << 6))
                pending.append((ntil, loops, la, lb))
            tunnel_of.append(0xFFFF)
            ntil += 1
    n_face_tilings = ntil
    for (til, loops, la, lb) in pending:
        t = tunnel(stored(loops[la]), stored(loops[lb]))
        rest = [lp for i, lp in enumerate(loops) if i not in (la, lb)]
        t = t + triangulate(rest)
        for (a, b, c) in t:
            tri.extend((a, b, c))
        tiling_start.append(len(tri))
        tunnel_of[til] = ntil
        interior.append(0)
        tunnel_of.append(0xFFFF)
        ntil += 1
    # --- self checks -------------------------------------------------------------------------
    # (1) single positive corner v0: in the core (x,y,z) frame the normal points AWAY from v0.
    t0 = tri[tiling_start[offset[1]]:tiling_start[offset[1] + 1]]
    mid = lambda e: tuple((CORNER[EDGE[e][0]][i] + CORNER[EDGE[e][1]][i]) / 2 for i in range(3))
    a, b, c = (mid(e) for e in t0)
    nrm = cross(sub(b, a), sub(c, a))
    assert dot(nrm, sub(CORNER[0], a)) < 0, "orientation self-check failed"
    # (2) per tiling: each directed cube-surface... every polygon edge interior to the cell is used
    #     twice with opposite directions; boundary (cube-face) segments once.
    for til in range(ntil):
        tt = tri[tiling_start[til]:tiling_start[til + 1]]
        half = {}
        for k in range(0, len(tt), 3):
            v = tt[k:k + 3]
            for i in range(3):
                key = (v[i], v[(i + 1) % 3])
                assert key not in half, "duplicate directed edge in tiling"
                half[key] = 1
    # (3) a tunnel tiling replaces its face-test tiling inside the same cell: same boundary (the directed edges used
    #     once), so the neighbouring cells see no difference
    def boundary(til):
        tt = tri[tiling_start[til]:tiling_start[til + 1]]
        d = set()
        for k in range(0, len(tt), 3):
            v = tt[k:k + 3]
            for i in range(3):
                d.add((v[i], v[(i + 1) % 3]))
        return {e for e in d if (e[1], e[0]) not in d}
    for til in range(n_face_tilings):
        if tunnel_of[til] != 0xFFFF:
            assert interior[til] != 0
            assert boundary(til) == boundary(tunnel_of[til]), "tunnel tiling changes the cell boundary"
    max_tris = max(tiling_start[i + 1] - tiling_start[i] for i in range(ntil)) // 3
    with open(out_path, "w") as f:
        w = f.write
        w("/* GENERATED by tools/gen_mc_tables.py -- do not edit.\n")
        w(" * Marching-cubes tables restated from the published Lewiner/Chernyaev rules (face tests + interior tests);\n")
        w(" * replaces scikit-image's _marching_cubes_lewiner_luts (third-party, not in the reference tree),\n")
        w(" * call site Hunyuan3D-2/hy3dgen/shapegen/models/autoencoders/surface_extractors.py:69-73. */\n")
        w("#ifndef R3G_MC_TABLES_H\n#define R3G_MC_TABLES_H\n")
        w("#ifndef R3G_MC_TABLE_QUAL\n#define R3G_MC_TABLE_QUAL static const\n#endif\n")
        w(f"#define R3G_MC_NUM_TILINGS {ntil}\n#define R3G_MC_NUM_FACE_TILINGS {n_face_tilings}\n")
        w(f"#define R3G_MC_TRI_ENTRIES {len(tri)}\n#define R3G_MC_MAX_TRIS {max_tris}\n")
        w("/* scikit-image's `FLT_EPSILON = np.spacing(1.0)` (_marching_cubes_lewiner_cy.pyx; SURVEY.md Appendix A.5): the\n")
        w(" * one tiny constant of the vertex weights 1/(eps+|v|), of test_face and of test_internal -- 2^-52, not the\n")
        w(" * float32 epsilon of Lewiner's C++ (1.19e-7).  Shared by the oracle and the kernels. */\n")
        w("#define R3G_MC_EPS 2.220446049250313e-16\n")

        def arr(ctype, name, data, per=16):
            w(f"R3G_MC_TABLE_QUAL {ctype} {name}[{len(data)}] = {{\n")
            for i in range(0, len(data), per):
                w("  " + ",".join(str(x) for x in data[i:i + per]) + ",\n")
            w("};\n")
        arr("unsigned char", "r3g_mc_case", case)
        arr("unsigned char", "r3g_mc_amb_faces", amb_mask)
        arr("unsigned short", "r3g_mc_tiling_offset", offset)
        arr("unsigned short", "r3g_mc_tiling_start", tiling_start)
        arr("unsigned char", "r3g_mc_tri", tri, per=24)
        # interior test per tiling (0 = none): bits 0..1 mode (1 = closed-form slice along z: cases 4 / 10,
        # 2 = slice through the crossing of a reference edge: cases 6 / 7 / 12 / 13), bits 2..5 reference edge,
        # bit 6 sigma (1: are two POSITIVE corners joined through the interior, 0: two negative ones);
        # r3g_mc_tunnel[t] = tiling used instead of t when the answer is "joined" (0xFFFF = none)
        arr("unsigned char", "r3g_mc_interior", interior)
        arr("unsigned short", "r3g_mc_tunnel", tunnel_of)
        # geometry helpers
        arr("unsigned char", "r3g_mc_edge_corner", [c for e in EDGE for c in e], per=2)
        arr("unsigned char", "r3g_mc_corner_xyz", [c for p in CORNER for c in p], per=3)
        arr("unsigned char", "r3g_mc_face_corner", [c for fc in FACE for c in fc], per=4)
        # per edge: bit0..2 = (x,y,z) offset of the lower endpoint, bits 3..4 = axis the edge runs along
        info = []
        for (a, b) in EDGE:
            pa, pb = CORNER[a], CORNER[b]
            lo = [min(pa[i], pb[i]) for i in range(3)]
            axis = [i for i in range(3) if pa[i] != pb[i]][0]
            info.append(lo[0] | (lo[1] << 1) | (lo[2] << 2) | (axis << 3))
        arr("unsigned char", "r3g_mc_edge_info", info, per=12)
        # slice of the interior test through the iso-crossing of reference edge e = (u, w) (Lewiner test_interior,
        # `case 6/7/12/13`): the three parallel cube edges (b0,b1), (c0,c1), (d0,d1) in the direction u -> w, with
        # (c0,c1) the one diagonal to e in the slice: At = 0, Bt = v[b0] + (v[b1]-v[b0]) t, ...; t = v[u] / (v[u] - v[w])
        sl = []
        for (u, wv) in EDGE:
            pu, pw = CORNER[u], CORNER[wv]
            axis = [i for i in range(3) if pu[i] != pw[i]][0]
            lo, hi = [i for i in range(3) if i != axis]

            def flip(p, axes):
                q = list(p)
                for a_ in axes:
                    q[a_] = 1 - q[a_]
                return CORNER.index(tuple(q))
            for axes in ((lo,), (lo, hi), (hi,)):
                sl.extend((flip(pu, axes), flip(pw, axes)))
        arr("unsigned char", "r3g_mc_slice", sl, per=6)
        # dual marching cubes: per tiling, the patch (connected component of its triangles) of each cube edge, numbered
        # by smallest edge, 255 = edge not crossed; and the number of patches = the vertices the cell gives
        dual_patch, dual_npatch = [], []
        for til in range(ntil):
            tt = tri[tiling_start[til]:tiling_start[til + 1]]
            p, n = dual_patches([tt[k:k + 3] for k in range(0, len(tt), 3)])
            dual_patch.extend(p)
            dual_npatch.append(n)
        arr("unsigned char", "r3g_mc_dual_patch", dual_patch, per=12)
        arr("unsigned char", "r3g_mc_dual_npatch", dual_npatch)
        w("#endif\n")
    print(f"tilings={ntil} (tunnel {ntil - n_face_tilings}) tri_entries={len(tri)} max_tris={max_tris}", file=sys.stderr)


if __name__ == "__main__":
    here = os.path.dirname(os.path.abspath(__file__))
    main(os.path.join(here, "..", "include", "r3g_mc_tables.h"))
