"""ORACLE -- test infrastructure only.  numpy mirror of r3g_mesh_decimate (include/r3g.h describes the algorithm,
3d-re-gen_b200/csrc/decimate.cu implements it): the same rounds, vectorised per round, with the same float64 operations in
the same order -- elementwise only, no matmul / einsum / axis reductions whose summation order numpy may choose -- so the
two agree bit for bit.  Importable from tests/ and tools/."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)
MIN_COMPONENT = 4
_LO = np.uint64(0xFFFFFFFF)


def _cross(u, v):
    return np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1],
                     u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                     u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], 1)


def _dot(u, v):
    return (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2]


def _plane(n, d, s):
    """s u u^T for u = (n, d), packed (a2 ab ac ad b2 bc bd c2 cd d2)."""
    u = [n[:, 0], n[:, 1], n[:, 2], d]
    return np.stack([(u[i] * u[j]) * s for i in range(4) for j in range(i, 4)], 1)


def _err(q, p):
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    r0 = ((q[:, 0] * x + q[:, 1] * y) + q[:, 2] * z) + q[:, 3]
    r1 = ((q[:, 1] * x + q[:, 4] * y) + q[:, 5] * z) + q[:, 6]
    r2 = ((q[:, 2] * x + q[:, 5] * y) + q[:, 7] * z) + q[:, 8]
    r3 = ((q[:, 3] * x + q[:, 6] * y) + q[:, 8] * z) + q[:, 9]
    return ((r0 * x + r1 * y) + r2 * z) + r3


def _placement(q, a, b):
    c00 = q[:, 4] * q[:, 7] - q[:, 5] * q[:, 5]
    c01 = q[:, 2] * q[:, 5] - q[:, 1] * q[:, 7]
    c02 = q[:, 1] * q[:, 5] - q[:, 2] * q[:, 4]
    c11 = q[:, 0] * q[:, 7] - q[:, 2] * q[:, 2]
    c12 = q[:, 1] * q[:, 2] - q[:, 0] * q[:, 5]
    c22 = q[:, 0] * q[:, 4] - q[:, 1] * q[:, 1]
    det = (q[:, 0] * c00 + q[:, 1] * c01) + q[:, 2] * c02
    tr = (q[:, 0] + q[:, 4]) + q[:, 7]
    ok = np.abs(det) > ((1e-6 * tr) * tr) * tr
    with np.errstate(divide="ignore", invalid="ignore"):
        solved = np.stack([-((c00 * q[:, 3] + c01 * q[:, 6]) + c02 * q[:, 8]) / det,
                           -((c01 * q[:, 3] + c11 * q[:, 6]) + c12 * q[:, 8]) / det,
                           -((c02 * q[:, 3] + c12 * q[:, 6]) + c22 * q[:, 8]) / det], 1)
    mid = (a + b) * 0.5
    ea, eb, em = _err(q, a), _err(q, b), _err(q, mid)
    use_b = eb < ea
    best = np.where(use_b[:, None], b, a)
    use_m = em < np.where(use_b, eb, ea)
    best = np.where(use_m[:, None], mid, best)
    return np.where(ok[:, None], solved, best)


def _round_up_f32(x):
    """float32 of x rounded towards +inf (x >= 0), as bits."""
    with np.errstate(over="ignore"):
        f = x.astype(np.float32)
    low = f.astype(np.float64) < x
    f[low] = np.nextafter(f[low], np.float32(np.inf))
    return f.view(np.uint32).astype(np.uint64)


def _csr(src, dst, n):
    """CSR of the pairs (src, dst) sorted by (src, dst)."""
    order = np.lexsort((dst, src))
    off = np.zeros(n + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n), out=off[1:])
    return off, dst[order]


def _expand(off, ids):
    """For each id: the positions off[id] .. off[id+1]-1; returns (index into ids, position)."""
    cnt = off[ids + 1] - off[ids]
    rep = np.repeat(np.arange(len(ids)), cnt)
    start = np.repeat(off[ids] - np.cumsum(cnt) + cnt, cnt)
    return rep, start + np.arange(len(rep))


class _Adjacency:
    def __init__(self, F, nv):
        lf = np.flatnonzero(F[:, 0] >= 0)
        u = F[lf].astype(np.int64)
        w = u[:, [1, 2, 0]]
        keys = ((np.minimum(u, w).astype(np.uint64) << np.uint64(32)) | np.maximum(u, w).astype(np.uint64)).ravel()
        vals = (lf[:, None] * 3 + np.arange(3)).ravel()                    # ascending, as the device's input order
        order = np.argsort(keys, kind="stable")
        self.hkey, self.hval = keys[order], vals[order]
        self.ukey, self.estart, self.ecnt = np.unique(self.hkey, return_index=True, return_counts=True)
        self.he_edge = np.empty(3 * len(F), np.int64)
        self.he_edge[self.hval] = np.repeat(np.arange(len(self.ukey)), self.ecnt)
        self.a = (self.ukey >> np.uint64(32)).astype(np.int64)
        self.b = (self.ukey & _LO).astype(np.int64)
        self.boundary = np.zeros(nv, bool)
        self.frozen = np.zeros(nv, bool)
        for flag, sel in ((self.boundary, self.ecnt == 1), (self.frozen, self.ecnt > 2)):
            flag[self.a[sel]] = True
            flag[self.b[sel]] = True
        corner_v = u.ravel()
        corner_f = np.repeat(lf, 3)
        self.vf_off, self.vf = _csr(corner_v, corner_f, nv)
        self.nb_off, self.nb = _csr(np.concatenate([self.a, self.b]), np.concatenate([self.b, self.a]), nv)


def _quadrics(V, F, adj, nv):
    """Per-vertex sums in the device's order: faces ascending, each face's plane then its boundary edges by corner."""
    Fl = F.astype(np.int64)
    rep, pos = _expand(adj.vf_off, np.arange(nv))
    vert, face = rep, adj.vf[pos]
    c = Fl[face]
    p = [V[c[:, j]] for j in range(3)]
    n = _cross(p[1] - p[0], p[2] - p[0])
    nn = _dot(n, n)
    good = nn > 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        fq = _plane(n, -_dot(n, p[0]), 1.0 / np.sqrt(nn))
    seq = [(good, fq)]
    for j in range(3):
        j1 = (j + 1) % 3
        e = p[j1] - p[j]
        m = _cross(e, n)
        mm = _dot(m, m)
        at_v = (c[:, j] == vert) | (c[:, j1] == vert)
        bnd = adj.ecnt[adj.he_edge[face * 3 + j]] == 1
        with np.errstate(divide="ignore", invalid="ignore"):
            bq = _plane(m, -_dot(m, p[j]), (3.0 * _dot(e, e)) / mm)
        seq.append((good & at_v & bnd & (mm > 0.0), bq))
    # interleave: term index = 4 * (position in the vertex's face list) + (0 plane, 1 + j boundary edge j)
    Q = np.zeros((nv, 10))
    rank = pos - adj.vf_off[vert]
    for r in range(int(rank.max()) + 1 if len(rank) else 0):
        at = rank == r
        for use, q in seq:
            sel = at & use
            Q[vert[sel]] = Q[vert[sel]] + q[sel]
    return Q


def _cost(V, F, Q, adj, label, comp_nv):
    """(key per edge, NO_KEY if invalid; placement per edge)."""
    a, b, cnt = adj.a, adj.b, adj.ecnt
    E = len(a)
    valid = (cnt <= 2) & ~adj.frozen[a] & ~adj.frozen[b]
    valid &= ~((cnt == 2) & adj.boundary[a] & adj.boundary[b])
    valid &= comp_nv[label[a]] > MIN_COMPONENT
    # link condition: common neighbours of a and b, counted over a's neighbours x with an edge (b, x)
    rep, pos = _expand(adj.nb_off, a)
    x = adj.nb[pos]
    bb = b[rep]
    k = (np.minimum(bb, x).astype(np.uint64) << np.uint64(32)) | np.maximum(bb, x).astype(np.uint64)
    at = np.searchsorted(adj.ukey, k)
    found = (at < E) & (adj.ukey[np.minimum(at, E - 1)] == k)
    common = np.bincount(rep[found], minlength=E)
    valid &= common == cnt
    ids = np.flatnonzero(valid)
    q = Q[a[ids]] + Q[b[ids]]
    pa, pb = V[a[ids]], V[b[ids]]
    p = _placement(q, pa, pb)
    qmin = np.ones(len(ids))
    flip = np.zeros(len(ids), bool)
    Fl = F.astype(np.int64)
    for s, o in ((a[ids], b[ids]), (b[ids], a[ids])):
        rep, pos = _expand(adj.vf_off, s)
        c = Fl[adj.vf[pos]]
        keep = ~((c[:, 0] == o[rep]) | (c[:, 1] == o[rep]) | (c[:, 2] == o[rep]))
        rep, c = rep[keep], c[keep]
        x = [V[c[:, j]] for j in range(3)]
        y = [np.where((c[:, j] == s[rep])[:, None], p[rep], x[j]) for j in range(3)]
        n0 = _cross(x[1] - x[0], x[2] - x[0])
        e01, e12, e20 = y[1] - y[0], y[2] - y[1], y[0] - y[2]
        n1 = _cross(e01, y[2] - y[0])
        bad = (_dot(n0, n0) > 0.0) & ~(_dot(n0, n1) > 0.0)
        flip |= np.bincount(rep[bad], minlength=len(ids)) > 0
        l2 = (_dot(e01, e01) + _dot(e12, e12)) + _dot(e20, e20)
        with np.errstate(divide="ignore", invalid="ignore"):
            qual = np.where(l2 > 0.0, (np.sqrt(_dot(n1, n1)) * 3.4641016151377544) / l2, 0.0)
        np.minimum.at(qmin, rep, qual)
    qmin = np.where(qmin < 1e-3, 1e-3, qmin)
    err = _err(q, p)
    err = np.where(err > 0.0, err, 0.0)
    ab = pb - pa
    l2 = _dot(ab, ab)
    cost = (err + 1e-4 * (l2 * l2)) / qmin
    keys = np.full(E, NO_KEY, np.uint64)
    ok = ~flip
    keys[ids[ok]] = (_round_up_f32(cost[ok]) << np.uint64(32)) | ids[ok].astype(np.uint64)
    P = np.zeros((E, 3))
    P[ids] = p
    return keys, P


def decimate(verts, faces, target):
    """(verts float32 [V', 3], faces int32 [F', 3], rounds) -- what r3g_mesh_decimate returns for the same input."""
    verts = np.asarray(verts, np.float32)
    F = np.array(faces, np.int64).reshape(-1, 3)
    nv = len(verts)
    if len(F) and (F.min() < 0 or F.max() >= nv):
        raise ValueError("a face index is outside [0, nv)")
    V = verts.astype(np.float64)
    F[(F[:, 0] == F[:, 1]) | (F[:, 1] == F[:, 2]) | (F[:, 0] == F[:, 2])] = -1
    live = int((F[:, 0] >= 0).sum())
    remap = np.arange(nv)
    rounds = 0
    if live > target:
        adj = _Adjacency(F, nv)
        Q = _quadrics(V, F, adj, nv)
        lf = F[F[:, 0] >= 0]
        e = np.concatenate([lf[:, [0, 1]], lf[:, [1, 2]]])
        _, label = connected_components(coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(nv, nv)),
                                        directed=False)
        referenced = adj.vf_off[1:] > adj.vf_off[:-1]
        comp_nv = np.bincount(label[referenced], minlength=nv).astype(np.int64)
        while live > target:
            if rounds:
                adj = _Adjacency(F, nv)
            key, P = _cost(V, F, Q, adj, label, comp_nv)
            a, b = adj.a, adj.b
            m = np.full(nv, NO_KEY, np.uint64)
            val = key != NO_KEY
            np.minimum.at(m, a[val], key[val])
            np.minimum.at(m, b[val], key[val])
            M = m.copy()
            np.minimum.at(M, a, m[b])
            np.minimum.at(M, b, m[a])
            sel = val & (key == M[a]) & (key == M[b])
            c = label[a]
            comp_sel = np.bincount(c[sel], minlength=nv)
            comp_min = np.full(nv, NO_KEY, np.uint64)
            np.minimum.at(comp_min, c[sel], key[sel])
            sel &= (comp_nv[c] - comp_sel[c] >= MIN_COMPONENT) | (key == comp_min[c])
            nsel = int(sel.sum())
            if nsel == 0:
                break
            k = (live - target + 1) // 2
            if nsel > k:
                sel &= key <= np.sort(key[sel])[k - 1]
            ids = np.flatnonzero(sel)
            ka, kb = a[ids], b[ids]
            V[ka] = P[ids]
            Q[ka] = Q[ka] + Q[kb]
            remap[kb] = ka
            rep, pos = _expand(np.append(adj.estart, len(adj.hkey)), ids)
            F[adj.hval[pos] // 3] = -1
            np.subtract.at(comp_nv, label[ka], 1)
            alive = F[:, 0] >= 0
            F[alive] = remap[F[alive]]
            live -= len(pos)
            rounds += 1
    alive = F[:, 0] >= 0
    ref = np.zeros(nv, bool)
    ref[F[alive].ravel()] = True
    new = np.cumsum(ref) - 1
    return V[ref].astype(np.float32), new[F[alive]].astype(np.int32), rounds
