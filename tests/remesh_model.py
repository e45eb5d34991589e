"""float64 numpy model of the parallel remesher of csrc/ls_remesh.cu (largesteps_b200.remesh.remesh_botsch), stage by stage and
round by round, for tests/test_remesh_model.py and tests/test_gpu_remesh_botsch.py.

Meshes are (verts float32 (V, 3), faces int64 (F, 3)); a dead face is a row of -1 between a collapse round and compact().
Every float64 expression is evaluated in the order the kernels write it (the library is built with -fmad=false there), so
split, collapse, flip and compact agree with the device bit for bit, and relax up to the projection's choice among
equidistant faces.

    topology(faces, V)                         corner buckets, edges (a < b, by a then b), edge faces, face edges
    split(v, f, high)                          one pass: every edge longer than high at its midpoint
    collapse_round(v, f, low, high, live)      one round of independent local-minimum collapses -> (v, f, count)
    compact(v, f)                              drop dead faces and unreferenced vertices, order kept
    flip_round(v, f)                           one round of independent valence-improving flips -> (f, count)
    relax(v, f, V0, F0)                        Jacobi tangential relaxation, projected onto (V0, F0)
    remesh(v, f, iters, h, project)            the whole call
"""
import numpy as np

import distance_model

NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _mid(a, b):
    return (0.5 * (a + b)).astype(np.float32).astype(np.float64)


def _cos(n, m):
    with np.errstate(invalid="ignore", divide="ignore"):
        return _dot(n, m) / (np.sqrt(_dot(n, n)) * np.sqrt(_dot(m, m)))


class Topo:
    def __init__(self, faces, V):
        faces = np.asarray(faces, np.int64)
        self.faces, self.V = faces, V
        live = np.flatnonzero(faces[:, 0] >= 0)
        items = (4 * live[:, None] + np.arange(3)[None, :]).ravel()
        keys = faces[live].ravel()
        order = np.lexsort((items, keys))
        self.inc = items[order]
        self.inc_ptr = np.searchsorted(keys[order], np.arange(V + 1))
        self.valence = np.diff(self.inc_ptr)
        f, c = live.repeat(3), np.tile(np.arange(3), len(live))
        a, b = faces[f, c], faces[f, (c + 1) % 3]
        directed = dict(zip((a * V + b).tolist(), f.tolist()))
        fwd = a < b
        eorder = np.lexsort((b[fwd], a[fwd]))
        self.ev = np.stack([a[fwd][eorder], b[fwd][eorder]], 1)
        back = np.array([directed[int(y) * V + int(x)] for x, y in self.ev], np.int64).reshape(-1)
        self.ef = np.stack([f[fwd][eorder], back], 1)
        self.E = len(self.ev)
        self.eid = {int(x) * V + int(y): e for e, (x, y) in enumerate(self.ev.tolist())}
        self.fe = np.full((len(faces), 3), -1, np.int64)
        for k in range(3):
            x, y = faces[live, k], faces[live, (k + 1) % 3]
            lo, hi = np.minimum(x, y), np.maximum(x, y)
            self.fe[live, k] = [self.eid[int(p) * V + int(q)] for p, q in zip(lo, hi)]

    def corners(self, x):
        """For the vertices x (array): (owner position in x, corner item) of each of their corners, in bucket order."""
        x = np.asarray(x, np.int64)
        cnt = self.valence[x]
        owner = np.repeat(np.arange(len(x)), cnt)
        start = np.repeat(self.inc_ptr[x] - np.concatenate([[0], np.cumsum(cnt)[:-1]]), cnt)
        return owner, self.inc[start + np.arange(cnt.sum())]

    def nxt(self, item):
        return self.faces[item >> 2, ((item & 3) + 1) % 3]

    def prv(self, item):
        return self.faces[item >> 2, ((item & 3) + 2) % 3]

    def neighbours(self, x):
        s, e = self.inc_ptr[x], self.inc_ptr[x + 1]
        return self.nxt(self.inc[s:e])


def check(faces, V):
    """The BAD_* bits of ls_remesh_check."""
    faces = np.asarray(faces, np.int64)
    if (faces < 0).any() or (faces >= V).any():
        return 16
    bad = 0
    if ((faces[:, 0] == faces[:, 1]) | (faces[:, 1] == faces[:, 2]) | (faces[:, 2] == faces[:, 0])).any():
        bad |= 8
    cnt = {}
    for k in range(3):
        for x, y in zip(faces[:, k].tolist(), faces[:, (k + 1) % 3].tolist()):
            cnt[(x, y)] = cnt.get((x, y), 0) + 1
    for (x, y), n in cnt.items():
        m = cnt.get((y, x), 0)
        if x == y:
            continue
        if n + m == 1:
            bad |= 1
        elif n + m > 2:
            bad |= 2
        elif n != 1:
            bad |= 4
    return bad


def split(verts, faces, high):
    v = np.asarray(verts, np.float32)
    f = np.asarray(faces, np.int64).copy()
    V, F = len(v), len(f)
    t = Topo(f, V)
    p = v.astype(np.float64)
    d = p[t.ev[:, 0]] - p[t.ev[:, 1]]
    flag = _dot(d, d) > high * high
    rank = np.concatenate([[0], np.cumsum(flag)])
    n = int(rank[-1])
    newv = _mid(p[t.ev[flag, 0]], p[t.ev[flag, 1]]).astype(np.float32)
    out = np.concatenate([f, np.zeros((2 * n, 3), np.int64)])
    for fi in np.flatnonzero(flag[t.fe].any(1)):
        vv = f[fi]
        m, slots = [-1, -1, -1], []
        for k in range(3):
            e = t.fe[fi, k]
            if flag[e]:
                m[k] = V + rank[e]
                slots.append(F + 2 * rank[e] + (0 if t.ef[e, 0] == fi else 1))
        ns = len(slots)
        if ns == 1:
            k = [i for i in range(3) if m[i] >= 0][0]
            a, b, c = vv[k], vv[(k + 1) % 3], vv[(k + 2) % 3]
            tris = [(a, m[k], c), (m[k], b, c)]
        elif ns == 2:
            u = [i for i in range(3) if m[i] < 0][0]
            c, a, b = vv[u], vv[(u + 1) % 3], vv[(u + 2) % 3]
            m0, m1 = m[(u + 1) % 3], m[(u + 2) % 3]
            q0, q1 = _mid(p[a], p[b]), _mid(p[b], p[c])
            tris = [(m0, b, m1)]
            if _dot(p[a] - q1, p[a] - q1) <= _dot(q0 - p[c], q0 - p[c]):
                tris += [(a, m0, m1), (a, m1, c)]
            else:
                tris += [(a, m0, c), (m0, m1, c)]
        else:
            tris = [(m[0], m[1], m[2]), (vv[0], m[0], m[2]), (m[0], vv[1], m[1]), (m[2], m[1], vv[2])]
        out[fi] = tris[0]
        for s, tri in zip(slots, tris[1:]):
            out[s] = tri
    return np.concatenate([v, newv]), out, n


def collapse_round(verts, faces, low, high, live):
    v = np.asarray(verts, np.float32).copy()
    f = np.asarray(faces, np.int64).copy()
    t = Topo(f, len(v))
    p = v.astype(np.float64)
    a, b = t.ev[:, 0], t.ev[:, 1]
    pa, pb = p[a], p[b]
    d = pa - pb
    l2 = _dot(d, d)
    cand = np.flatnonzero(l2 < low * low) if live > 4 else np.zeros(0, np.int64)
    cand = cand[~((t.valence[a[cand]] == 3) & (t.valence[b[cand]] == 3))]      # an edge of a lone tetrahedron
    ok = np.ones(len(cand), bool)
    pm = _mid(pa[cand], pb[cand])
    for x, y in ((a[cand], b[cand]), (b[cand], a[cand])):
        own, it = t.corners(x)
        n, q = t.nxt(it), t.prv(it)
        dn = p[n] - pm[own]
        ok[own[(n != y[own]) & (_dot(dn, dn) > high * high)]] = False
        keep = (n != y[own]) & (q != y[own])
        px = p[x[own]]
        before = _cross(p[n] - px, p[q] - px)
        after = _cross(p[n] - pm[own], p[q] - pm[own])
        ok[own[keep & ~(_cos(before, after) >= 0.5)]] = False
    for i, e in enumerate(cand):
        if ok[i]:
            na, nb = t.neighbours(a[e]), t.neighbours(b[e])
            ok[i] = int((na[:, None] == nb[None, :]).sum()) == 2
    cand = cand[ok]
    keys = (np.sqrt(l2[cand]).astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | cand.astype(np.uint64)
    claim = np.full(len(v), NO_KEY, np.uint64)
    regions = []
    for e, k in zip(cand, keys):
        reg = np.concatenate([[a[e], b[e]], t.neighbours(a[e]), t.neighbours(b[e])])
        regions.append(reg)
        np.minimum.at(claim, reg, k)
    wins = [e for e, k, reg in zip(cand, keys, regions) if (claim[reg] == k).all()]
    for e in wins:
        x, y = a[e], b[e]
        v[x] = _mid(p[x], p[y]).astype(np.float32)
        for it in t.inc[t.inc_ptr[y]:t.inc_ptr[y + 1]]:
            fi, c = it >> 2, it & 3
            if (f[fi] == x).any():
                f[fi] = -1
            else:
                f[fi, c] = x
    return v, f, len(wins)


def compact(verts, faces):
    f = np.asarray(faces, np.int64)
    f = f[f[:, 0] >= 0]
    used = np.zeros(len(verts), bool)
    used[f.ravel()] = True
    vmap = np.cumsum(used) - 1
    return np.asarray(verts, np.float32)[used], vmap[f]


def _dev6(x):
    return np.abs(x - 6)


def flip_round(verts, faces):
    f = np.asarray(faces, np.int64).copy()
    t = Topo(f, len(verts))
    p = np.asarray(verts, np.float32).astype(np.float64)
    a, b = t.ev[:, 0], t.ev[:, 1]

    def third(fi):
        x, y, z = f[fi, 0], f[fi, 1], f[fi, 2]
        return np.where((x != a) & (x != b), x, np.where((y != a) & (y != b), y, z))

    c, d = third(t.ef[:, 0]), third(t.ef[:, 1])
    va, vb, vc, vd = (t.valence[x] for x in (a, b, c, d))
    gain = (_dev6(va) + _dev6(vb) + _dev6(vc) + _dev6(vd)) - (_dev6(va - 1) + _dev6(vb - 1) + _dev6(vc + 1) + _dev6(vd + 1))
    ok = (gain > 0) & (c != d)
    V = len(p)
    lo, hi = np.minimum(c, d), np.maximum(c, d)
    ok &= ~np.isin(lo * V + hi, a * V + b)
    pa, pb, pc, pd = p[a], p[b], p[c], p[d]
    n0, n1 = _cross(pb - pa, pc - pa), _cross(pa - pb, pd - pb)
    g0, g1 = _cross(pd - pa, pc - pa), _cross(pb - pd, pc - pd)
    ok &= (_dot(g0, g0) != 0) & (_dot(g1, g1) != 0)
    for g in (g0, g1):
        for n in (n0, n1):
            ok &= _cos(g, n) >= 0.5
    cand = np.flatnonzero(ok)
    keys = ((8 - gain[cand]).astype(np.uint64) << np.uint64(32)) | cand.astype(np.uint64)
    claim = np.full(V, NO_KEY, np.uint64)
    reg = np.stack([a[cand], b[cand], c[cand], d[cand]], 1)
    np.minimum.at(claim, reg.ravel(), np.repeat(keys, 4))
    win = cand[(claim[reg] == keys[:, None]).all(1)]
    f[t.ef[win, 0]] = np.stack([a[win], d[win], c[win]], 1)
    f[t.ef[win, 1]] = np.stack([d[win], b[win], c[win]], 1)
    return f, len(win)


def relax_unprojected(verts, faces):
    """The float32 positions of k_relax, before the projection."""
    f = np.asarray(faces, np.int64)
    t = Topo(f, len(verts))
    p = np.asarray(verts, np.float32).astype(np.float64)
    fn = _cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
    V = len(p)
    q, n = np.zeros((V, 3)), np.zeros((V, 3))
    for j in range(int(t.valence.max())):
        m = np.flatnonzero(t.valence > j)
        it = t.inc[t.inc_ptr[m] + j]
        q[m] = q[m] + p[t.nxt(it)]
        n[m] = n[m] + fn[it >> 2]
    k = t.valence.astype(np.float64)[:, None]
    q = q / k
    nl = np.sqrt(_dot(n, n))[:, None]
    n = n / nl
    d = p - q
    tt = _dot(n, d)[:, None]
    return (p - (d - n * tt)).astype(np.float32)


def relax(verts, faces, V0, F0):
    r = relax_unprojected(verts, faces)
    return distance_model.point_mesh(r, V0, F0)[2].astype(np.float32)


def remesh(verts, faces, iters, h, project=True):
    v, f = compact(verts, faces)
    V0, F0 = v.copy(), f.copy()
    high, low = 1.4 * h, 0.7 * h
    for _ in range(iters):
        v, f, _n = split(v, f, high)
        live = len(v)
        while True:
            v, f, n = collapse_round(v, f, low, high, live)
            live -= n
            if n == 0:
                break
        v, f = compact(v, f)
        while True:
            f, n = flip_round(v, f)
            if n == 0:
                break
        if not project:
            V0, F0 = v.copy(), f.copy()
        v = relax(v, f, V0, F0)
    return v, f


def euler(verts, faces):
    f = np.asarray(faces, np.int64)
    e = len({(min(x, y), max(x, y)) for k in range(3) for x, y in zip(f[:, k].tolist(), f[:, (k + 1) % 3].tolist())})
    return len(verts) - e + len(f)


def assert_invariants(verts, faces, chi):
    """Closed, edge-manifold, consistently oriented, Euler characteristic chi, no zero-area face, no unreferenced vertex, no NaN."""
    v, f = np.asarray(verts, np.float64), np.asarray(faces, np.int64)
    assert check(f, len(v)) == 0
    assert euler(v, f) == chi
    assert np.isfinite(v).all()
    assert np.array_equal(np.unique(f), np.arange(len(v)))
    n = _cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert (_dot(n, n) > 0).all()
