"""float64 numpy model of the adaptive remesher (remesh_botsch with a per-vertex target t and feature vertices), stage by stage,
built on the rounds of tests/remesh_model.py, for tests/test_remesh_adaptive_model.py and tests/test_gpu_remesh_adaptive.py.

Each vertex carries vhigh = 1.4 t and vlow = 0.7 t (float64) and a feature flag (bool).  Every float64 expression rounds as
the kernels write it, so split, collapse, flip and compact agree with the device bit for bit, attributes included.

    split(v, f, vhigh, vlow, feature)            -> (v, f, count, (vhigh, vlow, feature))
    collapse_round(v, f, live, vhigh, vlow, feature)  -> (v, f, count); the survivor keeps its bounds, so they do not change
    compact(v, f, vhigh, vlow, feature)          -> (v, f, (vhigh, vlow, feature))
    flip_round(v, f, feature)                    -> (f, count)
    relax(v, f, V0, F0, feature)                 -> v; a feature vertex keeps its position
    remesh(v, f, iters, t, project, feature)     -> (v, f, feature mask of the output)

split and collapse_round run remesh_model's rounds with per-edge bounds: an edge's bound is the mean of its ends' bounds, and
an edge at a feature gets a bound that never passes.  Collapse's ring test (every neighbour of an end x within vhigh[x] of
the midpoint) depends on the end, so it is applied here, and an edge that fails it gets the bound 0.
"""
import numpy as np

import remesh_model as RM


def _edges(verts, faces):
    t = RM.Topo(faces, len(verts))
    return t, t.ev[:, 0], t.ev[:, 1], np.asarray(verts, np.float32).astype(np.float64)


def split(verts, faces, vhigh, vlow, feature):
    t, a, b, p = _edges(verts, faces)
    high = np.where(feature[a] | feature[b], np.inf, (vhigh[a] + vhigh[b]) / 2)
    v, f, n = RM.split(verts, faces, high)                              # remesh_model compares |ab|^2 > high * high per edge
    d = p[a] - p[b]
    flag = RM._dot(d, d) > high * high
    ea, eb = a[flag], b[flag]
    return v, f, n, (np.concatenate([vhigh, (vhigh[ea] + vhigh[eb]) / 2]), np.concatenate([vlow, (vlow[ea] + vlow[eb]) / 2]),
                     np.concatenate([feature, np.zeros(n, bool)]))


def collapse_round(verts, faces, live, vhigh, vlow, feature):
    t, a, b, p = _edges(verts, faces)
    d = p[a] - p[b]
    lo = (vlow[a] + vlow[b]) / 2
    cand = np.flatnonzero((RM._dot(d, d) < lo * lo) & ~(feature[a] | feature[b]))
    ok = np.ones(len(cand), bool)
    pm = RM._mid(p[a[cand]], p[b[cand]])
    for x, y in ((a[cand], b[cand]), (b[cand], a[cand])):
        own, it = t.corners(x)
        n = t.nxt(it)
        dn = p[n] - pm[own]
        hx = vhigh[x[own]]
        ok[own[(n != y[own]) & (RM._dot(dn, dn) > hx * hx)]] = False
    low = np.zeros(t.E)
    low[cand[ok]] = lo[cand[ok]]
    return RM.collapse_round(verts, faces, low, np.inf, live)           # its own ring test never fails at high = inf


def compact(verts, faces, vhigh, vlow, feature):
    f = np.asarray(faces, np.int64)
    used = np.zeros(len(verts), bool)
    used[f[f[:, 0] >= 0].ravel()] = True
    v, f = RM.compact(verts, faces)
    return v, f, (vhigh[used], vlow[used], feature[used])


def flip_round(verts, faces, feature):
    """remesh_model.flip_round without the candidates whose a, b, c or d is a feature."""
    f = np.asarray(faces, np.int64).copy()
    t = RM.Topo(f, len(verts))
    p = np.asarray(verts, np.float32).astype(np.float64)
    a, b = t.ev[:, 0], t.ev[:, 1]

    def third(fi):
        x, y, z = f[fi, 0], f[fi, 1], f[fi, 2]
        return np.where((x != a) & (x != b), x, np.where((y != a) & (y != b), y, z))

    c, d = third(t.ef[:, 0]), third(t.ef[:, 1])
    va, vb, vc, vd = (t.valence[x] for x in (a, b, c, d))
    dev6 = RM._dev6
    gain = (dev6(va) + dev6(vb) + dev6(vc) + dev6(vd)) - (dev6(va - 1) + dev6(vb - 1) + dev6(vc + 1) + dev6(vd + 1))
    ok = (gain > 0) & (c != d) & ~(feature[a] | feature[b] | feature[c] | feature[d])
    V = len(p)
    lo, hi = np.minimum(c, d), np.maximum(c, d)
    ok &= ~np.isin(lo * V + hi, a * V + b)
    pa, pb, pc, pd = p[a], p[b], p[c], p[d]
    n0, n1 = RM._cross(pb - pa, pc - pa), RM._cross(pa - pb, pd - pb)
    g0, g1 = RM._cross(pd - pa, pc - pa), RM._cross(pb - pd, pc - pd)
    ok &= (RM._dot(g0, g0) != 0) & (RM._dot(g1, g1) != 0)
    for g in (g0, g1):
        for n in (n0, n1):
            ok &= RM._cos(g, n) >= 0.5
    cand = np.flatnonzero(ok)
    keys = ((8 - gain[cand]).astype(np.uint64) << np.uint64(32)) | cand.astype(np.uint64)
    claim = np.full(V, RM.NO_KEY, np.uint64)
    reg = np.stack([a[cand], b[cand], c[cand], d[cand]], 1)
    np.minimum.at(claim, reg.ravel(), np.repeat(keys, 4))
    win = cand[(claim[reg] == keys[:, None]).all(1)]
    f[t.ef[win, 0]] = np.stack([a[win], d[win], c[win]], 1)
    f[t.ef[win, 1]] = np.stack([d[win], b[win], c[win]], 1)
    return f, len(win)


def relax(verts, faces, V0, F0, feature):
    r = RM.relax(verts, faces, V0, F0)
    r[feature] = np.asarray(verts, np.float32)[feature]
    return r


def remesh(verts, faces, iters, t, project=True, feature=None):
    """t: a scalar or a (V,) array of targets; feature: a (V,) bool mask or None."""
    t = np.broadcast_to(np.asarray(t, np.float64), (len(verts),))
    mask = np.zeros(len(verts), bool) if feature is None else np.asarray(feature, bool)
    v, f, (vh, vl, ft) = compact(verts, faces, 1.4 * t, 0.7 * t, mask)
    V0, F0 = v.copy(), f.copy()
    for _ in range(iters):
        v, f, _n, (vh, vl, ft) = split(v, f, vh, vl, ft)
        live = len(v)
        while True:
            v, f, n = collapse_round(v, f, live, vh, vl, ft)
            live -= n
            if n == 0:
                break
        v, f, (vh, vl, ft) = compact(v, f, vh, vl, ft)
        while True:
            f, n = flip_round(v, f, ft)
            if n == 0:
                break
        if not project:
            V0, F0 = v.copy(), f.copy()
        v = relax(v, f, V0, F0, ft)
    return v, f, ft
