"""float64 numpy model of point-to-mesh distances and the mesh Hausdorff distance (libigl's point_mesh_squared_distance and
hausdorff), for tests/test_distance_model.py, tests/test_distance_host.py and tests/test_gpu_distance.py.

    closest_on_triangle(p, a, b, c)   vectorised closest point (Ericson's Voronoi regions; a degenerate triangle is its
                                      three segments, by the rule of csrc/ls_distance.cu)
    brute_force(P, V, F)              every face for every point (small meshes)
    point_mesh(P, V, F)               exact, with candidates from a cKDTree of the referenced vertices: the nearest vertex
                                      at distance d_v bounds the answer, and a face that holds a point at <= d_v has every
                                      corner within d_v + L_max (L_max the longest edge), so only faces at those vertices count
    hausdorff(VA, FA, VB, FB)         sqrt(max(max_a sqrD(a, B), max_b sqrD(b, A))) over every row of VA and VB
Ties: among faces at an equal float64 distance the lowest index wins.
"""
import numpy as np
from scipy.spatial import cKDTree

DEGENERATE = 2.0 ** -36   # LS_DIST_DEGENERATE


def _dot(u, v):
    return u[..., 0] * v[..., 0] + u[..., 1] * v[..., 1] + u[..., 2] * v[..., 2]


def closest_on_segment(p, a, b):
    ab, ap = b - a, p - a
    den = _dot(ab, ab)
    with np.errstate(invalid="ignore", divide="ignore"):
        t = np.where(den > 0, _dot(ap, ab) / np.where(den > 0, den, 1.0), 0.0)
    t = np.clip(t, 0.0, 1.0)
    c = a + t[..., None] * ab
    return _dot(p - c, p - c), c


def closest_on_triangle(p, a, b, c):
    """(sqrD, C) for arrays of points p and corners a, b, c of shape (..., 3), in float64."""
    p, a, b, c = (np.asarray(x, np.float64) for x in (p, a, b, c))
    p, a, b, c = np.broadcast_arrays(p, a, b, c)
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    n = np.cross(ab, ac)
    degen = _dot(n, n) <= DEGENERATE * _dot(ab, ab) * _dot(ac, ac)
    d1, d2, d3, d4, d5, d6 = _dot(ab, ap), _dot(ac, ap), _dot(ab, bp), _dot(ac, bp), _dot(ab, cp), _dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    rA = (d1 <= 0) & (d2 <= 0)
    rB = ~rA & (d3 >= 0) & (d4 <= d3)
    rC = ~rA & ~rB & (d6 >= 0) & (d5 <= d6)
    rest = ~(rA | rB | rC)
    rAB = rest & (vc <= 0) & (d1 >= 0) & (d3 <= 0)
    rAC = rest & ~rAB & (vb <= 0) & (d2 >= 0) & (d6 <= 0)
    rBC = rest & ~rAB & ~rAC & (va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0)
    rF = rest & ~(rAB | rAC | rBC)
    out = np.empty_like(p)
    with np.errstate(invalid="ignore", divide="ignore"):
        out[rA], out[rB], out[rC] = a[rA], b[rB], c[rC]
        v = d1 / (d1 - d3)
        out[rAB] = a[rAB] + v[rAB, None] * ab[rAB]
        v = d2 / (d2 - d6)
        out[rAC] = a[rAC] + v[rAC, None] * ac[rAC]
        v = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        out[rBC] = b[rBC] + v[rBC, None] * (c[rBC] - b[rBC])
        den = 1.0 / (va + vb + vc)
        out[rF] = a[rF] + ab[rF] * (vb * den)[rF, None] + ac[rF] * (vc * den)[rF, None]
    s = _dot(p - out, p - out)
    if degen.any():
        best, cb = closest_on_segment(p[degen], a[degen], b[degen])
        for u, w in ((b, c), (c, a)):
            s2, c2 = closest_on_segment(p[degen], u[degen], w[degen])
            better = s2 < best
            best = np.where(better, s2, best)
            cb = np.where(better[:, None], c2, cb)
        s[degen], out[degen] = best, cb
    return s, out


def _pick(qidx, fidx, s, c, n):
    """Per query the least s, ties to the lowest face index: (sqrD, I, C) of n queries."""
    order = np.lexsort((fidx, s, qidx))
    first = np.ones(len(order), bool)
    first[1:] = qidx[order][1:] != qidx[order][:-1]
    sel = order[first]
    sqrD = np.full(n, np.nan)
    I = np.full(n, -1, np.int64)
    C = np.full((n, 3), np.nan)
    sqrD[qidx[sel]], I[qidx[sel]], C[qidx[sel]] = s[sel], fidx[sel], c[sel]
    return sqrD, I, C


def brute_force(P, V, F, chunk=1 << 20):
    P, V, F = np.asarray(P, np.float64), np.asarray(V, np.float64), np.asarray(F, np.int64)
    n, nf = len(P), len(F)
    out = []
    step = max(1, chunk // max(nf, 1))
    for s0 in range(0, n, step):
        q = np.arange(s0, min(n, s0 + step))
        qi, fi = np.repeat(q, nf), np.tile(np.arange(nf), len(q))
        s, c = closest_on_triangle(P[qi], V[F[fi, 0]], V[F[fi, 1]], V[F[fi, 2]])
        out.append(_pick(qi - s0, fi, s, c, len(q)))
    return tuple(np.concatenate([o[k] for o in out]) for k in range(3))


def point_mesh(P, V, F, chunk=1 << 21):
    P, V, F = np.asarray(P, np.float64), np.asarray(V, np.float64), np.asarray(F, np.int64)
    n = len(P)
    nan = np.isnan(P).any(axis=1)
    used = np.unique(F)
    tree = cKDTree(V[used])
    E = np.concatenate([V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 1]], V[F[:, 0]] - V[F[:, 2]]])
    lmax = float(np.sqrt(_dot(E, E).max()))
    good = np.flatnonzero(~nan)
    dv, _ = tree.query(P[good])
    # vertex -> incident faces (CSR)
    vf = np.repeat(np.arange(len(F)), 3)
    order = np.argsort(F.ravel(), kind="stable")
    ptr = np.searchsorted(F.ravel()[order], np.arange(len(V) + 1))
    inc = vf[order]
    sqrD = np.full(n, np.nan)
    I = np.full(n, -1, np.int64)
    C = np.full((n, 3), np.nan)
    radius = (dv + lmax) * (1 + 1e-9) + 1e-300
    balls = tree.query_ball_point(P[good], radius)
    qs, fs = [], []
    for k, b in enumerate(balls):
        vs = used[np.asarray(b, np.int64)]
        f = np.unique(np.concatenate([inc[ptr[v]:ptr[v + 1]] for v in vs]))
        qs.append(np.full(len(f), good[k]))
        fs.append(f)
    if not qs:
        return sqrD, I, C
    qi, fi = np.concatenate(qs), np.concatenate(fs)
    for s0 in range(0, len(qi), chunk):
        q, f = qi[s0:s0 + chunk], fi[s0:s0 + chunk]
        s, c = closest_on_triangle(P[q], V[F[f, 0]], V[F[f, 1]], V[F[f, 2]])
        d, i, cc = _pick(q, f, s, c, n)
        hit = i >= 0
        better = hit & ((I < 0) | (d < sqrD) | ((d == sqrD) & (i < I)))
        sqrD[better], I[better], C[better] = d[better], i[better], cc[better]
    return sqrD, I, C


def hausdorff(VA, FA, VB, FB):
    a = point_mesh(VA, VB, FB)[0]
    b = point_mesh(VB, VA, FA)[0]
    m = max(a.max(), b.max())     # NaN-propagating
    return float(np.sqrt(m))
