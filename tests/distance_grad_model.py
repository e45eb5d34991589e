"""float64 numpy model of the backward of point-to-mesh squared distances (ls_distance_grad_f32, largesteps_b200.distance), for
tests/test_distance_grad_model.py, tests/test_distance_grad_host.py and tests/test_gpu_distance_grad.py.

    weights(p, a, b, c)               beta (..., 3): the weights of the closest point on (a, b, c), from the Voronoi regions of
                                      distance_model.closest_on_triangle (a degenerate triangle: its segments ab, bc, ca, the
                                      first strictly nearer one wins)
    grads(P, V, F, I, C, g)           (grad P, grad V) of sum_q g[q] sqrD[q] given the query's (I, C):
                                        grad P[q] = 2 g[q] (P[q] - C[q])
                                        grad V[k] += -2 g[q] beta_k (P[q] - C[q]) for each corner k of face I[q]
                                      rows with I = -1 get NaN in grad P and add nothing to grad V
"""
import numpy as np

import distance_model as dm


def _segment_t(p, a, b):
    ab, ap = b - a, p - a
    den = dm._dot(ab, ab)
    with np.errstate(invalid="ignore", divide="ignore"):
        t = np.where(den > 0, dm._dot(ap, ab) / np.where(den > 0, den, 1.0), 0.0)
    return np.clip(t, 0.0, 1.0)


def weights(p, a, b, c):
    p, a, b, c = (np.asarray(x, np.float64) for x in (p, a, b, c))
    p, a, b, c = np.broadcast_arrays(p, a, b, c)
    ab, ac, ap, bp, cp = b - a, c - a, p - a, p - b, p - c
    n = np.cross(ab, ac)
    degen = dm._dot(n, n) <= dm.DEGENERATE * dm._dot(ab, ab) * dm._dot(ac, ac)
    d1, d2, d3, d4, d5, d6 = (dm._dot(ab, ap), dm._dot(ac, ap), dm._dot(ab, bp), dm._dot(ac, bp), dm._dot(ab, cp),
                              dm._dot(ac, cp))
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    rA = (d1 <= 0) & (d2 <= 0)
    rB = ~rA & (d3 >= 0) & (d4 <= d3)
    rC = ~rA & ~rB & (d6 >= 0) & (d5 <= d6)
    rest = ~(rA | rB | rC)
    rAB = rest & (vc <= 0) & (d1 >= 0) & (d3 <= 0)
    rAC = rest & ~rAB & (vb <= 0) & (d2 >= 0) & (d6 <= 0)
    rBC = rest & ~rAB & ~rAC & (va <= 0) & (d4 - d3 >= 0) & (d5 - d6 >= 0)
    rF = rest & ~(rAB | rAC | rBC)
    beta = np.zeros(p.shape[:-1] + (3,))
    with np.errstate(invalid="ignore", divide="ignore"):
        beta[rA, 0] = 1.0
        beta[rB, 1] = 1.0
        beta[rC, 2] = 1.0
        v = d1 / (d1 - d3)
        beta[rAB, 0], beta[rAB, 1] = 1.0 - v[rAB], v[rAB]
        v = d2 / (d2 - d6)
        beta[rAC, 0], beta[rAC, 2] = 1.0 - v[rAC], v[rAC]
        v = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        beta[rBC, 1], beta[rBC, 2] = 1.0 - v[rBC], v[rBC]
        den = 1.0 / (va + vb + vc)
        v, t = vb * den, vc * den
        beta[rF, 0], beta[rF, 1], beta[rF, 2] = 1.0 - v[rF] - t[rF], v[rF], t[rF]
    if degen.any():
        q, A, B, Cc = p[degen], a[degen], b[degen], c[degen]
        best, _ = dm.closest_on_segment(q, A, B)
        t0 = _segment_t(q, A, B)
        bd = np.stack([1.0 - t0, t0, np.zeros_like(t0)], -1)
        s, _ = dm.closest_on_segment(q, B, Cc)
        t1 = _segment_t(q, B, Cc)
        better = s < best
        best = np.where(better, s, best)
        bd = np.where(better[:, None], np.stack([np.zeros_like(t1), 1.0 - t1, t1], -1), bd)
        s, _ = dm.closest_on_segment(q, Cc, A)
        t2 = _segment_t(q, Cc, A)
        better = s < best
        bd = np.where(better[:, None], np.stack([t2, np.zeros_like(t2), 1.0 - t2], -1), bd)
        beta[degen] = bd
    return beta


def grads(P, V, F, I, C, g):
    """(grad P (n,3), grad V (V,3)) in float64 of sum_q g[q] sqrD[q], from the query's face I and closest point C."""
    P, V, C, g = (np.asarray(x, np.float64) for x in (P, V, C, g))
    F, I = np.asarray(F, np.int64), np.asarray(I, np.int64)
    ok = I >= 0
    d = P - C
    gP = 2.0 * g[:, None] * d
    gP[~ok] = np.nan
    gV = np.zeros_like(V)
    q = np.flatnonzero(ok)
    if len(q):
        f = F[I[q]]
        beta = weights(P[q], V[f[:, 0]], V[f[:, 1]], V[f[:, 2]])
        for k in range(3):
            np.add.at(gV, f[:, k], (-2.0 * g[q] * beta[:, k])[:, None] * d[q])
    return gP, gV


def grad_terms_abs(P, V, F, I, C, g):
    """sum over the terms of each gradient entry of their absolute values: the scale of its rounding error"""
    P, V, C, g = (np.asarray(x, np.float64) for x in (P, V, C, g))
    F, I = np.asarray(F, np.int64), np.asarray(I, np.int64)
    aP = 2.0 * np.abs(g)[:, None] * np.abs(P - C)
    aV = np.zeros_like(V)
    q = np.flatnonzero(I >= 0)
    if len(q):
        f = F[I[q]]
        beta = np.abs(weights(P[q], V[f[:, 0]], V[f[:, 1]], V[f[:, 2]]))
        for k in range(3):
            np.add.at(aV, f[:, k], (2.0 * np.abs(g[q]) * beta[:, k])[:, None] * np.abs(P[q] - C[q]))
    return aP, aV
