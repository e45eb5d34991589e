"""CPU: the float64 gradient model of tests/distance_grad_model.py against central differences of distance_model.brute_force,
for points well inside one Voronoi region of a lone triangle (face, each edge, each vertex), on the segments of a degenerate
triangle, and on a small closed mesh away from ties.  Loss: sum_q G[q] sqrD[q] with seeded G."""
import numpy as np
import pytest

import distance_grad_model as gm
import distance_model as dm
from largesteps_b200 import workloads


def loss(P, V, F, G):
    return float((dm.brute_force(P, V, F)[0] * G).sum())


def central(P, V, F, G, h):
    gP, gV = np.zeros_like(P), np.zeros_like(V)
    for X, out in ((P, gP), (V, gV)):
        for idx in np.ndindex(*X.shape):
            x0 = X[idx]
            X[idx] = x0 + h
            up = loss(P, V, F, G)
            X[idx] = x0 - h
            dn = loss(P, V, F, G)
            X[idx] = x0
            out[idx] = (up - dn) / (2 * h)
    return gP, gV


def check(P, V, F, h, seed=0):
    P, V = np.asarray(P, np.float64), np.asarray(V, np.float64)
    G = np.random.default_rng(seed).uniform(0.5, 2.0, len(P)) * np.random.default_rng(seed + 1).choice([-1, 1], len(P))
    _, I, C = dm.brute_force(P, V, F)
    aP, aV = gm.grads(P, V, F, I, C, G)
    fP, fV = central(P.copy(), V.copy(), F, G, h)
    for a, f in ((aP, fP), (aV, fV)):
        np.testing.assert_allclose(a, f, rtol=1e-6, atol=1e-6 * np.abs(a).max())
    return I


TRI = np.array([[0.1, -0.05, 0.02], [1.2, 0.1, -0.1], [0.2, 0.9, 0.15]])


@pytest.mark.parametrize("region,point", [
    ("face", [0.45, 0.35, 0.6]),
    ("ab", [0.6, -0.6, 0.3]),
    ("ac", [-0.5, 0.5, -0.2]),
    ("bc", [1.1, 0.9, 0.4]),
    ("a", [-0.7, -0.6, 0.5]),
    ("b", [2.0, -0.4, -0.3]),
    ("c", [0.0, 1.9, 0.6]),
])
def test_lone_triangle_regions(region, point):
    F = np.array([[0, 1, 2]])
    P = np.array([point], np.float64)
    beta = gm.weights(P, *TRI[None].transpose(1, 0, 2))[0]
    want = {"face": (1, 1, 1), "ab": (1, 1, 0), "ac": (1, 0, 1), "bc": (0, 1, 1), "a": (1, 0, 0), "b": (0, 1, 0),
            "c": (0, 0, 1)}[region]
    assert tuple(int(x) for x in beta > 1e-3) == want, beta
    check(P, TRI, F, 1e-6)


def test_weights_reproduce_the_closest_point():
    rng = np.random.default_rng(2)
    tri = rng.normal(size=(5000, 3, 3))
    p = rng.normal(size=(5000, 3)) * 2
    _, c = dm.closest_on_triangle(p, tri[:, 0], tri[:, 1], tri[:, 2])
    beta = gm.weights(p, tri[:, 0], tri[:, 1], tri[:, 2])
    np.testing.assert_allclose(beta.sum(1), 1.0, rtol=0, atol=1e-14)
    np.testing.assert_allclose((beta[:, :, None] * tri).sum(1), c, rtol=0, atol=1e-12)


@pytest.mark.parametrize("point,seg", [([0.5, 1.0, 0.3], "ca"), ([0.5, -1.0, 0.3], "ab"), ([1.5, 1.0, -0.2], "bc")])
def test_degenerate_triangle_segments(point, seg):
    """A sliver below the degenerate threshold (sine 1e-6 at a): its three segments differ by ~1e-6 in squared distance, so
    the segment picked stays picked under a 1e-8 step, and the triangle stays degenerate."""
    V = np.array([[0.0, 0.0, 0.0], [2.0, 0.0, 0.0], [1.0, 1e-6, 0.0]])
    F = np.array([[0, 1, 2]])
    P = np.array([point])
    beta = gm.weights(P, V[0], V[1], V[2])[0]
    zero = {"ab": 2, "bc": 0, "ca": 1}[seg]
    assert beta[zero] == 0.0 and (np.delete(beta, zero) > 0.1).all(), beta
    check(P, V, F, 1e-8)


def test_small_mesh_away_from_ties():
    v, f = workloads.icosphere(1)
    V = v.astype(np.float64) * np.array([1.0, 0.8, 1.2])
    rng = np.random.default_rng(4)
    d = rng.normal(size=(400, 3))
    P = d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(0.6, 1.5, (400, 1)) * np.array([1.0, 0.8, 1.2])
    # keep points whose nearest face is nearer than every other by a margin (no tie under the step)
    qi, fi = np.repeat(np.arange(len(P)), len(f)), np.tile(np.arange(len(f)), len(P))
    s = dm.closest_on_triangle(P[qi], V[f[fi, 0]], V[f[fi, 1]], V[f[fi, 2]])[0].reshape(len(P), len(f))
    s.sort(1)
    P = P[(s[:, 1] - s[:, 0]) > 1e-4][:30]
    assert len(P) >= 20
    I = check(P, V, f, 1e-6, seed=3)
    assert len(np.unique(I)) >= 10
