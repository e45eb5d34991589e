"""CPU: the numpy model of the parallel remesher (tests/remesh_model.py) keeps its invariants on hand-made closed meshes and on
noisy icospheres and the bunny."""
import numpy as np
import pytest

import remesh_model as RM
from largesteps_b200 import workloads


def octahedron():
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float32)
    f = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]], np.int64)
    return v, f


def ico(scale_vertex=1.0):
    v, f = workloads.icosahedron()
    v = np.asarray(v, np.float32).copy()
    v[0] *= scale_vertex
    return v, np.asarray(f, np.int64)


def noisy(v, f, amp, seed=0):
    e = v[f[:, 1]] - v[f[:, 0]]
    mean = float(np.linalg.norm(e, axis=1).mean())
    return (v + np.random.default_rng(seed).normal(size=v.shape) * amp * mean).astype(np.float32), f, mean


def mean_edge(v, f):
    return float(np.linalg.norm(v[f[:, 1]] - v[f[:, 0]], axis=1).mean())


def test_check_flags():
    v, f = octahedron()
    assert RM.check(f, 6) == 0
    assert RM.check(f[1:], 6) & 1                                       # open
    assert RM.check(np.concatenate([f, f[:1, ::-1]]), 6) & 2            # three faces on an edge
    g = f.copy()
    g[0] = g[0, ::-1]
    assert RM.check(g, 6) & 4                                           # one face turned over
    assert RM.check(f, 5) == 16


def test_octahedron_rejects_every_flip():
    v, f = octahedron()
    g, n = RM.flip_round(v, f)
    assert n == 0 and np.array_equal(g, f)


def test_topology_numbers_edges_by_endpoints():
    v, f = octahedron()
    t = RM.Topo(f, 6)
    assert t.E == 12 and (t.ev[:, 0] < t.ev[:, 1]).all()
    keys = t.ev[:, 0] * 6 + t.ev[:, 1]
    assert (np.diff(keys) > 0).all()
    for e, (a, b) in enumerate(t.ev):
        f0, f1 = f[t.ef[e, 0]], f[t.ef[e, 1]]
        assert any(f0[k] == a and f0[(k + 1) % 3] == b for k in range(3))
        assert any(f1[k] == b and f1[(k + 1) % 3] == a for k in range(3))


def test_split_counts():
    v, f = octahedron()
    h = 0.5                                                             # every edge (sqrt 2) is longer than 1.4 h
    v2, f2, n = RM.split(v, f, 1.4 * h)
    assert n == 12 and len(v2) == 18 and len(f2) == 32
    RM.assert_invariants(v2, f2, 2)
    v3, f3, n = RM.split(v, f, 10.0)
    assert n == 0 and np.array_equal(f3, f)


def canonical(faces):
    """Each triangle rotated to start at its smallest index: equal sets of oriented triangles compare equal."""
    return sorted(tuple(np.roll(t, -int(np.argmin(t))).tolist()) for t in np.asarray(faces))


def test_split_two_edges_uses_the_shorter_diagonal():
    # AB, BC and BD are longer than 2; each face but ADC has two of them.  ACB takes the diagonal m_BC-A (2.5 < 3.25),
    # ABD the diagonal A-m_BD (2.5 < 3.25), and BCD ties at 3.5 and takes D-m_BC, the diagonal from the vertex after the
    # edge that is not split.
    v = np.array([[0, 0, 0], [3, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    A, B, C, D = range(4)
    f = np.array([[A, C, B], [A, B, D], [A, D, C], [B, C, D]], np.int64)
    v2, f2, n = RM.split(v, f, 2.0)
    assert n == 3 and len(v2) == 7 and len(f2) == 10
    at = {tuple(p.tolist()): i for i, p in enumerate(v2)}
    AB, BC, BD = at[(1.5, 0.0, 0.0)], at[(1.5, 0.5, 0.0)], at[(1.5, 0.0, 0.5)]
    want = [(C, BC, A), (BC, AB, A), (BC, B, AB),
            (A, AB, BD), (A, BD, D), (AB, B, BD),
            (A, D, C),
            (D, BD, BC), (D, BC, C), (BD, B, BC)]
    assert canonical(f2) == canonical(want)
    RM.assert_invariants(v2, f2, 2)


def assert_normals_kept(v0, f0, v1, f1):
    """Every face slot that is live after a collapse or flip round has turned its unit normal by less than 60 degrees."""
    v0, v1 = np.asarray(v0, np.float64), np.asarray(v1, np.float64)
    live = np.flatnonzero(np.asarray(f1)[:, 0] >= 0)

    def unit(v, f):
        n = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        return n / np.linalg.norm(n, axis=1, keepdims=True)

    cos = (unit(v0, np.asarray(f0)[live]) * unit(v1, np.asarray(f1)[live])).sum(1)
    assert (cos >= 0.5 - 1e-9).all(), float(cos.min())


@pytest.mark.parametrize("case", ["ico3", "bunny"])
def test_collapse_and_flip_keep_normals_within_60_degrees(case, bunny_mesh):
    v, f = (np.asarray(bunny_mesh[0], np.float32), bunny_mesh[1]) if case == "bunny" else workloads.icosphere(3)
    v, f, mean = noisy(np.asarray(v, np.float32), np.asarray(f, np.int64), 0.15, seed=3)
    rounds = 0
    for h in (2 * mean, 3 * mean):
        v1, f1, _ = RM.split(v, f, 1.4 * h)
        while True:
            v2, f2, n = RM.collapse_round(v1, f1, 0.7 * h, 1.4 * h, len(v1))
            assert_normals_kept(v1, f1, v2, f2)
            v1, f1, rounds = v2, f2, rounds + n
            if n == 0:
                break
        v1, f1 = RM.compact(v1, f1)
        while True:
            f2, n = RM.flip_round(v1, f1)
            assert_normals_kept(v1, f1, v1, f2)
            f1, rounds = f2, rounds + n
            if n == 0:
                break
    assert rounds > 0


def regular_tetrahedron(s, offset):
    v = np.array([[s, s, s], [s, -s, -s], [-s, s, -s], [-s, -s, s]], np.float32) + np.float32(offset)
    f = np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]], np.int64)
    return v, f


def with_small_components(v, f):
    """v, f plus a regular tetrahedron of edge 0.2 h 2 sqrt 2 and an octahedron of edge 0.3 h sqrt 2 (h the mean edge),
    away from it: both closed components have every edge below 0.7 h."""
    h = mean_edge(v, f)
    tv, tf = regular_tetrahedron(0.2 * h, [3.0, 0.0, 0.0])
    ov, of = octahedron()
    ov = (ov * np.float32(0.3 * h) + np.float32([0.0, 3.0, 0.0])).astype(np.float32)
    verts = np.concatenate([np.asarray(v, np.float32), tv, ov])
    faces = np.concatenate([f, tf + len(v), of + len(v) + 4])
    return verts, faces, h


def test_small_closed_components_stop_at_a_tetrahedron():
    v, f = workloads.icosphere(2)
    v, f, h = with_small_components(np.asarray(v, np.float32), np.asarray(f, np.int64))
    assert RM.check(f, len(v)) == 0 and RM.euler(v, f) == 6
    for project in (True, False):
        vo, fo = RM.remesh(v, f, 5, h, project)
        RM.assert_invariants(vo, fo, 6)
        assert np.bincount(fo.ravel()).min() >= 3
        assert len(vo) >= 162 + 4 + 4


@pytest.mark.parametrize("scale", [1.6, 0.4])
def test_icosahedron_with_one_vertex_moved(scale):
    v, f = ico(scale)
    h = mean_edge(v, f)
    for project in (True, False):
        vo, fo = RM.remesh(v, f, 5, h, project)
        RM.assert_invariants(vo, fo, 2)


def test_collapse_keeps_four_vertices():
    v, f = ico()
    vo, fo = RM.remesh(v, f, 3, 100.0)
    RM.assert_invariants(vo, fo, 2)
    assert len(vo) >= 4


@pytest.mark.parametrize("case", ["ico3", "ico4", "bunny"])
def test_noisy_meshes(case, bunny_mesh):
    if case == "bunny":
        v, f = bunny_mesh
        v = np.asarray(v, np.float32)
    else:
        v, f = workloads.icosphere(int(case[-1]))
    v, f, mean = noisy(np.asarray(v, np.float32), np.asarray(f, np.int64), 0.1)
    chi = RM.euler(v, f)
    for h in (0.5 * mean, 2 * mean):
        vo, fo = RM.remesh(v, f, 2, h, True)
        RM.assert_invariants(vo, fo, chi)
        e = np.linalg.norm(vo[fo[:, 1]] - vo[fo[:, 0]], axis=1)
        assert np.median(e) < 1.4 * h * 1.5
