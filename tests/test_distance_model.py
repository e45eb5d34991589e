"""CPU: the float64 distance model of tests/distance_model.py against brute force and against closest points known in closed
form: the seven Voronoi regions of a triangle, points on a vertex, an edge and a face, degenerate and duplicated faces, and an
unreferenced vertex that sets the Hausdorff distance."""
import numpy as np
import pytest

import distance_model as model

TRI = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0]])


def random_mesh(seed, V=60, F=90):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(V, 3)).astype(np.float32)
    f = np.stack([rng.choice(V, 3, replace=False) for _ in range(F)]).astype(np.int64)
    return v, f


@pytest.mark.parametrize("seed", range(4))
def test_candidate_search_equals_brute_force(seed):
    v, f = random_mesh(seed)
    rng = np.random.default_rng(100 + seed)
    P = np.concatenate([rng.normal(size=(300, 3)), 30 * rng.normal(size=(20, 3)), v[:10]]).astype(np.float32)
    s0, i0, c0 = model.brute_force(P, v, f)
    s1, i1, c1 = model.point_mesh(P, v, f)
    np.testing.assert_array_equal(s1, s0)
    np.testing.assert_array_equal(i1, i0)
    np.testing.assert_array_equal(c1, c0)
    np.testing.assert_array_equal(s1[-10:], 0.0)


@pytest.mark.parametrize("q,want", [
    ((-1.0, -1.0, 0.5), (0.0, 0.0, 0.0)),     # corner a
    ((2.0, -0.5, 0.5), (1.0, 0.0, 0.0)),      # corner b
    ((-0.5, 2.0, -0.5), (0.0, 1.0, 0.0)),     # corner c
    ((0.5, -1.0, 0.5), (0.5, 0.0, 0.0)),      # edge ab
    ((-1.0, 0.25, 0.5), (0.0, 0.25, 0.0)),    # edge ac
    ((1.0, 1.0, 0.5), (0.5, 0.5, 0.0)),       # edge bc
    ((0.25, 0.25, -2.0), (0.25, 0.25, 0.0)),  # face
])
def test_each_voronoi_region(q, want):
    s, c = model.closest_on_triangle(np.array([q]), TRI[0], TRI[1], TRI[2])
    np.testing.assert_allclose(c[0], want, atol=1e-15)
    np.testing.assert_allclose(s[0], np.sum((np.array(q) - want) ** 2), rtol=1e-15)


@pytest.mark.parametrize("q", [(1.0, 0.0, 0.0), (0.5, 0.5, 0.0), (0.25, 0.125, 0.0)])
def test_points_on_the_triangle_are_at_zero(q):
    s, c = model.closest_on_triangle(np.array([q]), TRI[0], TRI[1], TRI[2])
    assert s[0] == 0.0
    np.testing.assert_array_equal(c[0], q)


def test_degenerate_and_duplicated_faces():
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [5, 5, 5], [0, 1, 0]], np.float32)
    f = np.array([[0, 1, 2],      # collinear
                  [3, 3, 3],      # one point
                  [0, 0, 2],      # zero-length edge
                  [0, 1, 4],
                  [0, 1, 4]])     # duplicate of face 3
    P = np.array([[1.5, 1.0, 0.0], [5, 5, 6], [0.2, 0.2, 1.0], [3, 0, 0]], np.float32)
    s, i, c = model.brute_force(P, v, f)
    np.testing.assert_array_equal(s, [1.0, 1.0, 1.0, 1.0])
    np.testing.assert_array_equal(i, [0, 1, 3, 0])        # ties go to the lowest index: 0 before 2, 3 before its duplicate 4
    np.testing.assert_array_equal(c[1], [5, 5, 5])
    s1, i1, c1 = model.point_mesh(P, v, f)
    np.testing.assert_array_equal(s1, s)
    np.testing.assert_array_equal(i1, i)


def test_nan_query():
    v, f = random_mesh(7)
    P = np.array([[np.nan, 0, 0], [0, 0, 0]], np.float32)
    s, i, _ = model.point_mesh(P, v, f)
    assert np.isnan(s[0]) and i[0] == -1 and np.isfinite(s[1])


def test_unreferenced_vertex_counts_in_hausdorff():
    v, f = random_mesh(1)
    h = model.hausdorff(v, f, v, f)
    assert h == 0.0
    far = np.concatenate([v, [[10.0, 0.0, 0.0]]]).astype(np.float32)
    h_far = model.hausdorff(far, f, v, f)
    d = model.brute_force(far[-1:], v, f)[0][0]
    assert h_far == np.sqrt(d) > 5.0
    assert model.hausdorff(v, f, far, f) == h_far         # symmetric
