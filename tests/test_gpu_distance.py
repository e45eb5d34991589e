"""GPU: point-to-mesh squared distances and the Hausdorff distance (largesteps_b200.distance, csrc/ls_distance.cu) against the
float64 model of tests/distance_model.py.  Per query, sqrD is within 1e-12 (|q| + max|corner|)^2 of the model, C lies on
face I at squared distance sqrD, and the model's distance to face I is sqrD; results are bitwise reproducible across builds,
streams and index types; the error paths and pathological trees (coincident faces, a 2e6-face needle strip) behave."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
import distance_model as model
from largesteps_b200 import workloads
from largesteps_b200.distance import MeshDistance, hausdorff, point_mesh_squared_distance

pytestmark = pytest.mark.gpu
DEV = "cuda"


def t(x, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV) if dtype is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dtype)


def noisy(v, sigma, seed):
    return (v + np.random.default_rng(seed).normal(0, sigma, size=v.shape)).astype(np.float32)


def degenerate_mesh():
    g = np.load(os.path.join(GOLDEN, "mass.npz"))
    f = g["degen.faces"].astype(np.int64)
    return g["degen.verts"].astype(np.float32), np.concatenate([f, f[:1]])     # plus a duplicated face


def mesh(name):
    if name == "ico4":
        return workloads.icosphere(4)
    if name == "bunny":
        d = np.load(os.path.join(GOLDEN, "bunny_mesh.npz"))
        return d["verts"].astype(np.float32), d["faces"].astype(np.int64)
    if name == "plane200":
        v, f = workloads.plane(200)
        return noisy(v, 1e-3, 5), f
    return degenerate_mesh()


def queries(v, f, seed=0, m=400):
    """The mesh's own vertices, barycentric face samples, points offset along face normals by +-[1e-4, 1] x diagonal, far
    points at 100 x diagonal and random points in the bounding box."""
    rng = np.random.default_rng(seed)
    v64 = v.astype(np.float64)
    lo, hi = v64.min(0), v64.max(0)
    diag = float(np.linalg.norm(hi - lo))
    fi = rng.integers(0, len(f), m)
    b = rng.dirichlet(np.ones(3), m)
    on = (b[:, :, None] * v64[f[fi]]).sum(1)
    n = np.cross(v64[f[fi, 1]] - v64[f[fi, 0]], v64[f[fi, 2]] - v64[f[fi, 0]])
    nn = np.linalg.norm(n, axis=1, keepdims=True)
    n = np.where(nn > 0, n / np.where(nn > 0, nn, 1), 0)
    off = on + n * diag * rng.choice([-1, 1], (m, 1)) * 10.0 ** rng.uniform(-4, 0, (m, 1))
    d = rng.normal(size=(m // 4, 3))
    far = (lo + hi) / 2 + 100 * diag * d / np.linalg.norm(d, axis=1, keepdims=True)
    box = lo + (hi - lo) * rng.uniform(size=(m, 3))
    return np.concatenate([v64, on, off, far, box]).astype(np.float32)


def tol(P, v):
    return 1e-12 * (np.linalg.norm(P.astype(np.float64), axis=1) + np.linalg.norm(v.astype(np.float64), axis=1).max()) ** 2


def run(P, v, f, idx=torch.int64):
    md = MeshDistance(t(v), t(f, idx))
    s, i, c = md.squared_distance(t(P))
    md.check()
    return s.cpu().numpy(), i.cpu().numpy(), c.cpu().numpy()


def check_against_model(P, v, f, s, i, c):
    ms, mi, _ = model.point_mesh(P, v, f)
    tl = tol(P, v)
    assert (np.abs(s - ms) <= tl).all(), float((np.abs(s - ms) / tl).max())
    assert (i >= 0).all() and (i < len(f)).all()
    q = P.astype(np.float64)
    np.testing.assert_allclose(((q - c) ** 2).sum(1), s, rtol=1e-13, atol=1e-300)
    v64 = v.astype(np.float64)
    a, b, cc = v64[f[i, 0]], v64[f[i, 1]], v64[f[i, 2]]
    fs, _ = model.closest_on_triangle(q, a, b, cc)
    assert (np.abs(fs - s) <= tl).all()
    # C lies on face I: barycentric coordinates >= -1e-9 summing to 1 (non-degenerate faces), else on one of its segments
    e0, e1, r = b - a, cc - a, c - a
    d00, d01, d11 = (e0 * e0).sum(1), (e0 * e1).sum(1), (e1 * e1).sum(1)
    den = d00 * d11 - d01 ** 2
    ok = den > 1e-6 * d00 * d11
    d20, d21 = (r * e0).sum(1), (r * e1).sum(1)
    bv = np.where(ok, (d11 * d20 - d01 * d21) / np.where(ok, den, 1), 0)
    bw = np.where(ok, (d00 * d21 - d01 * d20) / np.where(ok, den, 1), 0)
    bu = 1 - bv - bw
    assert (np.minimum(np.minimum(bu, bv), bw)[ok] >= -1e-9).all()
    plane_off = model.closest_on_triangle(c, a, b, cc)[0]
    assert (plane_off <= 1e-12 * (np.linalg.norm(c, axis=1) + 1) ** 2).all()


@pytest.mark.parametrize("name", ["ico4", "bunny", "plane200", "degen"])
def test_matches_the_model(name):
    v, f = mesh(name)
    P = queries(v, f)
    s, i, c = run(P, v, f)
    used = np.unique(f)
    np.testing.assert_array_equal(s[used], 0.0)                     # the mesh's own (referenced) vertices
    check_against_model(P, v, f, s, i, c)


def test_bitwise_reproducible_across_index_types_builds_and_streams():
    v, f = mesh("bunny")
    P = queries(v, f, seed=3)
    ref = run(P, v, f, torch.int64)
    for out in (run(P, v, f, torch.int32), run(P, v, f, torch.int64)):
        for x, y in zip(ref, out):
            np.testing.assert_array_equal(x.view(np.uint8), y.view(np.uint8))
    md = MeshDistance(t(v), t(f))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        Pd = t(P)
        out = md.squared_distance(Pd)
    s.synchronize()
    for x, y in zip(ref, out):
        np.testing.assert_array_equal(x.view(np.uint8), y.cpu().numpy().view(np.uint8))


def test_error_paths_and_nan():
    v, f = mesh("ico4")
    vt, ft = t(v), t(f)
    with pytest.raises(ValueError):
        MeshDistance(vt, ft[:0])
    for bad in (-1, len(v)):
        fb = ft.clone()
        fb[5, 1] = bad
        with pytest.raises(IndexError):
            MeshDistance(vt, fb)
    with pytest.raises(RuntimeError):
        MeshDistance(vt.cpu(), ft.cpu())
    with pytest.raises(TypeError):
        MeshDistance(vt.double(), ft)
    s, i, c = point_mesh_squared_distance(t(np.zeros((0, 3), np.float32)), vt, ft)
    assert s.shape == (0,) and i.shape == (0,) and c.shape == (0, 3)
    P = np.array([[np.nan, 0, 0], [0, 0, 0], [0.1, np.nan, 2.0]], np.float32)
    s, i, c = (x.cpu().numpy() for x in point_mesh_squared_distance(t(P), vt, ft))
    assert np.isnan(s[[0, 2]]).all() and (i[[0, 2]] == -1).all() and np.isnan(c[[0, 2]]).all()
    assert np.isfinite(s[1]) and i[1] >= 0
    vn = v.copy()
    vn[3, 2] = np.nan
    s, i, _ = point_mesh_squared_distance(t(P[1:2]), t(vn), ft)
    assert np.isnan(s.item()) and i.item() == -1
    assert math.isnan(hausdorff(t(vn), ft, vt, ft)) and math.isnan(hausdorff(vt, ft, t(vn), ft))


def test_pathological_trees():
    rng = np.random.default_rng(9)
    # 10^5 copies of one triangle: every query ties on all of them, so face 0 wins
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32)
    f = np.zeros((100_000, 3), np.int64) + np.array([0, 1, 2])
    P = rng.normal(size=(256, 3)).astype(np.float32)
    s, i, c = run(P, v, f)
    ms, _, _ = model.brute_force(P, v, f[:1])
    assert (i == 0).all() and (np.abs(s - ms) <= tol(P, v)).all()
    # every vertex at one point
    v = np.ones((1000, 3), np.float32)
    f = rng.integers(0, 1000, size=(5000, 3))
    s, i, c = run(P, v, f)
    np.testing.assert_allclose(s, ((P.astype(np.float64) - 1) ** 2).sum(1), rtol=1e-15)
    assert (i == 0).all()
    # a strip of 2e6 needles: 1e6 + 1 vertex pairs along x, 1e-3 apart, 1e-6 wide
    n = 1_000_001
    x = np.arange(n) * 1e-3
    v = np.concatenate([np.stack([x, 0 * x, 0 * x], 1), np.stack([x, 0 * x + 1e-6, 0 * x], 1)]).astype(np.float32)
    a = np.arange(n - 1)
    f = np.concatenate([np.stack([a, a + 1, a + n], 1), np.stack([a + 1, a + n + 1, a + n], 1)])
    assert len(f) == 2_000_000
    P = np.concatenate([rng.uniform([-1, -0.1, -0.1], [1001, 0.1, 0.1], size=(3000, 3)),
                        rng.normal(size=(96, 3)) * 1e3]).astype(np.float32)
    s, i, c = run(P, v, f)
    check_against_model(P, v, f, s, i, c)


@pytest.mark.parametrize("pair", ["ico", "bunny", "plane"])
def test_hausdorff_matches_the_model(pair):
    if pair == "ico":
        (va, fa), (vb, fb) = workloads.icosphere(3), workloads.icosphere(5)
        vb = (vb * np.float32(1.01)).astype(np.float32)
    elif pair == "bunny":
        va, fa = mesh("bunny")
        vb, fb = noisy(va, 1e-3, 2), fa
    else:
        (va, fa), (vb, fb) = workloads.plane(200), workloads.plane(200, seed=1)
    h = hausdorff(t(va), t(fa), t(vb), t(fb))
    want = model.hausdorff(va, fa, vb, fb)
    tl = max(tol(va, vb).max(), tol(vb, va).max())
    assert abs(h * h - want * want) <= tl, (h, want)
    assert hausdorff(t(vb), t(fb), t(va), t(fa)) == h                 # symmetric


def flat_grid(n=1000):
    v, f = workloads.plane(n)
    v[:, 2] = 0.0
    return v, f


def test_hausdorff_on_a_million_vertex_grid():
    v, f = flat_grid()
    vt, ft = t(v), t(f)
    assert hausdorff(vt, ft, vt, ft) == 0.0
    delta = np.float32(3e-3)
    vd = v.copy()
    vd[:, 2] += delta
    h = hausdorff(t(vd), ft, vt, ft)
    assert abs(h - float(delta)) <= np.spacing(float(delta)), (h, float(delta))


@pytest.mark.parametrize("direction", ["AB", "BA"])
def test_plane1000_each_way(direction):
    A, B = workloads.plane(1000), workloads.plane(1000, seed=1)
    if direction == "BA":
        A, B = B, A
    (va, fa), (vb, fb) = A, B
    mb = MeshDistance(t(vb), t(fb))
    s, i, c = mb.squared_distance(t(va))
    mb.check()
    s, i, c = s.cpu().numpy(), i.cpu().numpy(), c.cpu().numpy()
    sel = np.random.default_rng(4).choice(len(va), 65_536, replace=False)
    check_against_model(va[sel], vb, fb, s[sel], i[sel], c[sel])
    ma = MeshDistance(t(va), t(fa))
    s2 = ma.squared_distance(t(vb))[0].cpu().numpy()
    h = mb.hausdorff(t(va), t(fa))
    assert h == math.sqrt(max(s.max(), s2.max()))


def test_shuffled_face_order():
    """Faces in a random order (as a remesher may number them) give bitwise the same distances; the face found may differ
    only where faces tie, and then it is at the same distance."""
    v, f = mesh("plane200")
    P = queries(v, f, seed=6)
    perm = np.random.default_rng(8).permutation(len(f))
    s0, i0, c0 = run(P, v, f)
    s1, i1, c1 = run(P, v, f[perm])
    check_against_model(P, v, f[perm], s1, i1, c1)
    np.testing.assert_array_equal(s1, s0)
    # where the faces differ, they tie (a closest point on a shared edge or vertex): both are at the same distance
    v64, q = v.astype(np.float64), P.astype(np.float64)
    other = f[perm[i1]]
    d_other = model.closest_on_triangle(q, v64[other[:, 0]], v64[other[:, 1]], v64[other[:, 2]])[0]
    assert (np.abs(d_other - s0) <= tol(P, v)).all()


def test_mesh_distance_keeps_its_own_vertices():
    """Changing B's vertices in place after MeshDistance(VB, FB) changes neither its BVH nor its query points."""
    (va, fa), (vb, fb) = workloads.icosphere(3), workloads.icosphere(4)
    VB = t(vb)
    mb = MeshDistance(VB, t(fb))
    want = mb.hausdorff(t(va), t(fa))
    VB.mul_(2.0)
    assert mb.hausdorff(t(va), t(fa)) == want == hausdorff(t(va), t(fa), t(vb), t(fb))
