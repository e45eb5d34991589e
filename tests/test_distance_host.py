"""CPU: the point-triangle and box-bound bodies of the distance query (csrc/ls_distance.cu, __host__ __device__) compiled for the
host by nvcc.  The closest point is checked against the float64 model of tests/distance_model.py on 10^5 seeded pairs,
degenerate triangles included; the box bound is checked never to exceed the exact squared distance, in rational arithmetic."""
import ctypes
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from conftest import ROOT
import largesteps_b200._native as N
import distance_model as model

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HARNESS = r"""
#include "ls_distance.cu"
extern "C" void host_closest(const float *p, const float *tri, int64_t m, double *sqrD, double *C) {
    for (int64_t i = 0; i < m; ++i) {
        const double q[3] = {p[3 * i], p[3 * i + 1], p[3 * i + 2]};
        double a[3], b[3], c[3];
        for (int d = 0; d < 3; ++d) {
            a[d] = tri[9 * i + d];
            b[d] = tri[9 * i + 3 + d];
            c[d] = tri[9 * i + 6 + d];
        }
        sqrD[i] = ls_closest_on_triangle(q, a, b, c, C + 3 * i);
    }
}
extern "C" void host_box(const float *p, const float *lo, const float *hi, int64_t m, double *lb) {
    for (int64_t i = 0; i < m; ++i) {
        const double q[3] = {p[3 * i], p[3 * i + 1], p[3 * i + 2]};
        lb[i] = ls_box_lower_bound(q, lo + 3 * i, hi + 3 * i);
    }
}
"""


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    d = tmp_path_factory.mktemp("distance_host")
    src, lib = d / "harness.cu", d / "libdistance_host.so"
    src.write_text(HARNESS)
    libdir = os.path.dirname(N.LIB_PATH)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I", os.path.join(ROOT, "large-steps-pytorch_b200", "csrc"), str(src), "-o", str(lib),
                        "-L", libdir, "-l:libls_b200.so", "-Xlinker", "-rpath=" + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    h = ctypes.CDLL(str(lib))
    h.host_closest.restype = None
    h.host_box.restype = None
    return h


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def host_closest(host_lib, p, tri):
    p = np.ascontiguousarray(p, np.float32)
    tri = np.ascontiguousarray(tri, np.float32).reshape(len(p), 9)
    s, c = np.zeros(len(p)), np.zeros((len(p), 3))
    host_lib.host_closest(_p(p), _p(tri), ctypes.c_int64(len(p)), _p(s), _p(c))
    return s, c


def seeded_pairs(m=100_000, seed=0):
    """Random triangles and points at several scales; four in ten triangles have a zero-length edge, (nearly) collinear
    corners, all corners equal or one short edge."""
    rng = np.random.default_rng(seed)
    tri = rng.normal(size=(m, 3, 3))
    q = rng.normal(size=(m, 3)) * rng.choice([0.1, 1.0, 10.0], size=(m, 1))
    kind = rng.integers(0, 10, size=m)
    tri[kind == 0, 1] = tri[kind == 0, 0]                                            # zero-length edge
    t = rng.uniform(-1, 2, size=(m, 1))
    tri[kind == 1, 2] = (tri[:, 0] + t * (tri[:, 1] - tri[:, 0]))[kind == 1]          # (nearly) collinear
    tri[kind == 2] = tri[kind == 2, :1]                                               # all corners equal
    tri[kind == 3, 2] = tri[kind == 3, 1] + 1e-3 * rng.normal(size=(m, 3))[kind == 3]  # a short edge
    scale = rng.choice([1e-3, 1.0, 1e3], size=(m, 1, 1))
    tri, q = (tri * scale).astype(np.float32), (q * scale[:, 0] + tri[:, 0] * scale[:, 0]).astype(np.float32)
    return q, tri


def test_closest_point_matches_the_model(host_lib):
    q, tri = seeded_pairs()
    s, c = host_closest(host_lib, q, tri)
    t = tri.astype(np.float64)
    ms, mc = model.closest_on_triangle(q, t[:, 0], t[:, 1], t[:, 2])
    scale = (np.linalg.norm(q.astype(np.float64), axis=1) + np.linalg.norm(t, axis=2).max(axis=1)) ** 2
    err = np.abs(s - ms) / scale
    assert err.max() <= 1e-12, (err.max(), int(err.argmax()))
    # the returned point is the one whose distance is returned
    d = c - q.astype(np.float64)
    np.testing.assert_allclose((d * d).sum(1), s, rtol=1e-15, atol=0)


def test_degenerate_triangles_are_their_segments(host_lib):
    tri = np.array([[[0, 0, 0], [1, 0, 0], [2, 0, 0]],          # collinear
                    [[0, 0, 0], [0, 0, 0], [2, 0, 0]],          # zero-length edge
                    [[1, 1, 1], [1, 1, 1], [1, 1, 1]],          # one point
                    [[2, 0, 0], [0, 0, 0], [1, 0, 0]]], np.float32)
    q = np.array([[1.5, 1, 0], [3, 0, 0], [1, 1, 3], [-1, 0, 1]], np.float32)
    s, c = host_closest(host_lib, q, tri)
    np.testing.assert_array_equal(s, [1.0, 1.0, 4.0, 2.0])
    np.testing.assert_array_equal(c, [[1.5, 0, 0], [2, 0, 0], [1, 1, 1], [0, 0, 0]])


def _exact_box(p, lo, hi):
    s = Fraction(0)
    for d in range(3):
        x, l, h = Fraction(float(p[d])), Fraction(float(lo[d])), Fraction(float(hi[d]))
        g = l - x if x < l else (x - h if x > h else Fraction(0))
        s += g * g
    return s


def test_box_lower_bound_never_exceeds_the_exact_distance(host_lib):
    rng = np.random.default_rng(3)
    m = 20_000
    # coordinates over many binades, so that the fp64 gaps are inexact; hi >= lo per axis
    e = rng.integers(-60, 60, size=(m, 3, 3))
    x = (rng.uniform(-1, 1, size=(m, 3, 3)) * 2.0 ** e).astype(np.float32)
    lo, hi = np.minimum(x[:, 0], x[:, 1]), np.maximum(x[:, 0], x[:, 1])
    p = x[:, 2].copy()
    p[: m // 4] = (lo[: m // 4] * (1 - 2.0 ** -23)).astype(np.float32)        # just outside a face of the box
    p, lo, hi = (np.ascontiguousarray(a) for a in (p, lo, hi))
    lb = np.zeros(m)
    host_lib.host_box(_p(p), _p(lo), _p(hi), ctypes.c_int64(m), _p(lb))
    assert (lb >= 0).all()
    tight = 0
    for i in range(m):
        ex = _exact_box(p[i], lo[i], hi[i])
        assert Fraction(float(lb[i])) <= ex, i
        tight += ex == 0 or float(lb[i]) >= float(ex) * (1 - 2.0 ** -45)
    assert tight == m                                                           # and it is a tight bound



def _exact_closest(p, a, b, c):
    """Ericson's regions in rational arithmetic: the exact squared distance from p to the triangle (a, b, c)."""
    F = [Fraction(float(x)) for x in (*p, *a, *b, *c)]
    p, a, b, c = F[0:3], F[3:6], F[6:9], F[9:12]
    sub = lambda u, v: [u[k] - v[k] for k in range(3)]
    dot = lambda u, v: sum(u[k] * v[k] for k in range(3))
    ab, ac, ap, bp, cp = sub(b, a), sub(c, a), sub(p, a), sub(p, b), sub(p, c)
    d1, d2, d3, d4, d5, d6 = dot(ab, ap), dot(ac, ap), dot(ab, bp), dot(ac, bp), dot(ab, cp), dot(ac, cp)
    vc, vb, va = d1 * d4 - d3 * d2, d5 * d2 - d1 * d6, d3 * d6 - d5 * d4
    if d1 <= 0 and d2 <= 0:
        w = a
    elif d3 >= 0 and d4 <= d3:
        w = b
    elif d6 >= 0 and d5 <= d6:
        w = c
    elif vc <= 0 and d1 >= 0 and d3 <= 0:
        t = d1 / (d1 - d3)
        w = [a[k] + t * ab[k] for k in range(3)]
    elif vb <= 0 and d2 >= 0 and d6 <= 0:
        t = d2 / (d2 - d6)
        w = [a[k] + t * ac[k] for k in range(3)]
    elif va <= 0 and d4 - d3 >= 0 and d5 - d6 >= 0:
        t = (d4 - d3) / ((d4 - d3) + (d5 - d6))
        w = [b[k] + t * (c[k] - b[k]) for k in range(3)]
    else:
        den = va + vb + vc
        w = [a[k] + ab[k] * vb / den + ac[k] * vc / den for k in range(3)]
    e = sub(p, w)
    return dot(e, e)


def sliver_pairs(m=3000, seed=5):
    """Triangles whose squared sine at corner a, after rounding to float32, lies in [2^-36, 2^-30]: just above the threshold
    below which a triangle is treated as its segments, where Ericson's barycentrics are least accurate."""
    rng = np.random.default_rng(seed)
    out_q, out_t = [], []
    while sum(len(q) for q in out_q) < m:
        a = rng.normal(size=(m, 3))
        u, v = rng.normal(size=(m, 3)), rng.normal(size=(m, 3))
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        v -= (v * u).sum(1, keepdims=True) * u
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        th = 2.0 ** rng.uniform(-18, -15, size=(m, 1)) * rng.choice([1, -1], size=(m, 1)) + rng.choice([0, np.pi], size=(m, 1))
        L = rng.uniform(0.2, 2.0, size=(m, 2))
        tri = np.stack([a, a + L[:, :1] * u, a + L[:, 1:] * (np.cos(th) * u + np.sin(th) * v)], 1).astype(np.float32)
        t = tri.astype(np.float64)
        ab, ac = t[:, 1] - t[:, 0], t[:, 2] - t[:, 0]
        s2 = (np.cross(ab, ac) ** 2).sum(1) / ((ab * ab).sum(1) * (ac * ac).sum(1))
        keep = (s2 > 2.0 ** -36) & (s2 <= 2.0 ** -30)
        bary = rng.dirichlet(np.ones(3), m)
        n = rng.normal(size=(m, 3)) * rng.choice([1e-4, 1e-2, 1.0, 10.0, 100.0], size=(m, 1))
        q = ((bary[:, :, None] * t).sum(1) + n).astype(np.float32)
        out_q.append(q[keep])
        out_t.append(tri[keep])
    return np.concatenate(out_q)[:m], np.concatenate(out_t)[:m]


def test_sliver_band_error_bound(host_lib):
    """Just above the degenerate threshold the leaf test may overestimate the exact squared distance by up to
    2e-12 (max|q| + max|corner|)^2 (DESIGN 4.5); it never falls below it by more than the prune slack 2^-40 (...)^2, which is
    what keeps the tie rule."""
    q, tri = sliver_pairs()
    s, _ = host_closest(host_lib, q, tri)
    scale = (np.abs(q.astype(np.float64)).max(1) + np.abs(tri.astype(np.float64)).max((1, 2))) ** 2
    err = np.array([float(Fraction(float(s[i])) - _exact_closest(q[i], tri[i, 0], tri[i, 1], tri[i, 2])) for i in range(len(q))])
    err /= scale
    print(f"sliver band: error / (max|q| + max|corner|)^2 in [{err.min():.3e}, {err.max():.3e}]")
    assert err.max() <= 2e-12, err.max()
    assert err.min() >= -2.0 ** -40, err.min()
