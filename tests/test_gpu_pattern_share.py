"""GPU: the pattern-only copy stores each distinct compact slice once (csrc/ls_pcg.cu pat_hash_kernel ..
pat_share_copy_kernel).  The built copy decodes to the matrix's columns row by row, and the solves are bitwise the ones of
the unshared layout (LS_PCG_PATSHARE=0)."""
import numpy as np
import pytest
import torch

from largesteps_b200 import workloads
from largesteps_b200.batch import BatchSolver
from largesteps_b200.geometry import compute_matrix, morton_order
from largesteps_b200.solvers import PCGSolver
from gpu_util import DEV, to_dev
from test_pattern_share_host import decode_rows, expected_rows, pat_slice

pytestmark = pytest.mark.gpu


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def far_block(n):
    v, f = workloads.plane(n, seed=0)
    V = v.shape[0]
    perm = np.arange(V)
    perm[:1000], perm[V - 1000:] = np.arange(V - 1000, V), np.arange(1000)
    return v, perm[f]


def morton_mesh(n):
    v, f = workloads.plane(n, seed=1)
    p = morton_order(torch.from_numpy(v.astype(np.float32)).to(DEV)).long().cpu().numpy()   # new -> old
    inv = np.empty_like(p)
    inv[p] = np.arange(len(p))
    return v[p], inv[f]


def with_fans(n=200):
    """a plane with three vertices of valence 40+: slices of 15+ pairs (never shared; the next slice keeps its own copy)"""
    v, f = workloads.plane(n, seed=0)
    V = v.shape[0]
    hubs = (15000, 19000, 19031)
    extra = np.array([[h, (h + 7 * k + 1) % V, (h + 7 * k + 4) % V] for h in hubs for k in range(20)])
    return v, np.concatenate([f, extra])


def with_isolated(v, f, n=70):
    extra = np.random.default_rng(0).normal(size=(n, 3)).astype(v.dtype) + 5.0
    return np.concatenate([v, extra]), f


def meshes(bunny_mesh):
    return {
        "plane1000": (*workloads.plane(1000, seed=0), dict(lambda_=1.0, alpha=0.95)),
        "bunny2": (*workloads.subdivide(*workloads.subdivide(*bunny_mesh)), dict(lambda_=19.0)),
        "icosphere5": (*workloads.icosphere(5), dict(lambda_=10.0)),
        "morton300": (*morton_mesh(300), dict(lambda_=1.0, alpha=0.95)),
        "farblock200": (*far_block(200), dict(lambda_=1.0, alpha=0.95)),
        "isolated": (*with_isolated(*workloads.icosphere(4)), dict(lambda_=10.0)),
        "fans200": (*with_fans(200), dict(lambda_=1.0, alpha=0.95)),
    }


@pytest.mark.parametrize("name", ["plane1000", "bunny2", "icosphere5", "morton300", "farblock200", "isolated", "fans200"])
def test_built_copy_decodes_to_the_matrix(name, bunny_mesh):
    v, f, kw = meshes(bunny_mesh)[name]
    M = compute_matrix(*to_dev(v, f), **kw)
    s = PCGSolver(M, reorder=False)
    d = s.pattern_copy(arrays=True)
    assert d["on"] == 1
    ns, poff, pc = d["slices"], d["poff"].astype(np.int64), d["words_array"]
    V = v.shape[0]
    idx = M.coalesce().indices().cpu().numpy()
    off = idx[0] != idx[1]
    rows, cols = idx[0][off], idx[1][off]
    rp = np.zeros(V + 1, np.int64)
    rp[1:] = np.cumsum(np.bincount(rows, minlength=V))
    got = decode_rows(poff, pc, ns)
    assert (got == expected_rows(rp, cols, V, got.shape[1] // 2)).all(), name
    wide = np.array([pat_slice(poff, i)[2] for i in range(ns)])
    if name == "farblock200":
        assert wide.any() and (~wide).any()
    if name == "fans200":
        w2 = np.array([pat_slice(poff, i)[1] for i in range(ns)])
        esc = np.flatnonzero(w2 >= 15)
        assert len(esc) >= 2 and (np.diff(esc) == 1).any()       # two escape slices in a row among them
        assert d["stored"] < ns
        for i in esc:                                            # an escape slice ends where the next one starts
            o0, n, wd = pat_slice(poff, i)
            assert (int(poff[i + 1]) & ~31) == o0 + n * (64 if wd else 32)
    if name == "plane1000":
        assert d["stored"] == 12 and 4 * d["words"] < 8192
    assert d["stored"] <= ns and s.describe()["pattern_slices_stored"] == d["stored"]


def solve_both(monkeypatch, make, run, env=None):
    out = []
    for share in ("1", "0"):
        monkeypatch.setenv("LS_PCG_PATSHARE", share)
        for k_, v_ in (env or {}).items():
            monkeypatch.setenv(k_, v_)
        out.append(run(make()))
    return out


@pytest.mark.parametrize("env", [{}, {"LS_PCG_CLUSTER": "0", "LS_PCG_RES": "1"}, {"LS_PCG_CLUSTER": "0", "LS_PCG_RES": "0"},
                                 {"LS_PCG_CLUSTER": "4"}], ids=lambda e: ",".join(f"{k[3:]}={v}" for k, v in e.items()) or "default")
def test_solutions_are_bitwise_those_of_the_unshared_copy(env, bunny_mesh, monkeypatch):
    rng = np.random.default_rng(5)
    cases = [(*workloads.plane(1000, seed=0), dict(lambda_=1.0, alpha=0.95)), (*workloads.icosphere(3), dict(lambda_=10.0)),
             (*workloads.subdivide(*bunny_mesh), dict(lambda_=19.0)), (*far_block(200), dict(lambda_=1.0, alpha=0.95))]
    for v, f, kw in cases:
        M = compute_matrix(*to_dev(v, f), **kw)
        V = v.shape[0]
        bs = [rng.normal(size=(V, k)).astype(np.float32) for k in (1, 2, 3)]
        b2 = (bs[2] + 1e-3 * rng.normal(size=bs[2].shape)).astype(np.float32)

        def run(s):
            xs = [s.solve(t(b)).cpu().numpy() for b in bs]
            its = [s.iterations]
            xs.append(s.solve(t(b2)).cpu().numpy())          # warm start from the previous (k = 3) solution
            its.append(s.iterations)
            return xs, its, s.describe()

        (xa, ia, da), (xb, ib, db) = solve_both(monkeypatch, lambda: PCGSolver(M, warm_start=True), run, env)
        assert ia == ib, (kw, da)
        for a, b in zip(xa, xb):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (kw, da)
        if da["sell_engine"] == 2:
            assert db["pattern_slices_stored"] == db["pattern_slices"] and da["pattern_slices_stored"] <= da["pattern_slices"]


def test_chebyshev_and_batch_bitwise(bunny_mesh, monkeypatch):
    rng = np.random.default_rng(9)
    v, f = workloads.plane(300, seed=2)
    M = compute_matrix(*to_dev(v, f), lambda_=1.0, alpha=0.95)
    b = rng.normal(size=(v.shape[0], 3)).astype(np.float32)

    def run(s):
        return s.solve(t(b)).cpu().numpy(), s.iterations, s.describe()["precond"]

    (xa, ia, pa), (xb, ib, pb) = solve_both(monkeypatch, lambda: PCGSolver(M, precond="chebyshev"), run, {"LS_PCG_CLUSTER": "0"})
    assert pa == pb == "chebyshev" and ia == ib and np.array_equal(xa.view(np.uint32), xb.view(np.uint32))

    batch = [(*workloads.icosphere(3), dict(lambda_=10.0)), (*workloads.plane(120, seed=1), dict(lambda_=1.0, alpha=0.9)),
             (*workloads.subdivide(*bunny_mesh), dict(lambda_=19.0))]
    Ms = [compute_matrix(*to_dev(v_, f_), **kw) for v_, f_, kw in batch]
    bs = [rng.normal(size=(v_.shape[0], 3)).astype(np.float32) for v_, _, _ in batch]
    for precond in ("jacobi", "chebyshev"):
        def runb(s):
            return [x.cpu().numpy() for x in s.solve([t(x) for x in bs])], s.iterations, s.plan()

        (xa, ia, pa), (xb, ib, pb) = solve_both(monkeypatch, lambda: BatchSolver(Ms, precond=precond), runb)
        assert ia == ib and pa == pb, precond                 # the batch plan does not depend on sharing
        for a, b_ in zip(xa, xb):
            assert np.array_equal(a.view(np.uint32), b_.view(np.uint32)), precond


@pytest.mark.parametrize("name", ["isolated", "fans200"])
def test_graph_mode_after_a_partially_shared_build(name, bunny_mesh, monkeypatch):
    """The sharing build borrows the solve's r and p areas as scratch; the graph-mode solver (also the fallback when a fused
    launch is refused) gathers their zero padding rows, so the build must leave them as it found them."""
    v, f, kw = meshes(bunny_mesh)[name]
    M = compute_matrix(*to_dev(v, f), **kw)
    rng = np.random.default_rng(3)
    bs = [rng.normal(size=(v.shape[0], k)).astype(np.float32) for k in (1, 2, 3)]

    def run(s):
        d = s.pattern_copy()
        xs = []
        for b in bs:
            xs.append(s.solve(t(b)).cpu().numpy())
            assert s.status == 1 and np.isfinite(xs[-1]).all(), (name, b.shape)
        return xs, s.describe()["algo"], d

    (xa, aa, da), (xb, ab, db) = solve_both(monkeypatch, lambda: PCGSolver(M, reorder=False), run, {"LS_PCG_MODE": "graph"})
    assert aa == ab == "graph"
    assert da["stored"] < da["slices"] and db["stored"] == db["slices"]     # shared in part, and not at all
    for a, b in zip(xa, xb):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name
