"""CPU: the single-mesh solver's launch plan (ls_pcg_plan in csrc/ls_pcg_plan.cu, the pure host function ls_pcg_create plans with) at its edges, for an
H100's 132 SMs and 227 KB of shared memory per CTA.  The LS_PCG_* switches are set in the environment, as for PCGSolver."""
import ctypes

import pytest

import largesteps_b200._native as N
from largesteps_b200 import solvers

SMS = 132
SMEM = 227 * 1024   # H100: shared memory per CTA with the opt-in carve-out
SWITCHES = ("LS_PCG_MODE", "LS_PCG_CLUSTER", "LS_PCG_RES", "LS_PCG_ONECTA", "LS_PCG_CLRES", "LS_PCG_SMALLCTA")


@pytest.fixture(autouse=True)
def default_switches(monkeypatch):
    for name in SWITCHES:
        monkeypatch.delenv(name, raising=False)


def plan(nslices, pattern=True, **kw):
    return solvers.plan(nslices, pattern, kw.pop("sm_count", SMS), SMEM, **kw)


def fused(grid, cluster, residency, threads, precond="jacobi"):
    return {"algo": "fused", "grid": grid, "cluster": cluster, "residency": residency, "threads": threads, "precond": precond}


def test_one_cta_up_to_one_slice_per_warp(monkeypatch):
    for ns in (1, 24):
        for pattern in (True, False):
            assert plan(ns, pattern) == fused(1, 1, 3, 768)
        assert plan(ns, precond="chebyshev") == fused(1, 1, 2, 768, "chebyshev")
    monkeypatch.setenv("LS_PCG_RES", "2")
    assert plan(24) == fused(1, 1, 2, 768)


def test_small_meshes_take_the_grid_with_256_thread_ctas():
    assert plan(25) == fused(25, 0, 2, 256)
    assert plan(132 * 16) == fused(132, 0, 2, 256)
    assert plan(132 * 16 + 1) == fused(132, 0, 2, 768)


@pytest.mark.parametrize("pattern,k,res2,res1", [(True, 3, 142, 278), (False, 3, 135, 251), (False, 4, 104, 195), (True, 4, 104, 195)])
def test_residency_boundaries_in_slices_per_cta(pattern, k, res2, res1):
    """RES 2 while x, p, r, s and the diagonal of a CTA's slices fit in shared memory, RES 1 while r, s and the diagonal do,
    then RES 0.  K = 4 has no pattern-only instantiation: its plan ignores the flag."""
    for per_cta, res in ((res2, 2), (res2 + 1, 1), (res1, 1), (res1 + 1, 0)):
        assert plan(SMS * per_cta, pattern, k=k) == fused(SMS, 0, res, 768), (per_cta, res)


def test_shared_memory_fits_the_budget_at_each_boundary():
    out = (ctypes.c_int64 * 8)()
    for k, pat, per_cta in ((3, 1, 142), (3, 1, 278), (3, 0, 135), (3, 0, 251), (4, 0, 104), (4, 0, 195), (3, 1, 24)):
        N.check(N.lib().ls_pcg_plan(SMS * per_cta, k, pat, 1, SMS, SMEM, 1, out))
        assert int(out[7]) == per_cta and 0 < int(out[6]) <= SMEM


def test_headline_and_large_planes():
    assert plan(1000 * 1000 // 32) == fused(132, 0, 1, 768)          # V = 1e6: RES 1
    assert plan(2000 * 2000 // 32)["residency"] == 0                  # V = 4e6: every vector in global memory


def test_the_grid_is_capped_at_255_ctas():
    assert plan(1000, sm_count=300)["grid"] == 255
    assert plan(200, sm_count=300)["grid"] == 200


def test_cluster_resident_regime(monkeypatch):
    monkeypatch.setenv("LS_PCG_CLRES", "384")
    assert plan(24) == fused(1, 1, 3, 768)
    for ns, threads in ((25, 256), (128, 256), (129, 768), (384, 768)):
        for pattern in (True, False):
            assert plan(ns, pattern) == fused(16, 16, 4, threads), ns
        assert plan(ns, precond="chebyshev")["cluster"] == 0           # Chebyshev never runs there
    assert plan(385)["cluster"] == 0
    monkeypatch.setenv("LS_PCG_SMALLCTA", "0")
    assert plan(25) == fused(16, 16, 4, 768)


@pytest.mark.parametrize("n", [4, 8, 16])
def test_forced_cluster_falls_back_to_the_grid_when_the_mesh_does_not_fit(n, monkeypatch):
    monkeypatch.setenv("LS_PCG_CLUSTER", str(n))
    cap = 140                          # slices per CTA at RES 2 in the cluster layout (pattern copy)
    assert plan(10) == fused(n, n, 4, 256)
    assert plan(n * cap) == fused(n, n, 2, 768)
    assert plan(n * cap + 1)["cluster"] == 0
    monkeypatch.setenv("LS_PCG_RES", "2")
    assert plan(10) == fused(n, n, 2, 768)


def test_no_cluster_means_the_grid_even_for_tiny_meshes(monkeypatch):
    monkeypatch.setenv("LS_PCG_CLUSTER", "0")
    assert plan(10) == fused(10, 0, 2, 256)
    monkeypatch.setenv("LS_PCG_SMALLCTA", "0")
    assert plan(10) == fused(10, 0, 2, 768)


def test_graph_mode(monkeypatch):
    assert plan(100, cooperative=False) == {"algo": "graph"}
    assert plan(10, cooperative=False) == fused(1, 1, 3, 768)          # one CTA needs no cooperative launch
    monkeypatch.setenv("LS_PCG_MODE", "graph")
    assert plan(10) == {"algo": "graph"} and plan(100) == {"algo": "graph"}


def test_auto_preconditioner(monkeypatch):
    auto = lambda ns: plan(ns, precond="auto")["precond"]
    assert [auto(ns) for ns in (1, 24, 25, 11616, 11617, 31250)] == ["jacobi", "jacobi", "chebyshev", "chebyshev", "jacobi", "jacobi"]
    monkeypatch.setenv("LS_PCG_CLRES", "384")
    assert [auto(ns) for ns in (25, 384, 385)] == ["jacobi", "jacobi", "chebyshev"]
    monkeypatch.setenv("LS_PCG_CLUSTER", "0")
    assert auto(25) == "chebyshev"


def test_bad_arguments_are_rejected():
    out = (ctypes.c_int64 * 8)()
    lib = N.lib()
    for args in ((0, 3, 1, 1, SMS, SMEM, 1), (10, 2, 1, 1, SMS, SMEM, 1), (10, 3, 1, 4, SMS, SMEM, 1), (10, 3, 1, 1, 0, SMEM, 1),
                 (10, 3, 1, 1, SMS, 0, 1)):
        assert lib.ls_pcg_plan(*args, out) == N.LS_ERR_BAD_ARG
    assert lib.ls_pcg_plan(10, 3, 1, 1, SMS, SMEM, 1, None) == N.LS_ERR_BAD_ARG
    with pytest.raises(ValueError, match="Unknown preconditioner"):
        plan(10, precond="ic0")
