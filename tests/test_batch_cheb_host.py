"""CPU: the batch plan with the Chebyshev preconditioner (ls_pcg_batch_plan_ex, a pure host function).

With 227 KB of shared memory per CTA (H100), a Chebyshev mesh keeps 24 more bytes per row in shared memory (the iterate and the
direction, K = 3 floats each) and always runs at RES 2:
  pattern-only copy: 94 slices per CTA -> 1 CTA up to 94 slices, 2 up to 188, 4 up to 376, 8 up to 752, 16 up to 1504
                     (48,128 rows);
  general copy:      91 slices per CTA -> 16 CTAs up to 1456 slices (46,592 rows).
Jacobi meshes keep their plan: RES 3 on one CTA up to 105 slices (102 general), RES 2 up to 140 (133) per CTA.
"""
import random

import pytest

from largesteps_b200 import batch

SMEM = 227 * 1024   # H100: shared memory per CTA with the opt-in carve-out


def test_chebyshev_cluster_sizes_never_res3():
    edges = {1: 1, 24: 1, 94: 1, 95: 2, 188: 2, 189: 4, 376: 4, 377: 8, 752: 8, 753: 16, 1504: 16}
    for ns, cs in edges.items():
        (got,), ng = batch.plan([ns], [True], SMEM, cheb=[1])
        assert got[:2] == (cs, 2) and ng == 1, (ns, got)
    for ns, cs in {91: 1, 92: 2, 182: 2, 183: 4, 728: 8, 729: 16, 1456: 16}.items():
        (got,), _ = batch.plan([ns], [False], SMEM, cheb=[1])
        assert got[:2] == (cs, 2), (ns, got)
    # never RES 3, at any size or budget
    for ns in range(1, 1505, 7):
        for pat in (True, False):
            try:
                (got,), _ = batch.plan([ns], [pat], SMEM, cheb=[1])
            except ValueError:
                continue
            assert got[1] == 2, (ns, pat, got)


def test_chebyshev_row_limit_names_the_mesh():
    batch.plan([1504], [True], SMEM, cheb=[1])     # 48,128 rows
    batch.plan([1456], [False], SMEM, cheb=[1])    # 46,592 rows
    for ns, pat in ((1505, True), (1457, False)):
        with pytest.raises(ValueError) as e:
            batch.plan([4, ns], [True, pat], SMEM, cheb=[0, 1])
        msg = str(e.value)
        assert "mesh 1" in msg and "from_differential" in msg and "Chebyshev" in msg, msg
    # the same mesh as Jacobi fits (68,096 / 71,680 rows)
    batch.plan([4, 1505], [True, True], SMEM, cheb=[0, 0])


def test_chebyshev_and_jacobi_meshes_form_different_groups():
    for ns in (3, 50, 94, 200, 700, 1400):
        plan, ng = batch.plan([ns, ns], [True, True], SMEM, cheb=[1, 0])
        assert ng == 2 and plan[0][2] != plan[1][2], (ns, plan)
    # same size where Jacobi and Chebyshev take the same cluster size and RES: still two launches
    plan, ng = batch.plan([150, 150], [True, True], SMEM, cheb=[0, 1])
    assert plan[0][:2] == plan[1][:2] == (2, 2) and ng == 2
    plan, ng = batch.plan([3, 81, 104, 704, 1400, 3, 104, 81], [1, 1, 0, 1, 1, 0, 0, 1], SMEM, cheb=[1, 0, 1, 1, 0, 1, 1, 1])
    assert [p[2] for p in plan] == [0, 1, 2, 3, 4, 5, 2, 0] and ng == 6   # numbered in order of first appearance
    assert [p[:2] for p in plan] == [(1, 2), (1, 3), (2, 2), (8, 2), (16, 2), (1, 2), (2, 2), (1, 2)]
    plan, ng = batch.plan([3, 5, 7, 90], [1] * 4, SMEM, cheb=[1] * 4)
    assert ng == 1 and {p for p in plan} == {(1, 2, 0)}


def test_a_mesh_plan_does_not_depend_on_the_batch():
    rng = random.Random(0)
    for _ in range(200):
        n = rng.randint(1, 10)
        ns = [rng.choice([1, 3, 24, 91, 92, 94, 95, 105, 106, 140, 141, 376, 377, 753, 1456]) for _ in range(n)]
        pt = [rng.randint(0, 1) for _ in range(n)]
        ch = [rng.randint(0, 1) for _ in range(n)]
        plan, _ = batch.plan(ns, pt, SMEM, cheb=ch)
        for i in range(n):
            (alone,), _ = batch.plan([ns[i]], [pt[i]], SMEM, cheb=[ch[i]])
            assert alone[:2] == plan[i][:2], (ns[i], pt[i], ch[i])


def test_jacobi_plan_is_unchanged():
    """An all-zero cheb list gives the plan of cheb = NULL (all Jacobi)."""
    rng = random.Random(1)
    for budget in (SMEM, 100 * 1024, 64 * 1024):
        for _ in range(300):
            n = rng.randint(1, 12)
            ns = [rng.randint(1, 1000) for _ in range(n)]
            pt = [rng.randint(0, 1) for _ in range(n)]
            try:
                want = batch.plan(ns, pt, budget)
            except ValueError as e:
                with pytest.raises(ValueError) as e2:
                    batch.plan(ns, pt, budget, cheb=[0] * n)
                assert str(e2.value).split(": ", 1)[1] == str(e).split(": ", 1)[1]
                continue
            assert batch.plan(ns, pt, budget, cheb=[0] * n) == want
    # the documented Jacobi edges, with cheb = NULL and all zero
    for ns, want in {105: (1, 3), 106: (1, 2), 140: (1, 2), 141: (2, 2), 2240: (16, 2)}.items():
        assert batch.plan([ns], [True], SMEM)[0][0][:2] == want
        assert batch.plan([ns], [True], SMEM, cheb=[0])[0][0][:2] == want


def test_bad_cheb_arguments_are_rejected():
    with pytest.raises(ValueError, match="cheb"):
        batch.plan([4, 4], [True, True], SMEM, cheb=[1])
    with pytest.raises(ValueError, match="cheb"):
        batch.plan([4], [True], SMEM, cheb=[1, 0])
    with pytest.raises(ValueError, match=r"cheb\[1\] = 2"):
        batch.plan([4, 4], [True, True], SMEM, cheb=[0, 2])
    with pytest.raises(ValueError, match="cheb"):
        batch.plan([4], [True], SMEM, cheb=[-1])
    with pytest.raises(ValueError):
        batch.plan([], [], SMEM, cheb=[])
    with pytest.raises(ValueError):
        batch.plan([0], [True], SMEM, cheb=[1])
    with pytest.raises(ValueError):
        batch.plan([4], [True], 0, cheb=[1])


def test_preconditioner_names():
    assert batch.preconditioners("jacobi", 2) == ["jacobi", "jacobi"]
    assert batch.preconditioners("chebyshev", 1) == ["chebyshev"]
    assert batch.preconditioners(["chebyshev", "jacobi"], 2) == ["chebyshev", "jacobi"]
    for bad in ("auto", "none", "Chebyshev", ["jacobi", "cheb"], [None, "jacobi"]):
        with pytest.raises(ValueError, match="Unknown preconditioner"):
            batch.preconditioners(bad, 2)
    with pytest.raises(ValueError, match="2 meshes"):
        batch.preconditioners(["jacobi"], 2)
    # checked before any handle is built (no GPU needed)
    with pytest.raises(ValueError, match="Unknown preconditioner"):
        batch.BatchSolver([object()], precond="auto")
    with pytest.raises(ValueError, match="Unknown preconditioner"):
        batch.from_differential_batch([object()], [object()], precond="ssor")
