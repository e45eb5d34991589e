"""CPU: the batch plan (ls_pcg_batch_plan_ex with cheb = NULL, a pure host function) and the host-side argument checks of the batched solve."""
import ctypes

import pytest

import largesteps_b200._native as N
from largesteps_b200 import batch

SMEM = 227 * 1024   # H100: shared memory per CTA with the opt-in carve-out


def test_cluster_sizes_and_residency():
    # pattern-only copy: RES 3 on one CTA up to 105 slices, RES 2 on one CTA up to 140, then 2 / 4 / 8 / 16 CTAs
    edges = {1: (1, 3), 105: (1, 3), 106: (1, 2), 140: (1, 2), 141: (2, 2), 280: (2, 2), 281: (4, 2), 561: (8, 2),
             1120: (8, 2), 1121: (16, 2), 2240: (16, 2)}
    for ns, want in edges.items():
        (got,), ng = batch.plan([ns], [True], SMEM)
        assert got[:2] == want and ng == 1, (ns, got)
    # the general copy keeps 3 more bytes per row (D^-1 instead of a class byte): smaller caps
    for ns, want in {102: (1, 3), 103: (1, 2), 133: (1, 2), 134: (2, 2), 2128: (16, 2)}.items():
        (got,), _ = batch.plan([ns], [False], SMEM)
        assert got[:2] == want, (ns, got)


def test_the_cluster_limit_is_documented_and_names_the_mesh():
    batch.plan([2240], [True], SMEM)          # 71,680 rows
    batch.plan([2128], [False], SMEM)         # 68,096 rows
    for ns, pat in ((2241, True), (2129, False)):
        with pytest.raises(ValueError) as e:
            batch.plan([4, ns], [True, pat], SMEM)
        assert "mesh 1" in str(e.value) and "from_differential" in str(e.value)


def test_groups_by_cluster_size_and_instantiation():
    plan, ng = batch.plan([3] * 5, [True] * 5, SMEM)
    assert ng == 1 and {p for p in plan} == {(1, 3, 0)}
    plan, ng = batch.plan([3, 81, 104, 704, 1650, 3, 104], [1, 1, 0, 1, 1, 0, 0], SMEM)
    assert ng == 5
    assert [p[2] for p in plan] == [0, 0, 1, 2, 3, 4, 1]   # numbered in order of first appearance
    assert [p[0] for p in plan] == [1, 1, 1, 8, 16, 1, 1]
    # a mesh's plan does not depend on the other meshes of the batch
    alone = [batch.plan([ns], [p], SMEM)[0][0][:2] for ns, p in ((3, 1), (81, 1), (104, 0), (704, 1), (1650, 1))]
    assert alone == [p[:2] for p in plan[:5]]
    # a smaller shared-memory budget needs larger clusters
    assert batch.plan([704], [True], 100 * 1024)[0][0][0] == 16


def test_plan_rejects_bad_input():
    with pytest.raises(ValueError):
        batch.plan([], [], SMEM)
    with pytest.raises(ValueError):
        batch.plan([0], [True], SMEM)
    with pytest.raises(ValueError):
        batch.plan([4], [True], 0)


def test_c_entry_points_validate_on_the_host():
    lib = N.lib()
    b = ctypes.c_void_p(0)
    hs = (ctypes.c_void_p * 2)(None, None)
    assert lib.ls_pcg_batch_create(ctypes.byref(b), None, 2, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_pcg_batch_create(ctypes.byref(b), hs, 0, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_pcg_batch_create(ctypes.byref(b), hs, 2, None) == N.LS_ERR_BAD_ARG and "NULL handle" in N.last_error()
    assert not b.value
    assert lib.ls_pcg_batch_solve(None, None, None, None, 3, 1e-7, 100, None, None, None) == N.LS_ERR_BAD_ARG
    assert "batch is NULL" in N.last_error()
    assert lib.ls_pcg_batch_destroy(None) == N.LS_OK


def test_from_differential_batch_rejects_an_empty_list():
    with pytest.raises(ValueError, match="at least one mesh"):
        batch.from_differential_batch([], [])
