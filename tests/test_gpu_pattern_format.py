"""GPU parity of the pattern-only copy's two slice layouts (16-bit column offsets, plain columns) and of its diagonal-class
limit: a matrix with equal off-diagonals but more distinct diagonals than the class table holds takes the general copy."""
import os

import numpy as np
import pytest
import torch

import oracle
from largesteps_b200 import workloads
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.parameterize import to_differential
from largesteps_b200.solvers import PCGSolver
from gpu_util import DEV, to_dev, rel_l2

pytestmark = pytest.mark.gpu


def check(M, u, r, c, val, V, engine):
    s = PCGSolver(M)
    assert s.describe()["sell_engine"] == engine
    x = s.solve(u)
    xd = oracle.DirectSolver(r, c, val, V).solve(u.cpu().numpy())
    assert rel_l2(x.cpu().numpy(), xd) < 1e-5
    assert torch.equal(x, s.solve(u))
    return s


def test_reordered_and_far_numbered_meshes_mix_compact_and_wide_slices(monkeypatch):
    # Morton order on 160K vertices puts some neighbours more than 32767 rows apart; the explicit renumbering guarantees
    # both slice layouts in the native order
    v, f = workloads.plane(400, seed=0)
    V = v.shape[0]
    perm = np.arange(V)
    perm[:1000], perm[V - 1000:] = np.arange(V - 1000, V), np.arange(1000)
    vp = np.empty_like(v)
    vp[perm] = v
    for verts, faces, force in ((v, f, True), (vp, perm[f], False)):
        if force:
            monkeypatch.setenv("LS_FORCE_REORDER", "1")
        else:
            monkeypatch.delenv("LS_FORCE_REORDER", raising=False)
        tv, tf = to_dev(verts, faces)
        M = compute_matrix(tv, tf, lambda_=1.0, alpha=0.95)
        u = to_differential(M, tv)
        r, c, val, Vn = oracle.compute_matrix(np.asarray(verts, np.float64), np.asarray(faces), lambda_=1.0, alpha=0.95)
        s = check(M, u, r, c, val, Vn, 2)
        if force:
            assert s.describe()["reordered"] == 1


def test_too_many_diagonal_classes_take_the_general_copy():
    v, f = workloads.plane(100, seed=0)
    r, c, val, V = oracle.compute_matrix(np.asarray(v, np.float64), np.asarray(f), lambda_=1.0, alpha=0.95)
    val = np.asarray(val, np.float64).copy()
    diag = r == c
    val[diag] += np.arange(V)[r[diag]] * 1e-3          # 10000 distinct diagonals, off-diagonals all equal
    val = val.astype(np.float32)
    M = torch.sparse_coo_tensor(torch.from_numpy(np.stack([r, c])).to(DEV), torch.from_numpy(val).to(DEV), (V, V)).coalesce()
    u = torch.from_numpy(np.random.default_rng(3).normal(size=(V, 3)).astype(np.float32)).to(DEV)
    check(M, u, r, c, val.astype(np.float64), V, 1)
