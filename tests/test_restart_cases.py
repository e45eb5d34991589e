"""CPU: the forced-restart cases of tests/restart_cases.py restart in the model with a margin no rounding difference between
device and model can cross, and the model's true-residual check has the semantics the device tests rely on."""
import numpy as np
import pytest

import oracle
import restart_cases as RC

_sys = {}


def system(name):
    if name not in _sys:
        v, f, kw = RC.MESHES[name]()
        _sys[name] = oracle.compute_matrix(v, f, **kw)
    return _sys[name]


def true_relres(r, c, val, V, b, x):
    A = oracle.solve._csr(r, c, val, V, np.float64)
    rt = b.astype(np.float64) - A @ x.astype(np.float64)
    bn = np.linalg.norm(b.astype(np.float64), axis=0)
    return np.where(bn > 0, np.linalg.norm(rt, axis=0) / np.where(bn > 0, bn, 1), 0.0)


@pytest.mark.parametrize("case", sorted(RC.CASES))
def test_forced_restart_cases_restart_with_margin(case):
    mesh, k, zh, pre, margin = RC.CASES[case]
    r, c, val, V = system(mesh)
    b = RC.rhs(V, k)
    x, it, rs, rec = RC.model(r, c, val, V, b, case, bf16_rows=zh, precond=pre, refine=RC.REFINE, theta=RC.THETA)
    assert rs == RC.REFINE and rec["status"] == 1
    assert rec["checks"][0]["need"].all()
    m = RC.margins(rec, RC.REFINE)
    assert len(m) == k and min(m) >= margin >= RC.MARGIN, m
    # the budget is spent: the second check restarts nothing whatever it finds, and relres is its true residual
    assert len(rec["checks"]) == 2 and not rec["checks"][1]["need"].any()
    np.testing.assert_allclose(rec["relres"], true_relres(r, c, val, V, b, x), rtol=1e-6)


def test_batch_cases_decide_with_margin():
    for i, (mesh, k, zh, pre, th, want) in enumerate(RC.BATCH_CASES):
        r, c, val, V = system(mesh)
        b = RC.rhs(V, k, seed=10 + i)
        _, _, rs, rec = RC.model(r, c, val, V, b, f"batch{i}", bf16_rows=zh, precond=pre, refine=RC.REFINE, theta=th)
        m = RC.margins(rec, RC.REFINE)
        assert rs == want and rec["status"] == 1, (i, rs)
        assert m and all(v >= RC.MARGIN or v <= 1 / RC.MARGIN for v in m), (i, m)


def test_model_budget_spent():
    """refine = 1 where the thresholds would restart twice: one restart, status converged, relres the true residual of
    the last check (above rtol)"""
    r, c, val, V = system("shuffled-stiff")
    b = RC.rhs(V, 3)
    x, it, rs, rec = RC.model(r, c, val, V, b, "jacobi-zh", bf16_rows=True, precond="jacobi", refine=RC.REFINE, theta=RC.THETA)
    last = rec["checks"][-1]
    assert rs == 1 and rec["status"] == 1
    assert (last["rr"] > np.maximum(last["tol"], last["floor"])).any()     # the thresholds alone would restart again
    rel = true_relres(r, c, val, V, b, x)
    np.testing.assert_allclose(rec["relres"], rel, rtol=1e-6)
    assert (rel > 1e-7).all()


def test_model_restart_requested_at_maxit():
    """convergence at exactly maxit followed by a failed check: the restart is counted, status 2, no iteration after it,
    x is the converged x of the first episode and relres is its true residual"""
    r, c, val, V = system("shuffled-stiff")
    b = RC.rhs(V, 3)
    x0_, n1, _, _ = RC.model(r, c, val, V, b, "jacobi-zh", bf16_rows=True, precond="jacobi", refine=0)
    x, it, rs, rec = RC.model(r, c, val, V, b, "jacobi-zh", bf16_rows=True, precond="jacobi", refine=RC.REFINE,
                              theta=RC.THETA, maxit=n1)
    assert it == n1 and rs == 1 and rec["status"] == 2 and len(rec["checks"]) == 1
    assert np.array_equal(x, x0_)
    np.testing.assert_allclose(rec["relres"], true_relres(r, c, val, V, b, x), rtol=1e-6)


def test_model_passed_column_is_left_alone():
    """a column whose check passes (here: converged on entry from an exact guess) is never touched again, the zero column
    stays 0, and the restarted column is the one that needed it"""
    r, c, val, V = system("shuffled-stiff")
    b, x0 = RC.warm_split(r, c, val, V, 3)
    x, it, rs, rec = RC.model(r, c, val, V, b, "split", bf16_rows=True, precond="jacobi", refine=RC.REFINE,
                              theta=RC.THETA, x0=x0)
    assert rs == 1 and rec["status"] == 1
    assert rec["checks"][0]["need"].tolist() == [True, False, False]
    assert rec["checks"][0]["rr"][1] == 0.0
    assert np.array_equal(x[:, 1], x0[:, 1]) and not x[:, 2].any()
    assert RC.margins(rec, RC.REFINE)[0] >= RC.MARGIN
    assert rec["relres"][1] == 0.0 and rec["relres"][2] == 0.0
    # the model without the check: the same columns 1 and 2
    xn, _, _, _ = RC.model(r, c, val, V, b, "split", bf16_rows=True, precond="jacobi", refine=0, x0=x0)
    assert np.array_equal(xn[:, 1:], x[:, 1:])


def test_model_zero_rhs():
    r, c, val, V = system("shuffled-stiff")
    b = np.zeros((V, 3), np.float32)
    x, it, rs, rec = RC.model(r, c, val, V, b, "zero", bf16_rows=True, precond="jacobi", refine=RC.REFINE, theta=RC.THETA)
    assert it == 0 and rs == 0 and rec["status"] == 1 and rec["checks"] == [] and not x.any()
    assert (rec["relres"] == 0).all()


def test_model_record_leaves_the_arithmetic_alone():
    """the record is an output only: the same x, iteration count and restarts with and without it"""
    r, c, val, V = system("shuffled-stiff")
    b = RC.rhs(V, 2, seed=5)
    for kw in (dict(refine=0), dict(refine=3, theta=1.0), dict(refine=1, maxit=50)):
        x1, it1, rs1 = oracle.fused_pcg_f32(r, c, val, V, b, precond="chebyshev", bf16_rows=False, **kw)
        x2, it2, rs2, _ = RC.model(r, c, val, V, b, "rec", precond="chebyshev", bf16_rows=False, **kw)
        assert it1 == it2 and rs1 == rs2 and np.array_equal(x1, x2)
