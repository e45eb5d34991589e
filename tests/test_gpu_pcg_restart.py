"""GPU: the fused solver's true-residual check and restart (restart_from_x(false) in ls_pcg_fused.cuh) against the numpy
model (oracle.fused_pcg_f32 with its record).

Every production solve ends in that check: x rows are gathered from the z buffer, b - A x is accumulated in fp64 over the
general SELL copy (the only place a pattern-copy instantiation reads it), each column restarts when its true residual sits
above both rtol ||b|| and theta 2^-24 || |A||x| ||, and info[2..5] reports the true residual it computed.  A wrong entry of
the general copy, a lost pending x += alpha p or a wrong restart only costs iterations or accuracy there; these tests compare
the check itself:
  * on every instantiation (the recipes of test_gpu_pcg_iterates.REACH, default refine = 1, theta = 3): relres is the true
    residual ||b - A x|| / ||b|| of the returned x, computed on the CPU in fp64; the restart count is the model's; a solve
    whose check passes returns the x and iteration count of the same solve without the check, bit for bit;
  * forced restarts (restart_cases.CASES: stiff meshes, refine = 1, theta = 1) on 17 instantiations, grid and cluster:
    restart count, status and relres against the model, a restart requested at exactly maxit, and the restart's own
    correction x(n1 + j) - x(n1): the model warm-started from the device's x(n1) (restart_from_x(false) sets alpha = beta
    = 0 as the warm start does) against the device, in the norm of the correction.  The converged x is compared too, but a
    restart moves it by ~3e-6 of ||x||_inf, below the device-against-model deviation of the first episode: that comparison
    sees the answer, not the restart.  Also a column whose check passes next to one that restarts (after a warm start), a
    zero right-hand side, and a batch that mixes a mesh that restarts with one that does not.

Thresholds: >= 10x the worst deviation measured on the unmodified build.  Measured on an H100 80GB HBM3 (700 W power limit),
worst over every case of this file (the file ran in 24 s there):
  relres against the CPU fp64 true residual, relative:              5.5e-8   -> RELRES_TOL 1e-6
  converged x, row deviation max_i |x_dev - x_model| / ||x_model||_inf:  zh 3.1e-6, fp32 2.6e-6   -> 5e-5
  restart correction, rel-L2, j = 1, 2, 3, 8:                       3.5e-3 (Chebyshev, 256-thread grid, pattern copy; 0 bit
                                                                    for bit in most cases)   -> CORR_TOL 5e-2
  restart count, status, first-episode count n1 (fp32 rows), bit-for-bit x of a passing check: exact, every case.
The correction is compared in rel-L2 only: it is 10-20 ulps of x per row, so a single ulp flip of x(n1 + j) moves its
max-norm row deviation by ~5 % (measured 5.6e-2 on the unmodified build).
Not compared: the iteration count of the episode after a restart.  It starts from the true residual, which sits at the
rounding level of x (a few 2^-24 || |A||x| ||), and device and model x(n1) differ by ~1e-6 relative: their restarted
residuals have the same size but different content, and the second episode's length differs by up to 24 iterations
(measured: 545-561 against the model's 558 with zh rows, 167 against 150 with Chebyshev, 518 against 539 with K = 4).
Value-only mutants of restart_from_x and what of this file catches them (see the commit that added the file): fp32
accumulation of A x, an unsquared floor, a kept alpha, a general-copy entry of slice 7 scaled by 1.001, the recursive rr in
info, a restart counted at every check, gamma from D^-1 r after a Chebyshev restart.  A kept beta is no mutant: every
column's beta is 0 once it converges (postB), and the check runs only after all have converged.
"""
import warnings

import numpy as np
import pytest

import largesteps_b200._native as N
import oracle
import restart_cases as RC
from largesteps_b200 import batch
from largesteps_b200.batch import BatchSolver
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.solvers import PCGSolver
from gpu_util import to_dev
from test_gpu_pcg_iterates import (GEN, GRID, ITER_WINDOW, NOSMALL, REACH, SINGLE, W, WS, ZERO_COLUMN, inst_id,
                                   reached, rhs_for, set_env, system, t)

pytestmark = pytest.mark.gpu

RELRES_TOL = 1e-6         # |relres_dev - relres_cpu| / relres_cpu: fp32 rounding of r and of the reported float
RESTART_TOL = {("fp32", "conv"): 5e-5, ("zh", "conv"): 5e-5}
# the restart's correction (check_correction): with fp32 rows after 1, 2, 3 and 8 iterations; with bf16 rows after 1 (later
# iterates differ by bf16 rounding flips of single rows, as in test_gpu_pcg_iterates)
CORR_ITS = {"fp32": (1, 2, 3, 8), "zh": (1,)}
CORR_TOL = {("fp32", 1): 5e-2, ("fp32", 2): 5e-2, ("fp32", 3): 5e-2, ("fp32", 8): 5e-2, ("zh", 1): 5e-2}   # rel-L2
RECORD = []               # (case, quantity, value): what the assertions saw, printed at the end of the module


@pytest.fixture(scope="module", autouse=True)
def _print_record():
    yield
    for row in RECORD:
        print("RECORD", *row)


def true_relres(r, c, val, V, b, x):
    A = oracle.solve._csr(r, c, val, V, np.float64)
    rt = b.astype(np.float64) - A @ np.asarray(x, np.float64)
    bn = np.linalg.norm(b.astype(np.float64), axis=0)
    return np.where(bn > 0, np.linalg.norm(rt, axis=0) / np.where(bn > 0, bn, 1), 0.0)


def check_relres(fails, case, relres, r, c, val, V, b, x):
    k = b.shape[1]
    got = np.asarray(relres[:k], np.float64)
    want = true_relres(r, c, val, V, b, x)
    for j in range(k):
        if want[j] == 0:
            if got[j] != 0:
                fails.append(f"{case}: column {j} is zero, relres {got[j]:.3e}")
            continue
        dev = abs(got[j] - want[j]) / want[j]
        RECORD.append((case, "relres", j, f"{got[j]:.4e}", f"{dev:.2e}"))
        if not dev <= RELRES_TOL:
            fails.append(f"{case}: column {j} relres {got[j]:.6e}, true residual {want[j]:.6e}")


def check_x(fails, case, prec, m, x, xm):
    x = np.asarray(x, np.float64)
    xm = np.asarray(xm, np.float64)
    dev = float(np.abs(x - xm).max() / max(np.abs(xm).max(), 1e-30))
    RECORD.append((case, f"x {prec} m={m}", dev))
    if not dev <= RESTART_TOL[(prec, m)]:
        fails.append(f"{case} {prec} m={m}: row deviation {dev:.2e}")


def solve(M, b, maxit, precond, refine, theta, x0=None):
    s = PCGSolver(M, maxit=maxit, refine=refine, theta=theta, precond=precond, warm_start=x0 is not None)
    if x0 is not None:
        s.guess_fwd = t(x0)
    n0 = N.launch_count()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)          # "stopped at maxit": expected where maxit is small
        x = s.solve(t(b)).cpu().numpy()
    assert N.launch_count() - n0 == 1, N.launch_count() - n0      # one launch of the fused kernel
    return s, x


def robust(rec, refine):
    """every threshold decision of the model's checks is at least RC.MARGIN away from its threshold (in norm)"""
    return all(m >= RC.MARGIN or m <= 1 / RC.MARGIN for m in RC.margins(rec, refine))


# ---------------------------------------------------------------- A. the guard on every instantiation, default refinement
@pytest.mark.parametrize("inst", SINGLE, ids=inst_id)
def test_guard_on_every_instantiation(inst, monkeypatch):
    K, res, nw, pat, sync, cheb, zh = inst
    env, name, k = REACH[inst]
    set_env(monkeypatch, env)
    M, (r, c, val, V) = system(name)
    b = rhs_for(inst, V, k)
    precond = "chebyshev" if cheb else "jacobi"
    mprec = "chebyshev" if (cheb and K == 3) else "jacobi"
    case = inst_id(inst)
    s, x = solve(M, b, 10000, precond, refine=1, theta=3.0)
    reached(s, inst, V)
    fails = []
    assert s.status == 1 and s.iterations > 0, (s.status, s.iterations)
    check_relres(fails, case, s.relres, r, c, val, V, b, x)
    if inst in ZERO_COLUMN:
        assert s.relres[1] == 0.0 and not x[:, 1].any()
    RECORD.append((case, "restarts", s.restarts))
    if name not in ("plane1000", "plane2000"):     # the model costs minutes at 10^6 rows and more
        _, _, rs, rec = RC.model(r, c, val, V, b, ("A", name), bf16_rows=zh, precond=mprec, refine=1, theta=3.0)
        if robust(rec, 1):
            assert s.restarts == rs, (s.restarts, rs)
        else:
            RECORD.append((case, "restart decision within 2x of its threshold: count not compared", rs, s.restarts))
    if s.restarts == 0:     # the check passed: it must not have touched x
        s0, x0 = solve(M, b, 10000, precond, refine=0, theta=3.0)
        assert s0.iterations == s.iterations and np.array_equal(x0.view(np.uint32), x.view(np.uint32))
    assert not fails, fails


# ---------------------------------------------------------------- B. forced restarts against the model
_stiff = {}


def stiff_system(name):
    """(M on the device, its coalesced COO on the CPU) of a restart_cases mesh"""
    if name not in _stiff:
        v, f, kw = RC.MESHES[name]()
        M = compute_matrix(*to_dev(v, f), **kw).coalesce()
        idx = M.indices().cpu().numpy()
        _stiff[name] = (M, (idx[0], idx[1], M.values().cpu().numpy(), int(M.shape[0])))
    return _stiff[name]


# instantiation -> (environment, restart_cases case).  The stiff 10^4-row plane reaches the grid and the RES 2 cluster
# instantiations (the 10^6- and 4 10^6-row planes' RES 1 and RES 0 pattern ones by switches), the stiff 2.6 10^3-row
# icospheres the RES 4 (768-thread) ones.  RES 3 and RES 4 with 256 threads have no case (see restart_cases).
CL = {"LS_PCG_CLUSTER": "4"}
FORCED = {
    (3, 2, WS, True, 0, False, True): ({}, "jacobi-zh"),
    (3, 2, WS, False, 0, False, True): ({**GEN}, "jacobi-zh"),
    (3, 2, W, True, 0, False, True): ({**NOSMALL}, "jacobi-zh"),
    (3, 1, W, True, 0, False, True): ({**NOSMALL, "LS_PCG_RES": "1"}, "jacobi-zh"),
    (3, 0, W, True, 0, False, True): ({**NOSMALL, "LS_PCG_RES": "0"}, "jacobi-zh"),
    (3, 2, W, True, 1, False, True): ({**CL}, "jacobi-zh"),
    (3, 2, W, False, 1, False, True): ({**CL, **GEN}, "jacobi-zh"),
    (3, 4, W, True, 1, False, True): ({**CL}, "small-jacobi-zh"),
    (3, 4, W, False, 1, False, True): ({**CL, **GEN}, "small-jacobi-zh"),
    (3, 2, WS, True, 0, True, False): ({}, "chebyshev"),
    (3, 2, WS, False, 0, True, False): ({**GEN}, "chebyshev"),
    (3, 2, W, True, 1, True, False): ({**CL}, "chebyshev"),
    (3, 2, W, False, 1, True, False): ({**CL, **GEN}, "chebyshev"),
    (4, 2, W, False, 0, False, False): ({**GRID}, "jacobi-fp32-k4"),
    (4, 0, W, False, 0, False, False): ({**GRID, "LS_PCG_RES": "0"}, "jacobi-fp32-k4"),
    (4, 2, W, False, 1, False, False): ({**CL}, "jacobi-fp32-k4"),
    (4, 4, W, False, 1, False, False): ({**CL}, "small-jacobi-fp32-k4"),
}


def check_correction(fails, case, prec, j, x1, xj, xmj):
    """the restart's own correction x(n1 + j) - x(n1), device against model, relative to the model's correction"""
    d = np.asarray(xj, np.float64) - np.asarray(x1, np.float64)
    dm = np.asarray(xmj, np.float64) - np.asarray(x1, np.float64)
    row = float(np.abs(d - dm).max() / max(np.abs(dm).max(), 1e-30))
    l2 = float(np.linalg.norm(d - dm) / max(np.linalg.norm(dm), 1e-30))
    RECORD.append((case, f"correction {prec} j={j}", row, l2))
    if not l2 <= CORR_TOL[(prec, j)]:
        fails.append(f"{case} {prec} j={j}: correction deviation {row:.2e} (row), {l2:.2e} (rel-L2)")


@pytest.mark.parametrize("inst", list(FORCED), ids=inst_id)
def test_forced_restart_matches_the_model(inst, monkeypatch):
    env, case = FORCED[inst]
    set_env(monkeypatch, env)
    mesh, k, zh, mprec, _ = RC.CASES[case]
    M, (r, c, val, V) = stiff_system(mesh)
    b = RC.rhs(V, k)
    precond = "chebyshev" if inst[5] else "jacobi"
    prec = "zh" if zh else "fp32"
    cid = inst_id(inst)
    mdl = lambda **kw: RC.model(r, c, val, V, b, case, bf16_rows=zh, precond=mprec, **kw)
    fails = []
    s, x = solve(M, b, 10000, precond, RC.REFINE, RC.THETA)
    reached(s, inst, V)
    xm, itm, rs, rec = mdl(refine=RC.REFINE, theta=RC.THETA)
    assert robust(rec, RC.REFINE)
    RECORD.append((cid, "restarts", s.restarts, "model", rs, "iterations", s.iterations, "model", itm))
    assert s.restarts == rs == 1 and s.status == rec["status"] == 1, (s.restarts, rs, s.status)
    check_x(fails, cid, prec, "conv", x, xm)          # the answer (a restart moves it by ~3e-6 only: this sees episode 1)
    check_relres(fails, cid, s.relres, r, c, val, V, b, x)
    # the first episode alone, then a solve that converges at exactly maxit = n1: the check asks for a restart, which is
    # counted (status 2, no iteration after it), and x and iterations are the first episode's
    s0, x0 = solve(M, b, 10000, precond, 0, RC.THETA)
    n1 = s0.iterations
    s1, x1 = solve(M, b, n1, precond, RC.REFINE, RC.THETA)
    assert (s1.iterations, s1.status, s1.restarts) == (n1, 2, 1), (s1.iterations, s1.status, s1.restarts)
    assert np.array_equal(x1.view(np.uint32), x0.view(np.uint32))
    check_relres(fails, cid + " maxit=n1", s1.relres, r, c, val, V, b, x1)
    if not zh:
        _, n1m, _, _ = mdl(refine=0)
        assert n1 == n1m, (n1, n1m)
    # the restarted recurrence: restart_from_x(false) starts from the device's own x(n1) with alpha = beta = 0, which is the
    # model's warm start from x(n1) (every column of these cases restarts); its correction is compared in its own norm
    for j in CORR_ITS[prec]:
        sj, xj = solve(M, b, n1 + j, precond, RC.REFINE, RC.THETA)
        assert (sj.iterations, sj.status, sj.restarts) == (n1 + j, 2, 1), (sj.iterations, sj.status, sj.restarts)
        xmj, itmj, _, _ = RC.model(r, c, val, V, b, (case, "from x1", cid), bf16_rows=zh, precond=mprec, x0=x1, maxit=j,
                                   refine=0)
        assert itmj == j
        check_correction(fails, cid, prec, j, x1, xj, xmj)
    assert not fails, fails


def test_passed_column_is_left_alone_after_a_warm_start(monkeypatch):
    """a warm start, then a restart of one column: column 0 restarts, column 1 (converged on entry from its exact guess)
    passes its check and column 2 is zero; the columns that did not restart are the refine = 0 solve's, bit for bit"""
    inst = (3, 2, WS, True, 0, False, True)
    set_env(monkeypatch, {})
    M, (r, c, val, V) = stiff_system("shuffled-stiff")
    b, x0 = RC.warm_split(r, c, val, V, 3)
    s, x = solve(M, b, 10000, "jacobi", RC.REFINE, RC.THETA, x0=x0)
    reached(s, inst, V)
    xm, itm, rs, rec = RC.model(r, c, val, V, b, "split", bf16_rows=True, precond="jacobi", refine=RC.REFINE, theta=RC.THETA,
                                x0=x0)
    assert rec["checks"][0]["need"].tolist() == [True, False, False] and robust(rec, RC.REFINE)
    RECORD.append(("warm split", "restarts", s.restarts, "iterations", s.iterations, "model", itm))
    assert s.restarts == rs == 1 and s.status == 1
    assert np.array_equal(x[:, 1], x0[:, 1]) and not x[:, 2].any()
    s0, xz = solve(M, b, 10000, "jacobi", 0, RC.THETA, x0=x0)
    assert np.array_equal(xz[:, 1:].view(np.uint32), x[:, 1:].view(np.uint32))
    fails = []
    check_x(fails, "warm split", "zh", "conv", x, xm)
    check_relres(fails, "warm split", s.relres, r, c, val, V, b, x)
    assert s.relres[1] == 0.0 and s.relres[2] == 0.0
    assert not fails, fails


@pytest.mark.parametrize("inst", [(3, 2, WS, True, 0, False, True), (3, 2, WS, False, 0, True, False)], ids=inst_id)
def test_zero_rhs(inst, monkeypatch):
    """b = 0: no iteration, no check, nothing restarted, x = 0, relres 0"""
    set_env(monkeypatch, FORCED[inst][0])
    M, (r, c, val, V) = stiff_system("shuffled-stiff")
    s, x = solve(M, np.zeros((V, 3), np.float32), 10000, "chebyshev" if inst[5] else "jacobi", RC.REFINE, RC.THETA)
    reached(s, inst, V)
    assert (s.iterations, s.status, s.restarts) == (0, 1, 0)
    assert not x.any() and s.relres[:3] == [0.0, 0.0, 0.0]


def _batch(monkeypatch, Ms, pre, bs, refine, thetas):
    it = iter(thetas)
    monkeypatch.setattr(batch, "PCGSolver", lambda M, **kw: PCGSolver(M, refine=refine, theta=next(it), **kw))
    s = BatchSolver(Ms, precond=pre, check=True)
    xs = [x.cpu().numpy() for x in s.solve([t(b) for b in bs])]
    return s, xs


def test_batch_restart_matches_the_model(monkeypatch):
    """one batch with a mesh that restarts (the stiff plane, pattern copy) and one that passes its check (icosphere 4 with
    cotan weights, general copy), each under Jacobi and Chebyshev: restarts, status, relres and x per mesh against the model,
    and the mesh that does not restart is its refine = 0 result bit for bit"""
    set_env(monkeypatch, {})
    Ms, coo, bs, pre, thetas = [], [], [], [], []
    for i, (mesh, k, _, p, th, _) in enumerate(RC.BATCH_CASES):
        M, (r, c, val, V) = stiff_system(mesh)
        Ms.append(M)
        coo.append((r, c, val, V))
        bs.append(RC.rhs(V, k, seed=10 + i))
        pre.append(p)
        thetas.append(th)
    s, xs = _batch(monkeypatch, Ms, pre, bs, RC.REFINE, thetas)
    s0, xs0 = _batch(monkeypatch, Ms, pre, bs, 0, thetas)
    sd, xsd = _batch(monkeypatch, Ms, pre, bs, 1, [3.0] * len(Ms))     # the default refinement: relres only
    plan, _ = s.plan()
    fails = []
    for i, ((_, res, _), (r, c, val, V), p, th) in enumerate(zip(plan, coo, pre, thetas)):
        want = RC.BATCH_CASES[i][5]
        zh = res == 2 and p == "jacobi"
        case = f"batch {i} {RC.BATCH_CASES[i][0]} {p} RES{res}{' pat' if s.solvers[i].describe()['sell_engine'] == 2 else ' gen'}"
        xm, itm, rs, rec = RC.model(r, c, val, V, bs[i], f"batch{i}", bf16_rows=zh, precond=p, refine=RC.REFINE, theta=th)
        assert robust(rec, RC.REFINE), (case, RC.margins(rec, RC.REFINE))
        RECORD.append((case, "restarts", s.restarts[i], "model", rs, "iterations", s.iterations[i], "model", itm))
        assert s.restarts[i] == rs == want and s.status[i] == rec["status"] == 1, (case, s.restarts, s.status)
        if want == 0 and abs(s.iterations[i] - itm) > ITER_WINDOW:     # (after a restart: not comparable, see above)
            fails.append(f"{case}: {s.iterations[i]} iterations, the model {itm}")
        check_x(fails, case, "zh" if zh else "fp32", "conv", xs[i], xm)
        check_relres(fails, case, s.relres[i], r, c, val, V, bs[i], xs[i])
        if want == 0:
            assert s.iterations[i] == s0.iterations[i] and np.array_equal(xs[i].view(np.uint32), xs0[i].view(np.uint32)), case
        assert sd.status[i] == 1
        check_relres(fails, case + " theta=3", sd.relres[i], r, c, val, V, bs[i], xsd[i])
    assert not fails, fails
