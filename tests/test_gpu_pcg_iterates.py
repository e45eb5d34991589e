"""GPU: the fused solver's iterates against the numpy model of its recurrence (oracle.fused_pcg_f32), for every built
instantiation of lsf::pcg_fused_kernel.

Every other solver test checks a converged answer, and the solve ends with a true-residual check over the general SELL copy
that restarts the iteration when the answer is off: an operator slightly wrong inside the iteration (a pattern-slice decode
error, a bf16 rounding slip, a wrong gather or Chebyshev coefficient) costs a few extra iterations there and nothing else.
With maxit = m and refine = 0 the kernel stops after exactly m iterations (status 2) and returns the m-th iterate of the
recurrence itself, which no restart touches; it is compared with the model's row by row.

The right-hand sides are random-normal: a smooth one would hide a wrong neighbour."""
import os
import warnings
from functools import partial

import numpy as np
import pytest
import torch

import oracle
import largesteps_b200._native as N
from largesteps_b200 import batch, solvers, workloads
from largesteps_b200.batch import BatchSolver
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.solvers import PCGSolver
from gpu_util import DEV, fan_mesh, rel_l2, to_dev
from test_gpu_pattern_share import far_block, morton_mesh, with_fans, with_isolated

pytestmark = pytest.mark.gpu

W, WS = 768, 256          # threads of the production CTA and of the 256-thread CTA (lsf::PT, lsf::PT_SMALL)

# The built instantiations, (K, RES, threads, PAT, SYNC, CHEB, ZH), as listed by ls_fused_a.cu (Jacobi), ls_fused_b.cu
# (Chebyshev), ls_fused_c.cu (K = 4 and the profiling ones) and ls_fused_batch.cu.  ZH (bf16 published rows): K = 3, Jacobi,
# RES != 3; in a batch, Jacobi at RES 2.
JACOBI = ([(3, r, W, p, 0, False, True) for r in (0, 1, 2) for p in (True, False)] +
          [(3, 2, WS, p, 0, False, True) for p in (True, False)] +
          [(3, 2, W, p, 1, False, True) for p in (True, False)] +
          [(3, 3, W, p, 1, False, False) for p in (True, False)] +
          [(3, 4, nw, p, 1, False, True) for nw in (W, WS) for p in (True, False)])
CHEBYSHEV = ([(3, r, W, p, 0, True, False) for r in (0, 1, 2) for p in (True, False)] +
             [(3, 2, WS, p, 0, True, False) for p in (True, False)] +
             [(3, 2, W, p, 1, True, False) for p in (True, False)])
K4 = [(4, 0, W, False, 0, False, False), (4, 1, W, False, 0, False, False), (4, 2, W, False, 0, False, False),
      (4, 2, W, False, 1, False, False), (4, 4, W, False, 1, False, False)]
PROFILING = ([(3, r, W, p, s, False, r != 3) for r, s in ((1, 0), (2, 0), (2, 1), (3, 1), (4, 1)) for p in (True, False)] +
             [(3, 4, WS, p, 1, False, True) for p in (True, False)])
BATCH = [(3, r, W, p, 1, c, r == 2 and not c) for r, c in ((3, False), (2, False), (2, True)) for p in (True, False)]
SINGLE = JACOBI + CHEBYSHEV + K4
assert len(JACOBI) == 16 and len(CHEBYSHEV) == 10 and len(K4) == 5 and len(PROFILING) == 12 and len(BATCH) == 6

# Device-against-model deviation, per row: max_i |x_dev - x_model|_i / ||x_model||_inf, by row precision of the published
# vector (fp32, or bf16 "zh") and iteration count m ("conv": run to rtol = 1e-7 without the true-residual restart).
# Thresholds: >= 10x the worst deviation measured on the unmodified build (H100), and >= 10x below the weakest deviation a
# value-only operator mutant produced (see the PR that added this file for the mutants).
# Measured on an H100 (700 W), worst over every case of this file, row deviation:
#   fp32: m = 1 1.3e-5 (Chebyshev, 256-thread grid), m = 2 4.6e-6, m = 3 3.3e-6, m = 8 3.2e-6, converged 3.3e-6
#   zh:   m = 1 1.5e-7, converged 1.9e-6 (plane2000); m = 2 1.3e-3, m = 3 8.8e-4, m = 8 6.0e-4 (bf16 rounding flips of
#         single rows)
# Weakest mutant signal (largest deviation of the mutant that is hardest to see): 5e-3 (fp32), 8e-4 (zh, m = 1).  A slice-local
# mutant (the SpMV sum of slice 7 scaled by 1.01) moves the zh converged x by 3.7e-4 .. 4.2e-3 on every mesh that has a slice 7.
# Under zh, m = 2, 3 and 8 have no such gap: only m = 1 and the converged run are compared.  The zh m = 1 comparison checks
# little more than one scalar per column: x_1 = alpha_1 z_0 with z_0 = bf16(D^-1 b), which does not involve the off-diagonal
# operator, so a slice-local operator error moves x_1 only through alpha_1 = r.z / z.Az.  What sees such an error row by row
# under zh is the converged run (an operator A' converges to A'^-1 b), which every zh case therefore has, the 10^6- and
# 4 10^6-row planes and the batch included.
ROW_TOL = {
    ("fp32", 1): 1.5e-4, ("fp32", 2): 5e-5, ("fp32", 3): 5e-5, ("fp32", 8): 5e-5, ("fp32", "conv"): 5e-5,
    ("zh", 1): 5e-6, ("zh", "conv"): 2e-5,
}
ITS = {"fp32": (1, 2, 3, 8), "zh": (1,)}
ITER_WINDOW = 3           # converged run: |iterations - model's| <=   (measured: 0 with fp32 rows, at most 1 with zh)
RECORD = []               # (case, precision, m, row deviation, rel-L2): what the assertions saw


def _rec(case, prec, m, x, xm):
    x = np.asarray(x, np.float64)
    xm = np.asarray(xm, np.float64)
    dev = float(np.abs(x - xm).max() / max(np.abs(xm).max(), 1e-30))
    rl = rel_l2(x, xm)
    RECORD.append((case, prec, m, dev, rl))
    return dev, rl


def _check(fails, case, prec, m, x, xm):
    dev, rl = _rec(case, prec, m, x, xm)
    tol = ROW_TOL[(prec, m)]
    if not (dev <= tol and rl <= tol):
        fails.append(f"{case} {prec} m={m}: row deviation {dev:.2e}, rel-L2 {rl:.2e} > {tol:.0e}")


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def device():
    p = torch.cuda.get_device_properties(DEV)
    return p.multi_processor_count, p.shared_memory_per_block_optin


# ---------------------------------------------------------------- meshes: the shapes where kernels go wrong
def _bunny():
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "bunny_mesh.npz"))
    return workloads.subdivide(d["verts"], d["faces"].astype(np.int64))


def one_triangle():
    return np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.array([[0, 1, 2]], np.int64)


UNI = dict(lambda_=1.0, alpha=0.95)
MESHES = {
    "triangle": lambda: (*one_triangle(), dict(lambda_=10.0)),                  # one slice, 3 rows
    "ico1": lambda: (*workloads.icosphere(1), dict(lambda_=10.0)),              # 42 rows: a partial second slice
    "ico2": lambda: (*workloads.icosphere(2), dict(lambda_=10.0)),              # 162 rows
    "ico3": lambda: (*workloads.icosphere(3), dict(lambda_=10.0)),              # 21 slices: one CTA
    "ico4": lambda: (*workloads.icosphere(4), dict(lambda_=10.0)),
    "ico4cot": lambda: (*workloads.icosphere(4), dict(lambda_=10.0, cotan=True)),
    "fan": lambda: (*fan_mesh(100), dict(lambda_=10.0)),                        # a hub row of 101 entries: a wide slice
    "bunny": lambda: (*_bunny(), dict(lambda_=19.0, cotan=True)),               # general copy
    "isolated": lambda: (*with_isolated(*workloads.icosphere(4)), dict(lambda_=10.0)),   # rows with only a diagonal
    "farblock200": lambda: (*far_block(200), UNI),                              # compact slices mixed with wide ones
    "fans200": lambda: (*with_fans(200), UNI),                                  # escape slices and the slices after them
    "morton300": lambda: (*morton_mesh(300), UNI),                              # many shared slices
    "shuffled": lambda: (*workloads.shuffle_vertices(*workloads.plane(100, seed=3)), UNI),   # 10^4 rows: Morton copy on
    "plane1000": lambda: (*workloads.plane(1000, seed=0), UNI),                 # the benchmark's configuration
    "plane2000": lambda: (*workloads.plane(2000, seed=0), UNI),                 # RES 0 by size
}

GRID = {"LS_PCG_CLUSTER": "0"}
NOSMALL = {"LS_PCG_CLUSTER": "0", "LS_PCG_SMALLCTA": "0"}
GEN = {"LS_PCG_PATTERN": "0"}

# instantiation -> (environment, mesh, k) that reach it; the preconditioner follows from CHEB (K = 4 always runs Jacobi)
REACH = {
    (3, 0, W, True, 0, False, True): ({}, "plane2000", 3),
    (3, 0, W, False, 0, False, True): ({**GRID, "LS_PCG_RES": "0", **GEN}, "bunny", 2),
    (3, 1, W, True, 0, False, True): ({}, "plane1000", 3),
    (3, 1, W, False, 0, False, True): ({**GRID, "LS_PCG_RES": "1", **GEN}, "shuffled", 3),
    (3, 2, W, True, 0, False, True): ({}, "morton300", 3),
    (3, 2, W, False, 0, False, True): ({**NOSMALL, **GEN}, "farblock200", 1),
    (3, 2, WS, True, 0, False, True): ({}, "fans200", 3),
    (3, 2, WS, False, 0, False, True): ({**GEN}, "isolated", 3),
    (3, 2, W, True, 1, False, True): ({"LS_PCG_RES": "2"}, "ico3", 3),
    (3, 2, W, False, 1, False, True): ({"LS_PCG_RES": "2", **GEN}, "fan", 2),
    (3, 3, W, True, 1, False, False): ({}, "triangle", 3),
    (3, 3, W, False, 1, False, False): ({**GEN}, "ico2", 1),
    (3, 4, W, True, 1, False, True): ({"LS_PCG_CLUSTER": "4"}, "isolated", 3),
    (3, 4, W, False, 1, False, True): ({"LS_PCG_CLUSTER": "4"}, "ico4cot", 3),
    (3, 4, WS, True, 1, False, True): ({"LS_PCG_CLUSTER": "4"}, "fan", 3),
    (3, 4, WS, False, 1, False, True): ({"LS_PCG_CLUSTER": "4", **GEN}, "ico1", 2),
    (3, 0, W, True, 0, True, False): ({**NOSMALL, "LS_PCG_RES": "0"}, "farblock200", 3),
    (3, 0, W, False, 0, True, False): ({**NOSMALL, "LS_PCG_RES": "0", **GEN}, "ico3", 3),
    (3, 1, W, True, 0, True, False): ({**NOSMALL, "LS_PCG_RES": "1"}, "morton300", 3),
    (3, 1, W, False, 0, True, False): ({**NOSMALL, "LS_PCG_RES": "1"}, "bunny", 3),
    (3, 2, W, True, 0, True, False): ({**NOSMALL}, "fans200", 3),
    (3, 2, W, False, 0, True, False): ({**NOSMALL, **GEN}, "shuffled", 3),
    (3, 2, WS, True, 0, True, False): ({**GRID}, "isolated", 3),
    (3, 2, WS, False, 0, True, False): ({}, "ico4cot", 2),
    (3, 2, W, True, 1, True, False): ({}, "ico3", 3),
    (3, 2, W, False, 1, True, False): ({**GEN}, "fan", 1),
    (4, 0, W, False, 0, False, False): ({**GRID, "LS_PCG_RES": "0"}, "ico4", 4),
    (4, 1, W, False, 0, False, False): ({**GRID, "LS_PCG_RES": "1"}, "farblock200", 4),
    (4, 2, W, False, 0, False, False): ({**GRID}, "isolated", 4),
    (4, 2, W, False, 1, False, False): ({}, "ico3", 4),
    (4, 4, W, False, 1, False, False): ({"LS_PCG_CLUSTER": "4"}, "ico4", 4),
}
assert set(REACH) == set(SINGLE)
ZERO_COLUMN = {(3, 2, WS, False, 0, False, True), (4, 2, W, False, 0, False, False)}   # b with one all-zero column


def inst_id(i):
    K, res, nw, pat, sync, cheb, zh = i
    return f"K{K}-RES{res}-{nw}t-{'pat' if pat else 'gen'}-{'cluster' if sync else 'grid'}{'-cheb' if cheb else ''}{'-zh' if zh else ''}"


_cache = {}


def system(name):
    """(M on the device, the matrix as the device received it: coalesced COO on the CPU)"""
    if name not in _cache:
        _cache.clear()
        v, f, kw = MESHES[name]()
        M = compute_matrix(*to_dev(v, f), **kw).coalesce()
        idx = M.indices().cpu().numpy()
        _cache[name] = (M, (idx[0], idx[1], M.values().cpu().numpy(), int(M.shape[0])))
    return _cache[name]


def set_env(monkeypatch, env):
    for k_ in ("LS_PCG_MODE", "LS_PCG_CLUSTER", "LS_PCG_RES", "LS_PCG_ONECTA", "LS_PCG_CLRES", "LS_PCG_SMALLCTA",
               "LS_PCG_PATTERN", "LS_PCG_PROFILE", "LS_PCG_CHEB_M", "LS_SPMM_ENGINE", "LS_SELL_TMA", "LS_FORCE_REORDER"):
        monkeypatch.delenv(k_, raising=False)
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)


def rhs_for(inst, V, k, seed=0):
    b = np.random.default_rng(seed).normal(size=(V, k)).astype(np.float32)
    if inst in ZERO_COLUMN:
        b[:, 1] = 0.0
    return b


def reached(s, inst, V):
    """the plan of handle `s` (and, for K = 4, the host plan of the same switches) is the instantiation `inst`"""
    K, res, nw, pat, sync, cheb, zh = inst
    d = s.describe()
    sms, smem = device()
    ns = (V + 31) // 32
    precond = "chebyshev" if cheb else "jacobi"
    got3 = {k_: d[k_] for k_ in ("grid", "cluster", "residency", "threads", "precond")}
    assert d["algo"] == "fused"
    if K == 3:
        got = (3, d["residency"], d["threads"], d["sell_engine"] == 2, 1 if d["cluster"] else 0, d["precond"] == "chebyshev",
               zh)
        assert got == inst, (inst_id(inst), d)
    else:   # describe() reports the 3-column configuration; the 4-column one comes from the same plan function
        p3 = solvers.plan(ns, d["sell_engine"] == 2, sms, smem, precond="jacobi", k=3)
        assert {k_: p3[k_] for k_ in got3} == got3, (p3, d)
        p4 = solvers.plan(ns, False, sms, smem, precond="jacobi", k=4)
        got = (4, p4["residency"], p4["threads"], False, 1 if p4["cluster"] else 0, False, False)
        assert got == inst, (inst_id(inst), p4)


def run_dev(M, b, m, precond, refine=0, x0=None, fused=True):
    s = PCGSolver(M, maxit=m, refine=refine, precond=precond, warm_start=x0 is not None)
    if x0 is not None:
        s.guess_fwd = t(x0)
    n0 = N.launch_count()
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)          # "stopped at maxit": expected
        x = s.solve(t(b)).cpu().numpy()
    if fused:   # one launch of the fused kernel (a refused launch falls back to the graph-mode solver: 3 kernels per iteration)
        assert N.launch_count() - n0 == 1, N.launch_count() - n0
    return s, x


def compare_converged(fails, case, prec, its, itm, x, xm):
    RECORD.append((case, prec, "iterations", abs(its - itm), 0.0))
    if abs(its - itm) > ITER_WINDOW:
        fails.append(f"{case}: {its} iterations, the model {itm}")
    _check(fails, case, prec, "conv", x, xm)


@pytest.mark.parametrize("inst", SINGLE, ids=inst_id)
def test_iterates_match_the_model(inst, monkeypatch):
    K, res, nw, pat, sync, cheb, zh = inst
    env, name, k = REACH[inst]
    set_env(monkeypatch, env)
    M, (r, c, val, V) = system(name)
    b = rhs_for(inst, V, k)
    precond = "chebyshev" if cheb else "jacobi"
    mprec = "chebyshev" if (cheb and K == 3) else "jacobi"
    prec = "zh" if zh else "fp32"
    model = lambda **kw: oracle.fused_pcg_f32(r, c, val, V, b, bf16_rows=zh, precond=mprec, **kw)
    fails = []
    its = ITS[prec]
    for m in its:
        s, x = run_dev(M, b, m, precond)
        if m == its[0]:
            reached(s, inst, V)
            if name == "shuffled":
                assert s.describe()["reordered"] == 1
        xm, itm, _ = model(maxit=m, refine=0)
        # stopped by maxit (status 2) unless the model converges first (the one-triangle mesh does within 3 iterations)
        assert s.iterations == itm and s.status in ((1, 2) if itm == m else (1,)), (m, itm, s.status, s.iterations)
        _check(fails, inst_id(inst), prec, m, x, xm)
    # converged without the restart: the same iteration count within a window, the same x
    s, x = run_dev(M, b, 10000, precond)
    xm, itm, _ = model(refine=0)
    assert s.status == 1
    compare_converged(fails, inst_id(inst), prec, s.iterations, itm, x, xm)
    # warm start from the model's 8th iterate: the fp64 true residual, per-column convergence on entry
    x0, _, _ = model(maxit=8, refine=0)
    m = 3 if prec == "fp32" else 1
    s, x = run_dev(M, b, m, precond, x0=x0)
    xm, itm, _ = model(maxit=m, refine=0, x0=x0)
    assert s.iterations == itm, (s.iterations, itm)
    _check(fails, inst_id(inst) + " warm", prec, m, x, xm)
    assert not fails, fails


@pytest.mark.parametrize("inst", [(3, 3, W, False, 1, False, False), (3, 2, WS, False, 0, False, True),
                                  (3, 2, WS, True, 0, False, True)], ids=inst_id)
def test_no_preconditioner(inst, monkeypatch):
    """precond='none' runs the Jacobi instantiations with D^-1 = 1 (the pattern copy's diagonal class table included)"""
    env, _, _ = REACH[inst]
    set_env(monkeypatch, env)
    name = "ico2" if inst[1] == 3 else "isolated"
    M, (r, c, val, V) = system(name)
    b = rhs_for(None, V, 3, seed=4)
    prec = "zh" if inst[6] else "fp32"
    fails = []
    for m in ITS[prec]:
        s, x = run_dev(M, b, m, "none")
        d = s.describe()
        assert d["precond"] == "none" and d["residency"] == inst[1] and d["threads"] == inst[2] and (d["sell_engine"] == 2) == inst[3]
        assert s.status == 2 and s.iterations == m
        xm, _, _ = oracle.fused_pcg_f32(r, c, val, V, b, maxit=m, refine=0, bf16_rows=inst[6], precond="none")
        _check(fails, "none " + inst_id(inst), prec, m, x, xm)
    s, x = run_dev(M, b, 10000, "none")
    xm, itm, _ = oracle.fused_pcg_f32(r, c, val, V, b, refine=0, bf16_rows=inst[6], precond="none")
    assert s.status == 1
    compare_converged(fails, "none " + inst_id(inst), prec, s.iterations, itm, x, xm)
    assert not fails, fails


@pytest.mark.parametrize("inst", PROFILING, ids=inst_id)
def test_profiling_instantiations_are_bitwise_the_production_ones(inst, monkeypatch):
    """LS_PCG_PROFILE=1 (read at solve time) swaps in the instantiation with per-phase clock reads; nothing else changes."""
    prod = tuple(inst)
    env, name, k = REACH[prod]
    set_env(monkeypatch, env)
    M, (r, c, val, V) = system(name)
    b = rhs_for(prod, V, k, seed=1)
    s = PCGSolver(M)
    reached(s, prod, V)
    x = s.solve(t(b)).cpu().numpy()
    it = s.iterations
    monkeypatch.setenv("LS_PCG_PROFILE", "1")
    xp = s.solve(t(b)).cpu().numpy()
    assert s.iterations == it and np.array_equal(x.view(np.uint32), xp.view(np.uint32))
    cyc = s.phase_cycles()
    assert cyc["iterations"] == it and cyc["phaseA"] > 0 and cyc["phaseB"] > 0      # the profiling kernel ran


BATCH_MESHES = [("ico2", "jacobi"), ("ico2cot", "jacobi"), ("ico5", "jacobi"), ("ico5cot", "jacobi"),
                ("ico3", "chebyshev"), ("plane60cot", "chebyshev")]


def test_batch_iterates_match_the_model(monkeypatch):
    """one heterogeneous batch that reaches every batch instantiation: RES 3 / RES 2 x pattern / general (Jacobi), and
    Chebyshev x pattern / general; each mesh's x_m and converged x (without the true-residual restart) are the model's"""
    set_env(monkeypatch, {})
    # the batch takes each mesh's refinement setting from its handle: build them without the restart
    monkeypatch.setattr(batch, "PCGSolver", partial(PCGSolver, refine=0))
    mk = {"ico2": (*workloads.icosphere(2), dict(lambda_=10.0)), "ico2cot": (*workloads.icosphere(2), dict(lambda_=10.0, cotan=True)),
          "ico5": (*workloads.icosphere(5), dict(lambda_=10.0)), "ico5cot": (*workloads.icosphere(5), dict(lambda_=10.0, cotan=True)),
          "ico3": (*workloads.icosphere(3), dict(lambda_=10.0)), "plane60cot": (*workloads.plane(60, seed=4), dict(lambda_=5.0, cotan=True))}
    Ms, coo = [], []
    for name, _ in BATCH_MESHES:
        v, f, kw = mk[name]
        M = compute_matrix(*to_dev(v, f), **kw).coalesce()
        idx = M.indices().cpu().numpy()
        Ms.append(M)
        coo.append((idx[0], idx[1], M.values().cpu().numpy(), int(M.shape[0])))
    pre = [p for _, p in BATCH_MESHES]
    bs = [np.random.default_rng(10 + i).normal(size=(V, 3)).astype(np.float32) for i, (_, _, _, V) in enumerate(coo)]
    fails = []
    for m in (1, 2, 3, 8, "conv"):
        s = BatchSolver(Ms, maxit=10000 if m == "conv" else m, precond=pre, check=True)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", RuntimeWarning)
            xs = [x.cpu().numpy() for x in s.solve([t(b) for b in bs])]
        if m == "conv":
            assert s.status == [1] * len(Ms), s.status
        else:
            assert s.status == [2] * len(Ms) and s.iterations == [m] * len(Ms), (s.status, s.iterations)
        plan, _ = s.plan()
        insts = []
        for i, ((cs, res, _), (r, c, val, V), p) in enumerate(zip(plan, coo, pre)):
            pat = s.solvers[i].describe()["sell_engine"] == 2
            cheb = p == "chebyshev"
            inst = (3, res, W, pat, 1, cheb, res == 2 and not cheb)
            insts.append(inst)
            prec, case = "zh" if inst[6] else "fp32", f"batch {BATCH_MESHES[i][0]} {inst_id(inst)}"
            if m == "conv":
                xm, itm, _ = oracle.fused_pcg_f32(r, c, val, V, bs[i], refine=0, bf16_rows=inst[6], precond=p)
                compare_converged(fails, case, prec, s.iterations[i], itm, xs[i], xm)
            elif m in ITS[prec]:
                xm, _, _ = oracle.fused_pcg_f32(r, c, val, V, bs[i], maxit=m, refine=0, bf16_rows=inst[6], precond=p)
                _check(fails, case, prec, m, xs[i], xm)
        assert sorted(insts) == sorted(BATCH), [inst_id(i) for i in insts]
    assert not fails, fails


@pytest.mark.parametrize("engine", [{}, {"LS_SELL_TMA": "0"}, {"LS_SPMM_ENGINE": "csr"}], ids=["sell-tma", "sell", "csr"])
def test_graph_mode_iterates_match_the_model(engine, monkeypatch):
    """LS_PCG_MODE=graph (classic PCG, three kernels per iteration) against oracle.jacobi_pcg_f32, with each SpMM engine,
    cold and warm (the residual b - A x0 from the fp32 SpMM; a guess worse than zero starts cold)."""
    set_env(monkeypatch, {"LS_PCG_MODE": "graph", **engine})
    fails = []
    for name, k in (("isolated", 3), ("fan", 2)):
        M, (r, c, val, V) = system(name)
        b = np.random.default_rng(2).normal(size=(V, k)).astype(np.float32)
        for m in (1, 2, 3, 8):
            s, x = run_dev(M, b, m, "jacobi", fused=False)
            d = s.describe()
            assert d["algo"] == "graph" and d["sell_engine"] == (0 if engine.get("LS_SPMM_ENGINE") == "csr" else 1)
            assert s.status == 2 and s.iterations == m
            xm, itm, _ = oracle.jacobi_pcg_f32(r, c, val, V, b, maxit=m)
            _check(fails, f"graph {name} {engine}", "fp32", m, x, xm)
        x0, _, _ = oracle.jacobi_pcg_f32(r, c, val, V, b, maxit=8)
        bad = np.zeros_like(b)
        bad[:, 0] = 30.0 * np.random.default_rng(3).normal(size=V)
        for guess, tag in ((x0, "warm"), (bad, "worse than zero")):
            s, x = run_dev(M, b, 3, "jacobi", x0=guess, fused=False)
            assert s.iterations == 3
            xm, _, _ = oracle.jacobi_pcg_f32(r, c, val, V, b, x0=guess, maxit=3)
            _check(fails, f"graph {name} {engine} {tag}", "fp32", 3, x, xm)
    assert not fails, fails


def test_the_tables_cover_every_built_instantiation():
    """Each instantiation of the tables above has a recipe that reaches it; the tests above each assert that theirs was
    reached (describe() / the plan), so a plan change that stops reaching one of them fails there."""
    assert set(REACH) == set(SINGLE) and len(SINGLE) == 31
    assert set(PROFILING) <= set(REACH)
    assert len(set(BATCH)) == 6
