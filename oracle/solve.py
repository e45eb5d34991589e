"""Oracle: CPU solves for M x = b (TEST INFRASTRUCTURE, see oracle/__init__.py).

  * DirectSolver          fp64 (or fp32) sparse direct solve -- the stand-in for the reference's
                          CholeskySolver (solvers.py:26-39 -> cholespy/CHOLMOD, absent here).
                          SuperLU in symmetric mode: factor once, solve many (V,k) right-hand sides.
  * dense_cholesky_solve  numpy LL^T for V <= ~3K, second opinion on DirectSolver.
  * reference_cg / ReferenceCG   restatement of ConjugateGradientSolver (solvers.py:41-126):
                          plain CG per axis, ABSOLUTE tolerance 1e-5, warm start kept for fwd/bwd.
  * to_differential       parameterize.py:30  (u = M @ v)
  * jacobi_pcg_f32        numpy model of the graph-mode device algorithm (fp32 vectors, fp64 dot products,
                          per-column alpha/beta/convergence, warm start with the worse-than-zero fallback).
  * fused_pcg_f32         numpy model of the fused kernel's recurrence (ls_pcg_fused.cuh): Jacobi, none or Chebyshev,
                          bf16 published rows, warm start, true-residual restart.  With maxit = m its x is the device's
                          m-th iterate, which tests/test_gpu_pcg_iterates.py compares row by row.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

f32 = np.float32


def _csr(rows, cols, vals, V, dtype):
    return sp.csr_matrix((np.asarray(vals).astype(dtype), (np.asarray(rows), np.asarray(cols))), shape=(V, V))


class DirectSolver:
    """Factor once (SuperLU, symmetric mode, MMD(A^T+A) ordering), then x = M^{-1} b for (V,k)."""

    def __init__(self, rows, cols, vals, V, dtype=np.float64):
        self.V = V
        self.dtype = dtype
        A = _csr(rows, cols, vals, V, dtype).tocsc()
        self.lu = spla.splu(A, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0,
                            options={"SymmetricMode": True})
        self.factor_nnz = int(self.lu.L.nnz + self.lu.U.nnz)

    def solve(self, b, backward=False):   # same signature as solvers.py:36 (M symmetric: bwd == fwd)
        return self.lu.solve(np.ascontiguousarray(b, dtype=self.dtype))


def dense_cholesky_solve(rows, cols, vals, V, b):
    A = _csr(rows, cols, vals, V, np.float64).toarray()
    Lc = np.linalg.cholesky(A)
    y = np.linalg.solve(Lc, np.asarray(b, dtype=np.float64))
    return np.linalg.solve(Lc.T, y)


def to_differential(rows, cols, vals, V, v):
    """parameterize.py:30 in fp32."""
    return (_csr(rows, cols, vals, V, f32) @ np.asarray(v, dtype=f32)).astype(f32)


def reference_cg(A, b, x0, tol=1e-5, maxit=100000):
    """solvers.py:58-84 (solve_axis), fp32.  `maxit` is a safety net the reference lacks."""
    x = x0.astype(f32).copy()
    r = (A @ x - b).astype(f32)                # solvers.py:70
    p = -r                                     # solvers.py:71
    r_norm = f32(np.sqrt(np.dot(r, r)))        # solvers.py:72
    it = 0
    while r_norm > tol and it < maxit:         # solvers.py:73 (absolute)
        Ap = (A @ p).astype(f32)               # solvers.py:74
        r2 = f32(r_norm * r_norm)              # solvers.py:75
        alpha = f32(r2 / f32(np.dot(p, Ap)))   # solvers.py:76
        x = (x + alpha * p).astype(f32)        # solvers.py:77
        r = (r + alpha * Ap).astype(f32)       # solvers.py:80
        r_norm = f32(np.sqrt(np.dot(r, r)))    # solvers.py:81
        beta = f32(f32(r_norm * r_norm) / r2)  # solvers.py:82
        p = (-r + beta * p).astype(f32)        # solvers.py:83
        it += 1
    return x, it


class ReferenceCG:
    """solvers.py:41-126: per-axis CG with separate fwd/bwd warm starts."""

    def __init__(self, rows, cols, vals, V):
        self.A = _csr(rows, cols, vals, V, f32)
        self.guess_fwd = None
        self.guess_bwd = None
        self.iters = []

    def solve(self, b, backward=False):
        b = np.asarray(b, dtype=f32)
        if self.guess_fwd is None:                              # solvers.py:102-105
            self.guess_bwd = np.zeros_like(b)
            self.guess_fwd = np.zeros_like(b)
        x0 = self.guess_bwd if backward else self.guess_fwd     # solvers.py:107-110
        if b.ndim != 2:                                         # solvers.py:112-113
            raise ValueError(f"Invalid array shape {b.shape} for ConjugateGradientSolver.solve: expected shape (a, b)")
        x = np.zeros_like(b)
        self.iters = []
        for axis in range(b.shape[1]):                          # solvers.py:115-118
            x[:, axis], it = reference_cg(self.A, b[:, axis], x0[:, axis])
            self.iters.append(it)
        if backward:                                            # solvers.py:120-124
            self.guess_bwd = x
        else:
            self.guess_fwd = x
        return x


def jacobi_pcg_f32(rows, cols, vals, V, b, x0=None, rtol=1e-7, maxit=10000, precond=True):
    """Model of the graph-mode device PCG: all k columns in lock-step with per-column alpha/beta/freeze,
    fp32 vectors, fp64 dot products, relative residual test ||r||_2 <= rtol ||b||_2 per column.
    Warm start (k_warm_load, k_init<K, true>): r = b - A x0 with the fp32 SpMM; a guess whose residual exceeds ||b|| in any
    column is worse than x = 0 and the solve starts cold instead."""
    A = _csr(rows, cols, vals, V, f32)
    b = np.asarray(b, dtype=f32)
    k = b.shape[1]
    dinv = (f32(1.0) / A.diagonal().astype(f32)) if precond else np.ones(V, dtype=f32)
    d = lambda u, w: np.einsum("ij,ij->j", u.astype(np.float64), w.astype(np.float64))
    bb = d(b, b)
    x, r = np.zeros_like(b), b.copy()
    if x0 is not None:
        xw = np.asarray(x0, dtype=f32).copy()
        rw = (b - (A @ xw).astype(f32)).astype(f32)
        if not (d(rw, rw) > bb).any():
            x, r = xw, rw
    z = (dinv[:, None] * r).astype(f32)
    p = z.copy()
    rz = d(r, z)
    rr = d(r, r)
    active = rr > (rtol * rtol) * bb
    it = 0
    while active.any() and it < maxit:
        Ap = (A @ p).astype(f32)
        pAp = d(p, Ap)
        alpha = np.where(active & (pAp > 0), rz / np.where(pAp == 0, 1, pAp), 0.0).astype(f32)
        x = (x + alpha[None, :] * p).astype(f32)
        r = (r - alpha[None, :] * Ap).astype(f32)
        z = (dinv[:, None] * r).astype(f32)
        rz_new = d(r, z)
        rr = d(r, r)
        beta = np.where(active, rz_new / np.where(rz == 0, 1, rz), 0.0).astype(f32)
        p = (z + beta[None, :] * p).astype(f32)
        rz = rz_new
        it += 1
        active = active & (rr > (rtol * rtol) * bb)
    relres = np.sqrt(rr / np.where(bb == 0, 1, bb))
    return x, it, relres


def _bf16(x):
    """round-to-nearest-even to bfloat16, returned as float32 (what cvt.rn.bf16.f32 + a 16-bit shift give on the device)"""
    u = np.ascontiguousarray(x, dtype=f32).view(np.uint32)
    r = ((u >> 16) & 1) + 0x7fff
    return ((u + r) & np.uint32(0xffff0000)).view(f32)


def gershgorin_bound(rows, cols, vals, V):
    """max_i sum_j |a_ij| / a_ii in fp32 (k_gershgorin): the bound of lambda_max(D^-1 A) the Chebyshev interval is built on."""
    A = _csr(rows, cols, vals, V, f32)
    sabs = np.asarray(abs(A).sum(axis=1), dtype=f32).ravel()
    dg = A.diagonal().astype(f32)
    return f32(np.max(np.where(dg > 0, sabs / np.where(dg > 0, dg, 1), 0), initial=0))


def chebyshev_coefficients(gersh, m=4):
    """(c0, c1[m - 1], c2[m - 1]) of the Chebyshev semi-iteration for D^-1 A on [b / 30, b], b = 1.02 gersh, computed in double
    and stored as float as ls_pcg_create does; m is clamped to 2..8 as LS_PCG_CHEB_M is."""
    m = min(max(int(m), 2), 8)
    bnd = 1.02 * float(gersh)
    a = bnd / 30.0
    th, de = 0.5 * (bnd + a), 0.5 * (bnd - a)
    sg = th / de
    rho = 1.0 / sg
    c1, c2 = [], []
    for _ in range(1, m):
        rn = 1.0 / (2.0 * sg - rho)
        c1.append(f32(rn * rho))
        c2.append(f32(2.0 * rn / de))
        rho = rn
    return f32(1.0 / th), np.array(c1, dtype=f32), np.array(c2, dtype=f32)


def _fma32(a, b, c):
    """fmaf(a, b, c): the fp32 product is exact in double, one rounding to fp32 at the end"""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(c, np.float64)).astype(f32)


def fused_pcg_f32(rows, cols, vals, V, b, rtol=1e-7, maxit=10000, bf16_rows=True, refine=1, theta=3.0, x0=None,
                  precond="jacobi", cheb_m=4, record=None):
    """Model of ls_pcg_fused.cuh.  Per iteration:
         phase B  r -= alpha s;  z = rnd(M^-1 r);  gamma' = r.z, rr = r.r        -> reduction 1 (beta, convergence)
         phase A  w = A z;  x += alpha_prev p;  p = z + beta p;  s = w + beta s;  delta = p.s   -> reduction 2 (alpha)
       and at convergence the true residual b - A x (fp64) decides whether to restart (see DESIGN.md 4.1).
       rows/cols/vals: the matrix as the device receives it (compute_matrix's coalesced COO, fp32 values).
       precond: "jacobi" (M = D), "none" (M = I) or "chebyshev": z = y_m of the Chebyshev semi-iteration (cheb_first /
       cheb_steps): y_1 = c0 D^-1 r, d_1 = y_1, d_j = c1 d_{j-1} + c2 D^-1 (r - A y_j), y_{j+1} = y_j + d_j, with fp32 rows
       (bf16_rows applies to Jacobi and "none" only).  The K = 4 instantiations run Jacobi whatever precond says: pass "jacobi".
       x0: warm start as restart_from_x(true): the fp64 true residual, per-column convergence on entry, and a cold start
       instead when ||b - A x0|| > ||b|| in any column.
       record: a dict to fill with what the device reports and decides beside x (the arithmetic does not change):
         "checks"  one dict per true-residual check: "it" (iterations so far), per column "rr" (||b - A x||^2 of the fp32
                   residual), "tol" (rtol^2 bb), "floor" ((theta 2^-24)^2 ||(|A||x|)||^2) and "need" (restart this column)
         "status"  1 converged (also when the restart budget is spent), 2 stopped at maxit (also when the last check asked
                   for a restart that no iteration was left to run); the model has no breakdown, so never the kernel's 3
                   (not SPD, or NaN)
         "relres"  per column what the kernel writes to info[2..5]: sqrt(rr / bb) of the last rr it stored for the column
                   (the true residual of the last check, else the warm start's, else the recursive one), 0 for b = 0
       Returns (x, iterations, restarts)."""
    if precond not in ("jacobi", "none", "chebyshev"):
        raise ValueError(f"unknown preconditioner {precond!r}")
    A = _csr(rows, cols, vals, V, f32)
    A64, Aabs = A.astype(np.float64), abs(A.astype(np.float64))
    b = np.asarray(b, dtype=f32)
    dinv = (f32(1.0) / A.diagonal().astype(f32)) if precond != "none" else np.ones(V, dtype=f32)
    d = lambda u, w: np.einsum("ij,ij->j", u.astype(np.float64), w.astype(np.float64))
    cheb = precond == "chebyshev"
    rnd = _bf16 if (bf16_rows and not cheb) else (lambda t: t)
    if cheb:
        c0, c1, c2 = chebyshev_coefficients(gershgorin_bound(rows, cols, vals, V), cheb_m)
        dc0 = (dinv * c0).astype(f32)

    def prec(r):   # (z, gamma = r.z)
        if not cheb:
            z = rnd((dinv[:, None] * r).astype(f32))
            return z, d(r, z)
        y = (dc0[:, None] * r).astype(f32)
        dd = y
        for j in range(len(c1)):
            t = (A @ y).astype(f32)
            g = (c2[j] * (dinv[:, None] * (r - t).astype(f32)).astype(f32)).astype(f32)
            dd = _fma32(c1[j], dd, g)
            y = (y + dd).astype(f32)
        return y, d(r, y)

    bb = d(b, b)
    x = np.zeros_like(b)
    r = b.copy()
    active = bb > 0
    it = restarts = checks = 0
    rep = bb.copy()                    # the rr the kernel holds per column (S->rr): what info[2..5] reports
    if x0 is not None:
        xw = np.asarray(x0, dtype=f32).copy()
        rw = (b.astype(np.float64) - A64 @ xw.astype(np.float64)).astype(f32)
        rrw = d(rw, rw)
        if not (rrw > bb).any():
            x, r = xw, rw
            active = ~(rrw <= (rtol * rtol) * bb)
            rep = rrw
    while True:
        z, gam = prec(r)
        p = np.zeros_like(b)
        s = np.zeros_like(b)
        alpha = np.zeros(b.shape[1], dtype=f32)
        beta = np.zeros(b.shape[1], dtype=f32)
        while active.any() and it < maxit:
            w = (A @ z).astype(f32)                                   # phase A
            x = (x + alpha[None, :] * p).astype(f32)
            p = (z + beta[None, :] * p).astype(f32)
            s = (w + beta[None, :] * s).astype(f32)
            dl = d(p, s)
            alpha = np.where(active & (dl > 0), gam / np.where(dl == 0, 1, dl), 0.0).astype(f32)
            r = (r - alpha[None, :] * s).astype(f32)                   # phase B
            z, gam_new = prec(r)
            rr = d(r, r)
            it += 1
            conv = rr <= (rtol * rtol) * bb
            beta = np.where(active & ~conv, gam_new / np.where(gam == 0, 1, gam), 0.0).astype(f32)
            gam = gam_new
            rep = np.where(active, rr, rep)
            active = active & ~conv
        x = (x + alpha[None, :] * p).astype(f32)                      # pending update
        if refine <= 0 or checks > refine or it == 0 or active.any():   # (active: stopped at maxit, no check)
            break
        rt = b.astype(np.float64) - A64 @ x.astype(np.float64)
        floor = Aabs @ np.abs(x.astype(np.float64))
        rrt, fl2 = d(rt, rt), d(floor, floor)
        checks += 1
        need = (rrt > (rtol * rtol) * bb) & (rrt > (theta * 2.0 ** -24) ** 2 * fl2) & (bb > 0) & (restarts < refine)
        rep = d(rt.astype(f32), rt.astype(f32))
        if record is not None:
            record.setdefault("checks", []).append(dict(it=it, rr=rrt, tol=(rtol * rtol) * bb,
                                                        floor=(theta * 2.0 ** -24) ** 2 * fl2, need=need))
        if not need.any():
            break
        restarts += 1
        r = rt.astype(f32)
        active = need
    if record is not None:
        record.setdefault("checks", [])
        record["status"] = 2 if active.any() else 1
        record["relres"] = np.where(bb > 0, np.sqrt(rep / np.where(bb > 0, bb, 1)), 0.0)
    return x, it, restarts
