"""Solver plug-ins -- same surface as the reference's largesteps/solvers.py.

    Solver                    interface: __init__(M), solve(b, backward=False)               (solvers.py:6-24)
    PCGSolver                 the GPU solver: fused Jacobi-PCG over all RHS columns (csrc/ls_pcg.cu)
    CholeskySolver            drop-in for solvers.py:26-39 (cholespy/CHOLMOD): PCGSolver, cold start, rtol 1e-7
    ConjugateGradientSolver   drop-in for solvers.py:41-126: PCGSolver with the reference's fwd/bwd warm starts
    DifferentiableSolve/solve autograd glue, identical contract to solvers.py:128-148

The reference's default path factorises M on the CPU with CHOLMOD and runs sparse triangular solves; this package
has no factorisation.  `CholeskySolver` keeps the *name and contract* ("x = M^-1 b, b (V,k) float32 contiguous on
M's device") and meets it to <= 1e-5 rel-L2 of a direct solve with a tight relative residual target.
"""
import ctypes
import warnings

import numpy as np

import torch
from torch.autograd import Function

from . import _native as N
from .geometry import csr_of, order_of

K_MAX = 4   # columns per pass of the native solver (wider right-hand sides are processed in chunks)
PRECOND = {"none": 0, "jacobi": 1, "chebyshev": 2, "auto": 3}   # ls_pcg_create's precond


class Solver:
    """Sparse linear system solver base class (solvers.py:6-24)."""

    def __init__(self, M):
        pass

    def solve(self, b, backward=False):
        """Solve the linear system M x = b.  `backward` tells whether this is the backward or forward solve."""
        raise NotImplementedError()


class PCGSolver(Solver):
    """Jacobi-preconditioned CG on the GPU, all columns of b in one pass.

    Parameters
    ----------
    M : torch.sparse_coo_tensor   system matrix (compute_matrix output, or any coalesced SPD float32 COO on CUDA)
    rtol : float     stop when ||r_j|| <= rtol ||b_j|| for every column j
    maxit : int      iteration cap (the reference CG has none and can spin forever, solvers.py:73)
    precond : {'jacobi', 'none', 'chebyshev', 'auto'}   'auto': chebyshev where it is measured faster (mid-size meshes), else jacobi.
                     'chebyshev': degree-3 Chebyshev polynomial in D^-1 M on top of Jacobi (C ABI precond = 2):
                     ~3x fewer CG iterations and all-reduces, ~1.3x more SpMVs (each with one grid barrier, no reduction)
    warm_start : bool   keep the previous solution as the next initial guess, separately for forward and backward
                        solves, as the reference CG does (solvers.py:102-110,120-124)
    strict : bool    raise NotConverged if maxit is reached (otherwise warn and return the last iterate)
    reorder : bool   let the solver re-order its private matrix copy along the Morton curve recorded by
                     compute_matrix (pure data-layout change: b and x stay in the caller's vertex numbering)
    check : bool     True: every solve synchronises, raises Breakdown / NotConverged (or warns).  False: the solve is
                     fully asynchronous on the current stream (one kernel launch, no host round trip); status and
                     iteration count are read lazily (`.iterations`, `.status`, `.raise_for_status()`), and a solve that
                     hit `maxit` or broke down is reported by a RuntimeWarning at the next call (never blocking).
    refine : int     accuracy guard (ls_pcg_set_refinement): after convergence the true residual b - M x is evaluated
                     with fp64 accumulation and the iteration restarts from it, at most `refine` times, if it sits more
                     than `theta` times above the floor fp32 storage of x imposes.  0 switches the check off.
    """

    def __init__(self, M, rtol=1e-7, maxit=10000, precond="jacobi", warm_start=False, strict=False, reorder=True,
                 check=True, refine=1, theta=3.0, workspace=None):
        if precond not in PRECOND:
            raise ValueError(f"Unknown preconditioner '{precond}'.")
        rowptr, col, val = csr_of(M)
        order = order_of(M) if reorder else None
        self.device = val.device
        self.V = int(M.shape[0])
        self.nnz = int(val.shape[0])
        self.rtol = float(rtol)
        self.maxit = int(maxit)
        self.warm_start = bool(warm_start)
        self.strict = bool(strict)
        self.check = bool(check)
        self.guess_fwd = None
        self.guess_bwd = None
        self._info_host = (ctypes.c_float * 8)()
        self._info_dev = None        # info of the last asynchronous solve: pinned host memory the kernel writes into
        self._info_event = None
        self._info_stale = False
        self._unreported = False     # an asynchronous solve whose status nobody has looked at yet
        self._handle = ctypes.c_void_p(0)
        lib = N.lib()
        with torch.cuda.device(self.device):
            nbytes = ctypes.c_size_t(0)
            N.check(lib.ls_pcg_workspace_bytes(self.V, self.nnz, K_MAX, ctypes.byref(nbytes)), "ls_pcg_workspace_bytes")
            if workspace is None:
                self._ws = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)   # owned by this object
            else:   # caller-provided device memory (largesteps_b200.remesh re-uses one arena across re-parameterisations)
                if workspace.numel() < nbytes.value or workspace.data_ptr() % 256 != 0 or workspace.device != self.device:
                    raise ValueError(f"workspace must be a 256-byte aligned uint8 tensor of >= {nbytes.value} bytes on {self.device}")
                self._ws = workspace
            N.check(lib.ls_pcg_create(ctypes.byref(self._handle), self.V, self.nnz, N.ptr(rowptr), N.ptr(col),
                                      N.ptr(val), N.ptr(order), PRECOND[precond], K_MAX, N.ptr(self._ws),
                                      nbytes.value, N.stream_ptr(self.device)), "ls_pcg_create")
            N.check(lib.ls_pcg_set_refinement(self._handle, int(refine), float(theta)), "ls_pcg_set_refinement")

    def __del__(self):
        h = getattr(self, "_handle", None)
        if h is not None and h.value:
            try:
                N.lib().ls_pcg_destroy(h)
            except Exception:
                pass
            self._handle = ctypes.c_void_p(0)

    # -- stats of the last solve ------------------------------------------------------------------------
    def _sync_info(self, block=True):
        """Fetch [iterations, status, relres..., restarts] of the last asynchronous solve.  block=False: only if the
        solve has already finished (returns False otherwise)."""
        if self._info_stale:
            if block:
                self._info_event.synchronize()
            elif not self._info_event.query():
                return False
            for j in range(8):
                self._info_host[j] = float(self._info_dev[j])
            self._info_stale = False
        return True

    def _report_previous(self):
        # the reference's direct solve cannot fail to converge; this iterative one can (maxit, breakdown on a non-SPD
        # matrix): say so at the next call instead of staying silent, without ever blocking the stream
        if self._unreported and self._sync_info(block=False):
            self._unreported = False
            st = int(self._info_host[1])
            if st == 2:
                warnings.warn(f"{type(self).__name__}: the previous solve stopped at maxit={self.maxit} "
                              f"(relres {[float(self._info_host[2 + j]) for j in range(3)]})", RuntimeWarning)
            elif st == 3:
                warnings.warn(f"{type(self).__name__}: the previous solve broke down after {int(self._info_host[0])} iterations "
                              "(matrix not SPD, or NaN in the right-hand side)", RuntimeWarning)

    @property
    def iterations(self):
        self._sync_info()
        return int(self._info_host[0])

    @property
    def relres(self):
        self._sync_info()
        return [float(self._info_host[2 + j]) for j in range(4)]

    @property
    def status(self):
        """0/1 converged, 2 iteration cap reached, 3 breakdown (not SPD / NaN) -- of the last solve."""
        self._sync_info()
        self._unreported = False
        return int(self._info_host[1])

    @property
    def restarts(self):
        """restarts from the true residual the last solve needed (see `refine`)."""
        self._sync_info()
        return int(self._info_host[6])

    def raise_for_status(self):
        st = self.status
        if st == 3:
            raise N.Breakdown(f"CG breakdown after {self.iterations} iterations (matrix not SPD or NaN in the right-hand side)")
        if st == 2:
            raise N.NotConverged(f"PCG did not reach rtol={self.rtol} within maxit={self.maxit} (relres {self.relres})")

    def describe(self):
        out = (ctypes.c_int64 * 8)()
        N.check(N.lib().ls_pcg_describe(self._handle, out), "ls_pcg_describe")
        o = [int(v) for v in out]
        pat = self.pattern_copy()
        # pattern-only copy: slices stored (identical ones share a copy) and the bytes of its column words
        pat = {"pattern_slices": pat["slices"], "pattern_slices_stored": pat["stored"], "pattern_column_bytes": 4 * pat["words"]}
        if o[4] >= 10:    # fused two-synchronisation solver (csrc/ls_pcg_fused.cuh)
            return {"algo": "fused", "sell_engine": o[0], "sell_entries": o[1], "grid": o[2], "cluster": o[3],
                    "residency": o[4] - 10, "precond": {0: "none", 1: "jacobi", 2: "chebyshev"}.get(o[5], o[5]), "threads": o[6],
                    "reordered": o[7],
                    "persistent": 2 if o[4] - 10 >= 1 else 1, "persistent_grid": o[2], **pat}
        # graph-mode solver (csrc/ls_pcg.cu): three kernels per iteration; "persistent" and "persistent_grid" are 0
        keys = ("sell_engine", "sell_entries", "spmm_grid", "vec_grid", "persistent", "persistent_grid", "planned", "reordered")
        d = dict(zip(keys, o))
        d["algo"] = "graph"
        d.update(pat)
        return d

    def pattern_copy(self, arrays=False):
        """The pattern-only matrix copy (csrc/ls_sell_kernel.cuh): {"on", "slices", "stored", "words"} and, with arrays=True
        and the copy on, "poff" (slices + 1 offsets: bit 0 wide, bits 1-4 pairs per row) and "words_array" (uint32)."""
        info = (ctypes.c_int64 * 4)()
        N.check(N.lib().ls_pcg_pattern_copy(self._handle, info, None, None, None), "ls_pcg_pattern_copy")
        d = dict(zip(("on", "slices", "stored", "words"), [int(v) for v in info]))
        if arrays and d["on"]:
            poff = np.zeros(d["slices"] + 1, np.int32)
            words = np.zeros(max(d["words"], 1), np.uint32)
            with torch.cuda.device(self.device):
                N.check(N.lib().ls_pcg_pattern_copy(self._handle, info, poff.ctypes.data_as(ctypes.POINTER(ctypes.c_int32)),
                                                    words.ctypes.data_as(ctypes.POINTER(ctypes.c_uint32)), N.stream_ptr(self.device)),
                        "ls_pcg_pattern_copy")
            d["poff"], d["words_array"] = poff, words[:d["words"]]
        return d

    def phase_cycles(self, per_cta=False):
        g = self.describe()["persistent_grid"] if per_cta else 0
        n = 8 + 8 * g
        out = (ctypes.c_int64 * n)()
        with torch.cuda.device(self.device):
            N.check(N.lib().ls_pcg_phase_cycles(self._handle, out, n, N.stream_ptr(self.device)), "ls_pcg_phase_cycles")
        keys = ("phaseA", "sync_ps", "phaseB", "sync_rz", "restart", "_0", "_", "iterations")
        d = dict(zip(keys, [int(v) for v in out[:8]]))
        if per_cta:
            d["per_cta"] = [[int(out[8 + 8 * c + j]) for j in range(8)] for c in range(g)]
        return d

    def spmm_bytes(self, k=3):
        return int(N.lib().ls_pcg_spmm_bytes(self._handle, k))

    def bench_spmm(self, k=3, launches=1):
        with torch.cuda.device(self.device):
            N.check(N.lib().ls_pcg_bench_spmm(self._handle, k, launches, N.stream_ptr(self.device)), "ls_pcg_bench_spmm")

    def spmv_put(self, x):
        """Set the stand-alone SpMM's input (ls_pcg_spmv_put) to x, (V, k) float32 on the device, k <= 4; the outputs read
        NaN until a launch (bench_spmm, bench_kernels) writes them."""
        N.require_cuda(x, "x")
        if x.dim() != 2 or x.shape[0] != self.V or x.dtype != torch.float32:
            raise ValueError(f"x must be ({self.V}, k) float32, got {tuple(x.shape)} {x.dtype}")
        x = x.contiguous()
        with torch.cuda.device(self.device):
            N.check(N.lib().ls_pcg_spmv_put(self._handle, x.shape[1], N.ptr(x), N.stream_ptr(self.device)), "ls_pcg_spmv_put")

    def spmv_get(self, k):
        """The stand-alone SpMM's output (ls_pcg_spmv_get): (y (V, k) float32, the p.Ap epilogue's k float64 dot products)."""
        y = torch.empty(self.V, k, dtype=torch.float32, device=self.device)
        dot = torch.empty(k, dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            N.check(N.lib().ls_pcg_spmv_get(self._handle, k, N.ptr(y), N.ptr(dot), N.stream_ptr(self.device)), "ls_pcg_spmv_get")
        return y, dot

    # -- the plug-in entry point --------------------------------------------------------------------------
    def solve(self, b, backward=False):
        if b.dim() != 2:
            raise ValueError(f"Invalid array shape {b.shape} for {type(self).__name__}.solve: expected shape (a, b)")
        N.require_cuda(b, "b")
        if b.device != self.device:
            raise RuntimeError(f"b is on {b.device} but the system matrix is on {self.device}")
        if b.dtype != torch.float32:
            raise TypeError(f"b must be float32, got {b.dtype}")
        if b.shape[0] != self.V:
            raise ValueError(f"b has {b.shape[0]} rows, the system matrix has {self.V}")
        self._report_previous()
        b = b.detach().contiguous()
        k = b.shape[1]
        x0 = None
        if self.warm_start:
            x0 = self.guess_bwd if backward else self.guess_fwd
            if x0 is not None and x0.shape != b.shape:
                x0 = None
        x = torch.empty_like(b)
        lib = N.lib()
        with torch.cuda.device(self.device):
            st = N.stream_ptr(self.device)
            for k0 in range(0, k, K_MAX):
                kk = min(K_MAX, k - k0)
                if k <= K_MAX:
                    bb, xx, gg = b, x, x0
                else:   # wide RHS: contiguous column chunks
                    bb = b[:, k0:k0 + kk].contiguous()
                    xx = torch.empty_like(bb)
                    gg = x0[:, k0:k0 + kk].contiguous() if x0 is not None else None
                if self.check:
                    rc = lib.ls_pcg_solve(self._handle, N.ptr(bb), N.ptr(xx), N.ptr(gg), kk, self.rtol, self.maxit,
                                          None, self._info_host, st)
                    self._info_stale = False
                    if rc == N.LS_ERR_NOT_CONVERGED and not self.strict:
                        warnings.warn(f"{type(self).__name__}: {N.last_error()}", RuntimeWarning)
                    else:
                        N.check(rc, "ls_pcg_solve")
                else:
                    if self._info_dev is None:   # mapped pinned host memory: the kernel's last store lands here, no copy is queued
                        self._info_dev = torch.zeros(8, dtype=torch.float32).pin_memory()
                        self._info_event = torch.cuda.Event()
                    N.check(lib.ls_pcg_solve(self._handle, N.ptr(bb), N.ptr(xx), N.ptr(gg), kk, self.rtol, self.maxit,
                                             N.ptr(self._info_dev), None, st), "ls_pcg_solve")
                    self._info_event.record(torch.cuda.current_stream(self.device))
                    self._info_stale = True
                    self._unreported = True
                if k > K_MAX:
                    x[:, k0:k0 + kk] = xx
        if self.warm_start:
            if backward:
                self.guess_bwd = x
            else:
                self.guess_fwd = x
        return x


def bench_kernels(solvers, which, launches, k=3):
    """Launch the in-solver SpMM `launches` times back-to-back from C, rotating over `solvers` (timing harness).
    which: 0 SpMM+dot, 4 SpMM without the dot epilogue; any other value raises ValueError."""
    arr = (ctypes.c_void_p * len(solvers))(*[s._handle for s in solvers])
    dev = solvers[0].device
    with torch.cuda.device(dev):
        N.check(N.lib().ls_pcg_bench(arr, len(solvers), k, which, launches, N.stream_ptr(dev)), "ls_pcg_bench")


def workspace_bytes(V, nnz):
    """Device bytes a solver handle for a (V, V) matrix with nnz entries needs (ls_pcg_workspace_bytes)."""
    nbytes = ctypes.c_size_t(0)
    N.check(N.lib().ls_pcg_workspace_bytes(int(V), int(nnz), K_MAX, ctypes.byref(nbytes)), "ls_pcg_workspace_bytes")
    return nbytes.value


def plan(nslices, pattern, sm_count, max_smem, precond="jacobi", k=3, cooperative=True):
    """The fused solver's launch plan (ls_pcg_plan, host only) for a mesh of `nslices` slices of 32 rows, with the pattern-only
    matrix copy or not, on a device with `sm_count` SMs, `max_smem` bytes of shared memory per CTA and cooperative launch or not.
    The LS_PCG_* switches of the plan are read from the environment, as PCGSolver reads them.  Returns the keys of
    PCGSolver.describe() the plan decides: {"algo": "graph"}, or "algo", "grid", "cluster", "residency", "threads", "precond"."""
    if precond not in PRECOND:
        raise ValueError(f"Unknown preconditioner '{precond}'.")
    out = (ctypes.c_int64 * 8)()
    N.check(N.lib().ls_pcg_plan(int(nslices), int(k), 1 if pattern else 0, PRECOND[precond], int(sm_count), int(max_smem),
                                1 if cooperative else 0, out), "ls_pcg_plan")
    on, grid, cluster, res, threads, pc = (int(v) for v in out[:6])
    if not on:
        return {"algo": "graph"}
    return {"algo": "fused", "grid": grid, "cluster": cluster, "residency": res, "threads": threads,
            "precond": {0: "none", 1: "jacobi", 2: "chebyshev"}[pc]}


class CholeskySolver(PCGSolver):
    """Drop-in for the reference CholeskySolver (solvers.py:26-39).  No factorisation happens: the system is
    solved by the device PCG from a cold start to a relative residual of 1e-7 (<= 1e-5 rel-L2 of a direct solve).
    One asynchronous kernel launch per solve (`check=False`); `.raise_for_status()` checks the last solve on demand."""

    def __init__(self, M, workspace=None):
        # like cholespy's solve, the call is asynchronous; a solve that did not converge is reported at the next call
        super().__init__(M, rtol=1e-7, maxit=10000, precond="auto", warm_start=False, check=False, refine=1,
                         workspace=workspace)


class ConjugateGradientSolver(PCGSolver):
    """Drop-in for the reference ConjugateGradientSolver (solvers.py:41-126): keeps its separate forward/backward
    warm starts; uses a *relative* tolerance and an iteration cap instead of the reference's absolute 1e-5."""

    def __init__(self, M, workspace=None):
        super().__init__(M, rtol=1e-7, maxit=10000, precond="auto", warm_start=True, workspace=workspace)


class DifferentiableSolve(Function):
    """Differentiable function to solve the linear system (solvers.py:128-145).

    forward: x = solver.solve(b); backward: grad_b = solver.solve(grad_x, backward=True)  (M is symmetric).
    """

    @staticmethod
    def forward(ctx, solver, b):
        ctx.solver = solver
        return solver.solve(b, backward=False)

    @staticmethod
    def backward(ctx, grad_output):
        solver_grad = None   # one gradient per forward input
        b_grad = None
        if ctx.needs_input_grad[1]:
            b_grad = ctx.solver.solve(grad_output.contiguous(), backward=True)
        return (solver_grad, b_grad)


# Alias for DifferentiableSolve function (solvers.py:148)
solve = DifferentiableSolve.apply
