"""Builds and binds oracle/cg_port.c (TEST INFRASTRUCTURE / CPU BASELINE ONLY, see oracle/__init__.py).

`CPortCG` is the multi-threaded (OpenMP) C restatement of the reference's ConjugateGradientSolver
(solvers.py:41-126) with the reference's semantics: fp32, absolute tolerance 1e-5, per-axis solves, separate
forward/backward warm starts.  It exists so that the CPU baseline next to the GPU numbers can use every host core."""
import ctypes
import os
import subprocess

import numpy as np
import scipy.sparse as sp

_HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(_HERE, "cg_port.c")
OUT_DIR = os.path.join(_HERE, "_build")
LIB = os.path.join(OUT_DIR, "libcg_port.so")
_lib = None


def build(force=False):
    """gcc -O3 -fopenmp -shared -fPIC cg_port.c -> oracle/_build/libcg_port.so"""
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
        os.makedirs(OUT_DIR, exist_ok=True)
        # portable flags on purpose: the .so may be built on one machine and run on another (different CPU)
        subprocess.run(["gcc", "-O3", "-fopenmp", "-shared", "-fPIC", SRC, "-o", LIB, "-lm"], check=True)
    return LIB


def lib():
    global _lib
    if _lib is None:
        h = ctypes.CDLL(build())
        h.lsref_num_threads.restype = ctypes.c_int
        h.lsref_set_num_threads.argtypes = [ctypes.c_int]
        h.lsref_cg_solve.restype = ctypes.c_int
        h.lsref_cg_solve.argtypes = [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 6 + [ctypes.c_float, ctypes.c_int,
                                                                                            ctypes.c_void_p]
        h.lsref_sell_spmv_f32.restype = None
        h.lsref_sell_spmv_f32.argtypes = [ctypes.c_int64, ctypes.c_int] + [ctypes.c_void_p] * 5
        _lib = h
    return _lib


def sell32(rowptr, col=None):
    """Padded width of every row in the solver's SELL-32 copy: the longest row of its slice of 32 rows (int64, (V,)).
    `col` is not needed (the widths depend on the row lengths only); it is accepted so that callers can pass a CSR as is."""
    lens = np.diff(np.asarray(rowptr, dtype=np.int64))
    V = lens.shape[0]
    pad = np.zeros(-V % 32, np.int64)
    w = np.concatenate([lens, pad]).reshape(-1, 32).max(axis=1)
    return np.repeat(w, 32)[:V]


def sell_spmv_f32(rowptr, col, val, x):
    """y = A x with the SELL-32 kernels' exact arithmetic (lsref_sell_spmv_f32): x (V, K) float32, K >= 1; y (V, K) float32."""
    rowptr = np.ascontiguousarray(rowptr, dtype=np.int32)
    col = np.ascontiguousarray(col, dtype=np.int32)
    val = np.ascontiguousarray(val, dtype=np.float32)
    x = np.ascontiguousarray(x, dtype=np.float32)
    V, K = x.shape
    assert rowptr.shape[0] == V + 1 and col.shape[0] >= rowptr[-1] and val.shape[0] >= rowptr[-1]
    y = np.empty((V, K), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    lib().lsref_sell_spmv_f32(V, K, p(rowptr), p(col), p(val), p(x), p(y))
    return y


def host_cpu_budget():
    """What this process may actually use: CPUs in its affinity mask and the cgroup CPU quota (cores), if any."""
    try:
        ncpu = len(os.sched_getaffinity(0))
    except AttributeError:
        ncpu = os.cpu_count() or 1
    quota = None
    raw = None
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            raw = open(path).read().strip()
        except OSError:
            continue
        try:
            if path.endswith("cpu.max"):
                a, b = raw.split()
                quota = None if a == "max" else float(a) / float(b)
            else:
                qv = float(raw)
                per = float(open("/sys/fs/cgroup/cpu/cpu.cfs_period_us").read())
                quota = None if qv <= 0 else qv / per
        except Exception:
            quota = None
        break
    return {"affinity_cpus": ncpu, "quota_cores": quota, "cgroup_cpu_max": raw}


def pin_to_allowed_cores(n):
    """Restrict this process to the first n CPUs of its affinity mask (OpenMP threads inherit it): keeps the team on a fixed
    set of cores instead of migrating across a large shared host."""
    try:
        cpus = sorted(os.sched_getaffinity(0))
        os.sched_setaffinity(0, set(cpus[:max(1, n)]))
        return cpus[:max(1, n)]
    except (AttributeError, OSError):
        return None


class CPortCG:
    """Same interface as oracle.ReferenceCG / the reference's ConjugateGradientSolver."""

    def __init__(self, rows, cols, vals, V):
        A = sp.csr_matrix((np.asarray(vals, dtype=np.float32), (np.asarray(rows), np.asarray(cols))), shape=(V, V))
        A.sort_indices()
        self.V = V
        self.rowptr = np.ascontiguousarray(A.indptr, dtype=np.int32)
        self.col = np.ascontiguousarray(A.indices, dtype=np.int32)
        self.val = np.ascontiguousarray(A.data, dtype=np.float32)
        self.guess_fwd = None
        self.guess_bwd = None
        self.iters = []
        self.threads = lib().lsref_num_threads()

    def autotune_threads(self, b, probe_iters=8):
        """Pick the OpenMP thread count.  The boxes run under a cgroup CPU quota (see host_cpu_budget): the default of one
        thread per logical CPU can be 500x slower than one thread per allowed core.  Candidates are therefore centred on the
        quota (quota/2, quota, 2 quota, capped by the affinity mask) and the fastest over a few CG iterations wins."""
        import time
        budget = host_cpu_budget()
        ncpu = budget["affinity_cpus"]
        q = budget["quota_cores"]
        if q:
            cands = sorted({max(1, min(ncpu, int(round(c)))) for c in (q / 2, q, 2 * q)})
        else:   # no visible quota (it may still exist one level up): scan powers of two
            cands = [t for t in (4, 8, 16, 32, 64, 128, 256) if t <= ncpu] or [ncpu]
        save = (self.guess_fwd, self.guess_bwd)
        best_t, best_dt = cands[0], float("inf")
        for t in cands:
            lib().lsref_set_num_threads(t)
            self.guess_fwd = None
            self.solve(b, maxit=1)                     # thread pool start-up at this size
            dt = float("inf")
            for _ in range(3):                         # best of three: shared hosts are noisy
                self.guess_fwd = None
                t0 = time.perf_counter()
                self.solve(b, maxit=probe_iters)
                dt = min(dt, time.perf_counter() - t0)
            if dt < best_dt:
                best_t, best_dt = t, dt
        lib().lsref_set_num_threads(best_t)
        self.threads = best_t
        self.guess_fwd, self.guess_bwd = save
        self.iters = []
        return best_t

    def solve(self, b, backward=False, tol=1e-5, maxit=100000):
        b = np.ascontiguousarray(b, dtype=np.float32)
        if b.ndim != 2:                                         # solvers.py:112-113
            raise ValueError(f"Invalid array shape {b.shape} for ConjugateGradientSolver.solve: expected shape (a, b)")
        if self.guess_fwd is None:                              # solvers.py:102-105
            self.guess_bwd = np.zeros_like(b)
            self.guess_fwd = np.zeros_like(b)
        x0 = np.ascontiguousarray(self.guess_bwd if backward else self.guess_fwd)
        x = np.empty_like(b)
        k = b.shape[1]
        iters = (ctypes.c_int * k)()
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        rc = lib().lsref_cg_solve(self.V, k, p(self.rowptr), p(self.col), p(self.val), p(b), p(x0), p(x),
                                  tol, maxit, iters)
        if rc != 0:
            raise MemoryError("cg_port: out of memory")
        self.iters = list(iters)
        if backward:                                            # solvers.py:120-124
            self.guess_bwd = x
        else:
            self.guess_fwd = x
        return x
