"""The cases that force the fused solver's true-residual restart, chosen with the numpy model (oracle.fused_pcg_f32), and
what the model says about them.  tests/test_restart_cases.py pins the choice on the CPU (with the CPU-assembled matrix);
tests/test_gpu_pcg_restart.py runs the same cases on the device (with the device-assembled matrix).

A case restarts when the true residual at convergence sits above both rtol ||b|| and the floor theta 2^-24 || |A||x| ||.
On the stiff variant of a mesh (lambda = 1, alpha = 0.999) the floor is the larger threshold, and the true residual at the
first check sits 1-5x above 2^-24 || |A||x| || (theta = 1): 4x and more only with Jacobi on the 10^4-row plane (3.9-4.5x),
2-2.6x with Jacobi on the 2.6 10^3-row meshes, 2.3-2.5x with Chebyshev, and 1.5-2x on meshes of 642 rows (icosphere 3).
At theta = 3, refine = 1 (the default) the first check of the 10^4-row plane lies within 1.3-1.5x of its threshold, and
with refine = 3 the check after a restart lies within 1-2x of it in every case the model can afford.  So every case runs
with refine = 1, theta = 1: the one decision the thresholds make (the first check) restarts with at least the case's margin,
and the second check is decided by the spent budget alone.  The margin each case is held to is the largest round number its
decisions clear: 3.5x for Jacobi on the 10^4-row plane (jacobi-zh: 3.96, 4.47, 4.04), 4x for K = 4 there, 2x elsewhere.
The instantiations that only meshes of at most ~640 rows reach (RES 3, and RES 4 with 256 threads) have no case: there the
first check sits 1.5-2x above its threshold, which a device-against-model comparison cannot pin."""
import numpy as np

import oracle
from largesteps_b200 import workloads

STIFF = dict(lambda_=1.0, alpha=0.999)
REFINE, THETA = 1, 1.0
MARGIN = 2.0              # the smallest margin of any case: ||r|| / threshold >= MARGIN or <= 1 / MARGIN (in norm)


# name -> (verts, faces, compute_matrix keywords)
MESHES = {
    "shuffled-stiff": lambda: (*workloads.shuffle_vertices(*workloads.plane(100, seed=3)), STIFF),   # 10^4 rows, Morton copy
    "ico4cot": lambda: (*workloads.icosphere(4), dict(lambda_=10.0, cotan=True)),                     # general copy
    "isolated-stiff": lambda: (*_with_isolated(*workloads.icosphere(4)), STIFF),                     # 2632 rows: RES 4
    "ico4-stiff": lambda: (*workloads.icosphere(4), STIFF),                                           # 2562 rows: RES 4
}

# forced-restart cases: name -> (mesh, k, bf16 rows, preconditioner of the model, margin of the first check)
CASES = {
    "jacobi-zh": ("shuffled-stiff", 3, True, "jacobi", 3.5),
    "jacobi-fp32-k4": ("shuffled-stiff", 4, False, "jacobi", 4.0),
    "chebyshev": ("shuffled-stiff", 3, False, "chebyshev", 2.0),
    "small-jacobi-zh": ("isolated-stiff", 3, True, "jacobi", 2.0),
    "small-jacobi-fp32-k4": ("ico4-stiff", 4, False, "jacobi", 2.0),
}


def _with_isolated(v, f, n=70):
    """test_gpu_pattern_share.with_isolated: rows with only a diagonal"""
    extra = np.random.default_rng(0).normal(size=(n, 3)).astype(v.dtype) + 5.0
    return np.concatenate([v, extra]), f
# batch: (mesh, k, bf16 rows, preconditioner, theta, restarts) per mesh; the mesh that must not restart passes its check on
# the floor of theta = 8 (a handle's theta is its own)
BATCH_CASES = [("shuffled-stiff", 3, True, "jacobi", THETA, 1), ("ico4cot", 3, True, "jacobi", 8.0, 0),
               ("shuffled-stiff", 3, False, "chebyshev", THETA, 1), ("ico4cot", 3, False, "chebyshev", 8.0, 0)]


def rhs(V, k, seed=0):
    return np.random.default_rng(seed).normal(size=(V, k)).astype(np.float32)


def warm_split(r, c, val, V, k, seed=0):
    """(b, x0) of the per-column case: column 0 random (it restarts), column 1 the 97th column of A with the exact solution
    e_97 as its guess (its residual is exactly 0: converged on entry, and its check passes whatever the thresholds),
    column 2 all zero"""
    b = rhs(V, k, seed)
    b[:, 1] = 0.0
    sel = c == 97
    b[r[sel], 1] = val[sel]
    b[:, 2] = 0.0
    x0 = np.zeros_like(b)
    x0[97, 1] = 1.0
    return b, x0


_models = {}


def model(r, c, val, V, b, key, **kw):
    """oracle.fused_pcg_f32 with its record, cached on the case key and every argument: (x, iterations, restarts, record)"""
    arr = lambda a: (a.shape, hash(np.ascontiguousarray(a).tobytes()))
    full = (key, V, arr(b), arr(val), tuple(sorted((k_, v_ if np.isscalar(v_) or v_ is None else arr(v_)) for k_, v_ in kw.items())))
    if full not in _models:
        rec = {}
        x, it, rs = oracle.fused_pcg_f32(r, c, val, V, b, record=rec, **kw)
        _models[full] = (x, it, rs, rec)
    return _models[full]


def margins(rec, refine):
    """per threshold decision (a check with restart budget left, b != 0): ||r|| / max(rtol ||b||, theta 2^-24 || |A||x| ||)"""
    out = []
    for i, ch in enumerate(rec["checks"]):
        if i >= refine:
            continue
        thr = np.maximum(ch["tol"], ch["floor"])
        for j in range(len(thr)):
            if ch["tol"][j] > 0:
                out.append(float(np.sqrt(ch["rr"][j] / thr[j])))
    return out
