"""Differential parameterization -- same surface as the reference's largesteps/parameterize.py.

    to_differential(L, v)                      u = M v            (parameterize.py:19-30)
    from_differential(L, u, method='Cholesky') v = M^-1 u         (parameterize.py:32-61), differentiable w.r.t. u

The solver cache keeps the reference's semantics (parameterize.py:5-17): keyed by (id(L), method), dropped by a
weakref callback when the matrix is garbage collected.
"""
import weakref

import torch

from . import _native as N
from .geometry import csr_of, is_symmetric_by_construction, values_with_graph
from .solvers import CholeskySolver, ConjugateGradientSolver, PCGSolver, solve

# Cache for the system solvers
_cache = {}


def cache_put(key, value, A):
    # Called when 'A' is garbage collected
    def cleanup_callback(wr):
        _cache.pop(key, None)

    wr = weakref.ref(A, cleanup_callback)
    _cache[key] = (value, wr)


class _SpMM(torch.autograd.Function):
    """y = M x through the library's CSR SpMM.  The gradient w.r.t. x is M^T g.  Every matrix this package builds (system
    matrices, both Laplacians) is symmetric, like the reference's (geometry.py:56,94), and gets M g.  Any other matrix gets
    the SpMM of its transpose, `M.t().coalesce()`, built at the first backward and kept for the next.

    The gradient w.r.t. M's values is the sampled product gval[e] = <g[row_e], x[col_e]> (ls_spmm_csr_grad_val_f32).  It goes
    to `vals`, M's values as the cotangent assembly built them (geometry.values_with_graph), when there is one, else as a
    sparse tensor on M's coalesced pattern to M itself."""

    @staticmethod
    def forward(ctx, L, vals, v):
        ctx.L = L
        ctx.Lt = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            ctx.save_for_backward(v)
        return spmm(L, v)

    @staticmethod
    def backward(ctx, g):
        L = ctx.L
        g = g.contiguous()
        gv = None
        if ctx.needs_input_grad[2]:    # d/dv (L v) = L^T g
            if is_symmetric_by_construction(L):
                gv = spmm(L, g)
            else:
                if ctx.Lt is None:     # held here: csr_of caches the transpose's CSR for as long as it lives
                    ctx.Lt = L.t().coalesce()
                gv = spmm(ctx.Lt, g)
        gL = gvals = None
        if ctx.needs_input_grad[1]:
            (v,) = ctx.saved_tensors
            gvals = spmm_grad_values(L, g, v)
        elif ctx.needs_input_grad[0]:
            (v,) = ctx.saved_tensors
            Lc = L if L.is_coalesced() else L.coalesce()
            gL = torch.sparse_coo_tensor(Lc.indices(), spmm_grad_values(L, g, v), L.shape, is_coalesced=True)
        return gL, gvals, gv


def spmm_grad_values(L, gy, x):
    """gval[e] = sum_k gy[row_e, k] x[col_e, k] over L's coalesced pattern (ls_spmm_csr_grad_val_f32): the gradient of
    (L @ x) w.r.t. L's values, in the order of L.coalesce().values().  gy, x: (V,k) or (V,) float32 CUDA."""
    _require_square(L)
    rowptr, col, val = csr_of(L)
    for t, name in ((gy, "gy"), (x, "x")):
        N.require_cuda(t, name)
        if t.device != val.device:
            raise RuntimeError(f"{name} is on {t.device} but the matrix is on {val.device}")
        if t.dtype != torch.float32:
            raise TypeError(f"{name} must be float32, got {t.dtype}")
    g2 = (gy.unsqueeze(1) if gy.dim() == 1 else gy).detach().contiguous()
    x2 = (x.unsqueeze(1) if x.dim() == 1 else x).detach().contiguous()
    if g2.dim() != 2 or g2.shape != x2.shape or x2.shape[0] != L.shape[1]:
        raise ValueError(f"shape mismatch: L is {tuple(L.shape)}, gy is {tuple(gy.shape)}, x is {tuple(x.shape)}")
    out = torch.empty(val.shape[0], dtype=torch.float32, device=val.device)
    if out.numel() == 0:   # no entries: torch gives empty tensors no storage, and the C entry point rejects NULL
        return out
    k = x2.shape[1]
    with torch.cuda.device(x2.device):
        N.check(N.lib().ls_spmm_csr_grad_val_f32(L.shape[0], N.ptr(rowptr), N.ptr(col), N.ptr(x2), k, N.ptr(g2), k, k,
                                                 N.ptr(out), N.stream_ptr(x2.device)), "ls_spmm_csr_grad_val_f32")
    return out


def spmm_autograd(L, v):
    """L @ v, differentiable w.r.t. v and w.r.t. L's values when either asks for it."""
    if v.requires_grad or L.requires_grad:
        return _SpMM.apply(L, values_with_graph(L), v)
    return spmm(L, v)


def _require_square(L):
    # the C entry points take one V for the rows of L, of x and of y
    if L.dim() != 2 or L.shape[0] != L.shape[1]:
        raise ValueError(f"L must be a square (V, V) matrix, got {tuple(L.shape)}")


def spmm(L, v):
    """Non-differentiable y = L @ v on the device (ls_spmm_csr_f32). L: (V,V); v: (V,k) or (V,) float32 CUDA."""
    _require_square(L)
    rowptr, col, val = csr_of(L)
    N.require_cuda(v, "v")
    if v.device != val.device:
        raise RuntimeError(f"v is on {v.device} but the matrix is on {val.device}")
    if v.dtype != torch.float32:
        raise TypeError(f"v must be float32, got {v.dtype}")
    squeeze = v.dim() == 1
    x = (v.unsqueeze(1) if squeeze else v).detach().contiguous()
    if x.dim() != 2 or x.shape[0] != L.shape[1]:
        raise ValueError(f"shape mismatch: L is {tuple(L.shape)}, v is {tuple(v.shape)}")
    if val.numel() == 0:   # no entries: torch gives empty tensors no storage, and the C entry point rejects NULL
        y = torch.zeros_like(x)
        return y.squeeze(1) if squeeze else y
    y = torch.empty_like(x)
    k = x.shape[1]
    with torch.cuda.device(x.device):
        N.check(N.lib().ls_spmm_csr_f32(L.shape[0], N.ptr(rowptr), N.ptr(col), N.ptr(val), N.ptr(x), k, N.ptr(y), k, k,
                                        N.stream_ptr(x.device)), "ls_spmm_csr_f32")
    return y.squeeze(1) if squeeze else y


def to_differential(L, v):
    """Convert vertex coordinates to the differential parameterization: u = L @ v (parameterize.py:30).

    L : torch.sparse.Tensor   (I + l*L) matrix;   v : torch.Tensor   vertex coordinates (V,3) float32 CUDA.
    Differentiable w.r.t. v, and w.r.t. L's values when L carries a graph (a cotangent matrix built from positions that
    require grad), as the reference's `L @ v` is.
    """
    return spmm_autograd(L, v)


def from_differential(L, u, method='Cholesky'):
    """Convert differential coordinates back to Cartesian: solve L v = u (parameterize.py:32-61).

    If this is the first time we call this function on a given matrix L, the solver is cached. It will be destroyed
    once the matrix is garbage collected.

    method : {'Cholesky', 'CG', 'PCG'}
        'Cholesky' and 'CG' are the reference's names and keep their contracts (cold-start direct-solve accuracy;
        warm-started CG).  'PCG' is the native solver with its defaults.  All three run csrc/ls_pcg.cu.
    """
    key = (id(L), method)
    if key not in _cache.keys():
        if method == 'Cholesky':
            solver = CholeskySolver(L)
        elif method == 'CG':
            solver = ConjugateGradientSolver(L)
        elif method == 'PCG':
            solver = PCGSolver(L)
        else:
            raise ValueError(f"Unknown solver type '{method}'.")
        cache_put(key, solver, L)
    else:
        solver = _cache[key][0]
    return solve(solver, u)
