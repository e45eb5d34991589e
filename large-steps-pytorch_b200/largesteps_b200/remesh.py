"""Re-parameterisation after a remesh (SURVEY 8 f4): scripts/main.py:137-169 on the GPU.

When the remesher has changed the connectivity the reference rebuilds everything from scratch:
    M = compute_matrix(v_unique, f_unique, lambda_, alpha)      two device sorts + sparse adds        (main.py:161)
    u_unique = to_differential(M, v_unique)                                                            (main.py:162)
    ... and the next from_differential re-factorises M with CHOLMOD on the CPU (seconds at 1M vertices, solvers.py:33-34).
Here assembly, solver set-up and the first solve are a few milliseconds of device work; what is left is allocator traffic
(~1 GB of fresh buffers per re-parameterisation at V = 1e6).  `Reparameterizer` keeps ONE arena across remeshes: the matrix,
its CSR/SELL copies and the solver workspace of the new mesh overwrite those of the old one -- no cudaMalloc, no free.

    rp = Reparameterizer(lambda_=19.0)            # or alpha=..., cotan=...
    M, u = rp.update(v_unique, f_unique)          # after every remesh; from_differential(M, u) is then a pure solve

The matrix of the previous update() becomes invalid (its storage is reused), exactly like the reference drops its old M.
"""
import torch

from . import _native as N
from . import geometry
from .parameterize import cache_put, to_differential, _cache
from .solvers import CholeskySolver, ConjugateGradientSolver, PCGSolver, workspace_bytes


class Arena:
    """Bump allocator over one device buffer, reset at every re-parameterisation."""

    def __init__(self, headroom=1.3):
        self.buf = None
        self.off = 0
        self.headroom = float(headroom)

    def reserve(self, nbytes, dev):
        if self.buf is None or self.buf.numel() < nbytes or self.buf.device != dev:
            self.buf = None                                   # release the old arena before asking for a larger one
            self.buf = torch.empty(int(nbytes * self.headroom) + 4096, dtype=torch.uint8, device=dev)
        self.off = (-self.buf.data_ptr()) % 256

    def take(self, nbytes, dev):
        nbytes = max(int(nbytes), 1)
        if self.buf is None or self.off + nbytes > self.buf.numel():
            raise MemoryError("arena exhausted: Reparameterizer.update() reserves an upper bound, this should not happen")
        out = self.buf[self.off: self.off + nbytes]
        self.off = (self.off + nbytes + 255) // 256 * 256
        return out


def _upper_bound_bytes(V, F, method_k=4):
    import ctypes
    nnz_max = V + 6 * F                                        # nnz(M) = V + 2E and E <= 3F
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_assemble_workspace_bytes(F, V, ctypes.byref(nb)), "ls_assemble_workspace_bytes")
    total = nb.value
    total += 16 * nnz_max + 2 * 4 * (nnz_max + 8) + 4 * (V + 9)          # COO indices, values, CSR columns, row pointers
    N.check(N.lib().ls_order_workspace_bytes(V, ctypes.byref(nb)), "ls_order_workspace_bytes")
    total += nb.value + 4 * (V + 8)
    total += workspace_bytes(V, nnz_max)
    return total + 16 * 256


class Reparameterizer:
    def __init__(self, lambda_=19.0, alpha=None, cotan=False, method="Cholesky", headroom=1.3):
        if method not in ("Cholesky", "CG", "PCG"):
            raise ValueError(f"Unknown solver type '{method}'.")
        self.lambda_, self.alpha, self.cotan, self.method = lambda_, alpha, cotan, method
        self.arena = Arena(headroom)
        self.M = None
        self.solver = None

    def update(self, verts, faces):
        """Assemble M for the new connectivity, build its solver, prime the from_differential cache, return (M, u = M v)."""
        N.require_cuda(verts, "verts")
        V, F = int(verts.shape[0]), int(faces.shape[0])
        # the previous solver handle points into the arena: destroy it before its memory is overwritten
        if self.M is not None:
            _cache.pop((id(self.M), self.method), None)
        self.solver = None
        self.M = None
        self.arena.reserve(_upper_bound_bytes(V, F), verts.device)
        # graph-free, as the reference's remesh block runs under torch.no_grad() (scripts/main.py)
        M = geometry.compute_matrix(verts.detach(), faces, self.lambda_, alpha=self.alpha, cotan=self.cotan, alloc=self.arena)
        ws = self.arena.take(workspace_bytes(V, M._nnz()), verts.device)
        cls = {"Cholesky": CholeskySolver, "CG": ConjugateGradientSolver, "PCG": PCGSolver}[self.method]
        solver = cls(M, workspace=ws)
        cache_put((id(M), self.method), solver, M)
        self.M, self.solver = M, solver
        return M, to_differential(M, verts)
