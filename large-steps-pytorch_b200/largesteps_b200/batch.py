"""Batched solves: many meshes with different system matrices in one call (csrc/ls_pcg_batch.cu, ls_pcg_batch_*).

    BatchSolver(Ms)                            x_i = M_i^-1 b_i for every mesh i, one launch per plan group
    from_differential_batch(Ms, us, method)    [M_i^-1 u_i], differentiable w.r.t. every u_i (packed=True: one (sum V_i, 3))
    pack_meshes(verts_list, faces_list)        B meshes as one mesh + offsets, for the mesh ops of the rest of the step

One small or mid-size mesh does not fill the GPU: a mesh of <= 24 slices of 32 rows runs on one CTA, and the cooperative grid
of a mid-size mesh spends its iterations in grid all-reduces.  The batch solver runs one thread-block cluster (1..16 CTAs) per
mesh and many meshes per launch; the clusters never wait on each other, and each mesh stops on its own convergence.

Meshes that share ONE matrix are already a single solve with 3B columns (`from_differential(M, torch.cat(us, 1))`): this module
is for different matrices.  A mesh larger than one cluster of 16 CTAs (about 70K vertices) is rejected: solve it with
`from_differential`.

The preconditioner is chosen per mesh (`precond`): Jacobi (the default) or the degree-3 Chebyshev polynomial over Jacobi, as
PCGSolver's precond='chebyshev'.  A Chebyshev mesh needs about a third of the outer iterations (two cluster all-reduces each)
for about 1.3x the SpMVs; its steps synchronise its cluster with a bare barrier.
"""
import ctypes
import warnings
import weakref
from typing import NamedTuple

import torch
from torch.autograd import Function

from . import _native as N
from . import meshops
from .solvers import PCGSolver

K_BATCH = 3   # columns per batched solve
PRECONDS = ("jacobi", "chebyshev")


def preconditioners(precond, n):
    """'jacobi', 'chebyshev', or a list of one of those per mesh -> the list of n preconditioner names."""
    ps = [precond] * n if isinstance(precond, str) else list(precond)
    if len(ps) != n:
        raise ValueError(f"got {len(ps)} preconditioners for {n} meshes")
    for i, p in enumerate(ps):
        if not isinstance(p, str) or p not in PRECONDS:
            raise ValueError(f"Unknown preconditioner {p!r} for mesh {i}: the batched solve takes 'jacobi' or 'chebyshev'.")
    return ps


def plan(nslices, pattern, max_smem, cheb=None):
    """The batch plan (ls_pcg_batch_plan_ex, host only): per mesh (cluster size, residency level, plan group) and the number of
    groups, i.e. of launches per solve.  nslices: slices of 32 rows per mesh; pattern: pattern-only matrix copy per mesh;
    cheb (optional, None = all Jacobi): per mesh 1 for the Chebyshev preconditioner, 0 for Jacobi."""
    n = len(nslices)
    if n == 0:
        raise ValueError("the batch is empty")
    if cheb is not None and len(cheb) != n:
        raise ValueError(f"got {len(cheb)} cheb entries for {n} meshes")
    ns = (ctypes.c_int32 * n)(*[int(s) for s in nslices])
    pt = (ctypes.c_int32 * n)(*[1 if p else 0 for p in pattern])
    cs, rs, gr = (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)()
    ng = ctypes.c_int32(0)
    ch = None if cheb is None else (ctypes.c_int32 * n)(*[int(c) for c in cheb])
    N.check(N.lib().ls_pcg_batch_plan_ex(n, ns, pt, ch, int(max_smem), cs, rs, gr, ctypes.byref(ng)), "ls_pcg_batch_plan_ex")
    return [(int(cs[i]), int(rs[i]), int(gr[i])) for i in range(n)], int(ng.value)


class BatchSolver:
    """Preconditioned CG for a list of matrices, all meshes in one call.

    Parameters
    ----------
    Ms : list of torch.sparse_coo_tensor   system matrices (compute_matrix outputs) on one CUDA device
    rtol, maxit : as PCGSolver, per mesh
    warm_start : bool   keep the previous solution as the next initial guess, separately for forward and backward solves
    strict : bool       a mesh that reaches maxit raises NotConverged naming its index (the solve then synchronises)
    check : bool        True: every solve synchronises and warns about a mesh that reached maxit.  False: fully asynchronous;
                        `.iterations`, `.status`, `.relres` are read lazily.
    precond : 'jacobi' (default), 'chebyshev', or a list of one of those per mesh.  'chebyshev' is PCGSolver's degree-3
                        Chebyshev polynomial over Jacobi; it runs each mesh on a cluster with the iterate and direction in
                        shared memory (smaller caps per CTA, never the one-CTA RES 3 path).  `.iterations` counts outer iterations.
    """

    def __init__(self, Ms, rtol=1e-7, maxit=10000, warm_start=False, strict=False, check=False, precond="jacobi"):
        Ms = list(Ms)
        if len(Ms) == 0:
            raise ValueError("BatchSolver needs at least one matrix")
        self.precond = preconditioners(precond, len(Ms))
        # one handle per mesh (the single-mesh solver's own matrix copy, Morton order, diagonal classes, Chebyshev coefficients)
        self.solvers = [PCGSolver(M, rtol=rtol, maxit=maxit, precond=p, check=True) for M, p in zip(Ms, self.precond)]
        self.device = self.solvers[0].device
        for i, s in enumerate(self.solvers):
            if s.device != self.device:
                raise RuntimeError(f"matrix {i} is on {s.device}, matrix 0 on {self.device}: a batch runs on one device")
        self.n = len(Ms)
        self.sizes = [s.V for s in self.solvers]
        self.rows = sum(self.sizes)
        self.rtol = float(rtol)
        self.maxit = int(maxit)
        self.warm_start = bool(warm_start)
        self.strict = bool(strict)
        self.check = bool(check)
        self.guess_fwd = None
        self.guess_bwd = None
        self._info = torch.zeros(8 * self.n, dtype=torch.float32).pin_memory()   # the kernels write each mesh's record here
        self._info_event = None
        self._batch = ctypes.c_void_p(0)
        handles = (ctypes.c_void_p * self.n)(*[s._handle.value for s in self.solvers])
        with torch.cuda.device(self.device):
            N.check(N.lib().ls_pcg_batch_create(ctypes.byref(self._batch), handles, self.n, N.stream_ptr(self.device)),
                    "ls_pcg_batch_create")

    def __del__(self):
        b = getattr(self, "_batch", None)
        if b is not None and b.value:
            try:
                N.lib().ls_pcg_batch_destroy(b)
            except Exception:
                pass
            self._batch = ctypes.c_void_p(0)

    def plan(self):
        """[(cluster size, residency, group)] per mesh and the number of launches per solve."""
        smem = torch.cuda.get_device_properties(self.device).shared_memory_per_block_optin
        d = [s.describe() for s in self.solvers]
        return plan([(v + 31) // 32 for v in self.sizes], [e["sell_engine"] == 2 for e in d], smem,
                    cheb=[1 if e.get("precond") == "chebyshev" else 0 for e in d])

    # -- per-mesh stats of the last solve -----------------------------------------------------------------
    def _records(self):
        if self._info_event is not None:
            self._info_event.synchronize()
        return self._info.view(self.n, 8)

    @property
    def iterations(self):
        return [int(v) for v in self._records()[:, 0].tolist()]

    @property
    def status(self):
        """per mesh: 1 converged, 2 iteration cap reached, 3 breakdown (not SPD / NaN)."""
        return [int(v) for v in self._records()[:, 1].tolist()]

    @property
    def relres(self):
        return [[float(v) for v in r] for r in self._records()[:, 2:6].tolist()]

    @property
    def restarts(self):
        """per mesh: restarts from the true residual the last solve needed (see PCGSolver's `refine`)."""
        return [int(v) for v in self._records()[:, 6].tolist()]

    def raise_for_status(self):
        st = self.status
        for i, s in enumerate(st):
            if s == 3:
                raise N.Breakdown(f"mesh {i}: CG breakdown after {self.iterations[i]} iterations (matrix not SPD or NaN in the "
                                  "right-hand side)")
        for i, s in enumerate(st):
            if s == 2:
                raise N.NotConverged(f"mesh {i}: PCG did not reach rtol={self.rtol} within maxit={self.maxit} "
                                     f"(relres {self.relres[i][:3]})")

    # -- inputs ---------------------------------------------------------------------------------------------
    def validate(self, bs):
        """Checks a list of (V_i, k) tensors, or one packed (sum V_i, k) tensor, as PCGSolver.solve checks b."""
        packed = isinstance(bs, torch.Tensor)
        parts = [bs] if packed else list(bs)
        if not packed and len(parts) != self.n:
            raise ValueError(f"got {len(parts)} right-hand sides for {self.n} meshes")
        k = None
        for i, b in enumerate(parts):
            N.require_cuda(b, f"b[{i}]")
            if b.device != self.device:
                raise RuntimeError(f"b[{i}] is on {b.device} but the system matrices are on {self.device}")
            if b.dtype != torch.float32:
                raise TypeError(f"b[{i}] must be float32, got {b.dtype}")
            if b.dim() != 2:
                raise ValueError(f"b[{i}] has shape {tuple(b.shape)}: expected (V, k)")
            rows = self.rows if packed else self.sizes[i]
            if b.shape[0] != rows:
                raise ValueError(f"b[{i}] has {b.shape[0]} rows, expected {rows}")
            if k is None:
                k = b.shape[1]
            elif b.shape[1] != k:
                raise ValueError(f"b[{i}] has {b.shape[1]} columns, b[0] has {k}")
        if not 1 <= k <= K_BATCH:
            raise ValueError(f"the batched solve takes 1 to {K_BATCH} columns, got {k}")
        return parts

    def pack(self, bs):
        """A list of (V_i, k) tensors, or one packed (sum V_i, k) tensor -> the packed, contiguous (sum V_i, k) tensor."""
        parts = self.validate(bs)
        return (parts[0] if len(parts) == 1 else torch.cat(parts, 0)).detach().contiguous()

    def split(self, x):
        return list(torch.split(x, self.sizes, 0))

    # -- the solve --------------------------------------------------------------------------------------------
    def solve_packed(self, b, backward=False):
        """b: packed (sum V_i, k) float32, contiguous -> packed solution."""
        x0 = None
        if self.warm_start:
            x0 = self.guess_bwd if backward else self.guess_fwd
            if x0 is not None and x0.shape != b.shape:
                x0 = None
        x = torch.empty_like(b)
        lib = N.lib()
        sync = self.check or self.strict
        with torch.cuda.device(self.device):
            st = N.stream_ptr(self.device)
            host = (ctypes.c_float * (8 * self.n))() if sync else None
            rc = lib.ls_pcg_batch_solve(self._batch, N.ptr(b), N.ptr(x), N.ptr(x0), b.shape[1], self.rtol, self.maxit,
                                        N.ptr(self._info), host, st)
            if self._info_event is None:
                self._info_event = torch.cuda.Event()
            self._info_event.record(torch.cuda.current_stream(self.device))
            if rc == N.LS_ERR_NOT_CONVERGED and not self.strict:
                warnings.warn(f"BatchSolver: {N.last_error()}", RuntimeWarning)
            else:
                N.check(rc, "ls_pcg_batch_solve")
        if self.warm_start:
            if backward:
                self.guess_bwd = x
            else:
                self.guess_fwd = x
        return x

    def solve(self, bs, backward=False):
        """bs: list of (V_i, k) tensors (k <= 3) or one packed (sum V_i, k) tensor.  Returns the list of (V_i, k) solutions:
        views of one packed output."""
        return self.split(self.solve_packed(self.pack(bs), backward=backward))


class BatchSolve(Function):
    """x = solver.solve_packed(b); grad_b = solver.solve_packed(grad_x, backward=True) (every M_i is symmetric)."""

    @staticmethod
    def forward(ctx, solver, b):
        ctx.solver = solver
        return solver.solve_packed(b, backward=False)

    @staticmethod
    def backward(ctx, grad_output):
        b_grad = None
        if ctx.needs_input_grad[1]:
            b_grad = ctx.solver.solve_packed(grad_output.contiguous(), backward=True)
        return None, b_grad


# solvers keyed by (tuple(id(M_i)), method[, per-mesh preconditioners unless all Jacobi]), dropped as soon as any M_i is garbage collected (as parameterize._cache)
_cache = {}


def _cache_put(key, value, Ms):
    def cleanup_callback(wr):
        _cache.pop(key, None)

    _cache[key] = (value, [weakref.ref(M, cleanup_callback) for M in Ms])


def from_differential_batch(Ms, us, method='Cholesky', packed=False, precond='jacobi'):
    """Solve M_i v_i = u_i for every mesh i in one batched call; returns the list of (V_i, 3) tensors, differentiable w.r.t.
    every u_i.  method: 'Cholesky' (cold start, rtol 1e-7, as from_differential's) or 'CG' (separate forward and backward
    warm starts per mesh).  For meshes that share one matrix, call from_differential once on the concatenated columns.

    us may also be one packed (sum V_i, 3) tensor, mesh i's rows after mesh i-1's.  packed=True returns the packed
    (sum V_i, 3) solution itself (the list form is views of it), ready for the packed mesh ops (pack_meshes).
    precond: 'jacobi', 'chebyshev' or one of those per mesh, as BatchSolver; each choice keeps its own cached solver."""
    Ms = list(Ms)
    if not isinstance(us, torch.Tensor):
        us = list(us)
    if len(Ms) == 0:
        raise ValueError("from_differential_batch needs at least one mesh")
    if isinstance(us, list) and len(us) != len(Ms):
        raise ValueError(f"got {len(us)} right-hand sides for {len(Ms)} matrices")
    ps = preconditioners(precond, len(Ms))
    key = (tuple(id(M) for M in Ms), method)
    if any(p != "jacobi" for p in ps):
        key += (tuple(ps),)     # (an all-Jacobi batch keeps the two-part key)
    if key not in _cache:
        if method == 'Cholesky':
            solver = BatchSolver(Ms, rtol=1e-7, maxit=10000, warm_start=False, check=False, precond=ps)
        elif method == 'CG':
            solver = BatchSolver(Ms, rtol=1e-7, maxit=10000, warm_start=True, check=True, precond=ps)
        else:
            raise ValueError(f"Unknown solver type '{method}'.")
        _cache_put(key, solver, Ms)
    else:
        solver = _cache[key][0]
    solver.validate(us)
    if isinstance(us, torch.Tensor):
        b = us
    else:
        b = torch.cat(us, 0) if len(us) > 1 else us[0]
    x = BatchSolve.apply(solver, b.contiguous())
    return x if packed else list(torch.split(x, solver.sizes, 0))


class PackedMeshes(NamedTuple):
    """B meshes as one: verts (sum V_i, 3) and faces (sum F_i, 3), mesh i's indices shifted by vert_offsets[i]; the
    offsets (B + 1 int64 each) as device tensors and as host tuples of ints."""
    verts: torch.Tensor
    faces: torch.Tensor
    vert_offsets: torch.Tensor
    face_offsets: torch.Tensor
    vert_offsets_host: tuple
    face_offsets_host: tuple


def pack_meshes(verts_list, faces_list):
    """Packs B meshes into one for the per-face / per-vertex mesh ops.  compute_face_normals, gather_rows and
    massmatrix_voronoi give each mesh's own result on the packed mesh as they are; compute_vertex_normals_batch takes the
    offsets and gives each mesh's compute_vertex_normals.  The face index dtype is kept; verts stay differentiable."""
    verts_list, faces_list = list(verts_list), list(faces_list)
    if len(verts_list) == 0:
        raise ValueError("pack_meshes needs at least one mesh")
    if len(faces_list) != len(verts_list):
        raise ValueError(f"got {len(faces_list)} face arrays for {len(verts_list)} vertex arrays")
    dev, idt = verts_list[0].device, faces_list[0].dtype
    vo, fo = [0], [0]
    shifted = []
    for i, (v, f) in enumerate(zip(verts_list, faces_list)):
        if v.device != dev or f.device != dev:
            raise RuntimeError(f"mesh {i} is not on {dev}: a packed batch lives on one device")
        if v.dim() != 2 or v.shape[1] != 3 or f.dim() != 2 or f.shape[1] != 3:
            raise ValueError(f"mesh {i}: verts must be (V, 3) and faces (F, 3), got {tuple(v.shape)} and {tuple(f.shape)}")
        if f.dtype != idt or idt not in (torch.int32, torch.int64):
            raise TypeError(f"faces[{i}] is {f.dtype}: every faces tensor must be int32, or every one int64")
        shifted.append(f + vo[-1] if vo[-1] else f)
        vo.append(vo[-1] + v.shape[0])
        fo.append(fo[-1] + f.shape[0])
    if idt == torch.int32 and vo[-1] > 2 ** 31 - 1:
        raise ValueError("the packed mesh has more vertices than int32 faces can index")
    verts = torch.cat(verts_list, 0) if len(verts_list) > 1 else verts_list[0]
    faces = torch.cat(shifted, 0).contiguous() if len(shifted) > 1 else shifted[0].contiguous()
    vo_t = torch.tensor(vo, dtype=torch.int64, device=dev)
    fo_t = torch.tensor(fo, dtype=torch.int64, device=dev)
    meshops._remember_offsets(vo_t, tuple(vo))
    meshops._remember_offsets(fo_t, tuple(fo))
    return PackedMeshes(verts, faces, vo_t, fo_t, tuple(vo), tuple(fo))
