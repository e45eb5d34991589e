"""System-matrix assembly on the GPU -- same surface as the reference's largesteps/geometry.py.

    compute_matrix(verts, faces, lambda_, alpha=None, cotan=False) -> torch.sparse_coo_tensor   (geometry.py:96-133)
    laplacian_uniform(verts, faces)                                                            (geometry.py:65-94)
    laplacian_cot(verts, faces)                                                                (geometry.py:3-63)

The reference builds these with torch.unique(dim=1) + sparse adds + coalesce() (two device sorts over 2x6F int64
indices).  Here one sort-free CUDA pipeline (csrc/ls_assemble.cu) emits the coalesced, row-major sorted int64 COO
*and* the int32 CSR the solver streams, in one pass over per-row buckets.  The CSR is remembered alongside the
returned tensor (weakly, like the reference's solver cache parameterize.py:5-17) so that `from_differential` /
`to_differential` on that matrix need no conversion.

Differences worth knowing (see INTEGRATION.md): the device is taken from `verts` instead of being hard-coded to
'cuda' (geometry.py:60,83,125); `laplacian_cot` returns the coalesced matrix (the reference leaves it uncoalesced);
an isolated vertex gets an explicit 0 on the diagonal of a bare Laplacian (compute_matrix is identical: identity row).

Gradients: as in the reference, whose cotangent matrix is built from torch ops of the positions, the values of a cotangent
matrix carry a graph to `verts` when grad mode is on and `verts.requires_grad` (backward: ls_laplacian_cot_bwd_f32).  The
uniform matrices do not depend on the positions and never carry one.
"""
import ctypes
import warnings
import weakref

import torch

from . import _native as N

ORDER_MIN_V = 8192   # below this everything lives in L1/L2 anyway

# id(M) -> (weakref(M), rowptr int32 (V+1), col int32 (nnz), val float32 (nnz), order int32 (V) or None,
#           the same values with their autograd graph to the positions, or None)
_csr_cache = {}


class _TorchAlloc:
    """default allocator of the assembly: one torch tensor per buffer (largesteps_b200.remesh substitutes an arena)"""

    @staticmethod
    def take(nbytes, dev):
        return torch.empty(max(int(nbytes), 1), dtype=torch.uint8, device=dev)


_ESIZE = {torch.int64: 8, torch.int32: 4, torch.float32: 4}


def _view(buf, dtype, n):
    return buf[: n * _ESIZE[dtype]].view(dtype)


def _remember_csr(M, rowptr, col, val, order=None, val_graph=None):
    key = id(M)

    def _drop(_wr, key=key):
        _csr_cache.pop(key, None)

    _csr_cache[key] = (weakref.ref(M, _drop), rowptr, col, val, order, val_graph)


def order_of(M):
    """Locality order (new -> old vertex, int32) recorded by compute_matrix for this matrix, or None."""
    ent = _csr_cache.get(id(M))
    if ent is not None and ent[0]() is M:
        return ent[4]
    return None


def values_with_graph(M):
    """M's values as the differentiable (nnz,) tensor the cotangent assembly built them as, or None (no graph, or not a
    matrix of this package).  Products with M send their gradient here directly, in M's own order: handing torch's sparse
    constructor a sparse gradient would cost a sparse_mask, as much as a sort of all nnz entries."""
    ent = _csr_cache.get(id(M))
    if ent is not None and ent[0]() is M:
        return ent[5]
    return None


def morton_order(verts, alloc=_TorchAlloc):
    """perm[new] = old along a Morton curve of the vertex positions (csrc/ls_order.cu); deterministic."""
    N.require_cuda(verts, "verts")
    v = verts.detach().to(torch.float32).contiguous()
    V = v.shape[0]
    perm = _view(alloc.take(4 * (V + 8), v.device), torch.int32, V + 8)[:V]
    with torch.cuda.device(v.device):
        nbytes = ctypes.c_size_t(0)
        N.check(N.lib().ls_order_workspace_bytes(V, ctypes.byref(nbytes)), "ls_order_workspace_bytes")
        ws = alloc.take(nbytes.value, v.device)
        N.check(N.lib().ls_order_morton(N.ptr(v), V, N.ptr(perm), N.ptr(ws), nbytes.value, N.stream_ptr(v.device)),
                "ls_order_morton")
    return perm


def csr_of(M):
    """int32 CSR (rowptr, col, val) of a sparse COO system matrix; cached for matrices built by compute_matrix,
    converted on the device (ls_coo_to_csr) for any other coalesced torch sparse COO tensor."""
    ent = _csr_cache.get(id(M))
    if ent is not None and ent[0]() is M:
        return ent[1], ent[2], ent[3]
    if not isinstance(M, torch.Tensor) or M.layout != torch.sparse_coo:
        raise TypeError("expected a torch sparse COO matrix (as returned by compute_matrix)")
    N.require_cuda(M, "M")
    Mc = M if M.is_coalesced() else M.coalesce()
    idx = Mc.indices()
    val = Mc.values()
    if val.dtype != torch.float32:
        raise TypeError(f"system matrix must be float32, got {val.dtype}")
    V = Mc.shape[0]
    nnz = val.shape[0]
    rows = idx[0].contiguous()
    cols = idx[1].contiguous()
    rowptr = torch.empty(V + 1 + 8, dtype=torch.int32, device=M.device)[: V + 1]
    col = torch.empty(nnz + 8, dtype=torch.int32, device=M.device)[:nnz]
    with torch.cuda.device(M.device):
        N.check(N.lib().ls_coo_to_csr(N.ptr(rows), N.ptr(cols), nnz, V, N.ptr(rowptr), N.ptr(col),
                                      N.stream_ptr(M.device)), "ls_coo_to_csr")
    val = val.contiguous()
    _remember_csr(M, rowptr, col, val)
    return rowptr, col, val


def _assemble(verts, faces, shift, scale, cotan, alloc=_TorchAlloc):
    N.require_cuda(verts, "verts")
    N.require_cuda(faces, "faces")
    if faces.device != verts.device:
        raise RuntimeError("verts and faces must live on the same device")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"faces must have shape (F, 3), got {tuple(faces.shape)}")
    if verts.dim() != 2 or verts.shape[1] != 3:
        raise ValueError(f"verts must have shape (V, 3), got {tuple(verts.shape)}")
    if faces.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"faces must be int32 or int64, got {faces.dtype}")
    V = verts.shape[0]
    # the cotangent values depend on the positions: they carry a graph to verts when autograd asks for one
    graph = cotan and torch.is_grad_enabled() and verts.requires_grad
    if graph:
        val, idx, rowptr, col = _CotValues.apply(verts, faces, float(shift), float(scale), alloc)
    else:
        idx, val, rowptr, col = _fill(verts, faces, shift, scale, cotan, alloc)
    with warnings.catch_warnings():      # torch warns once that invariant checks are off; the kernel guarantees them
        warnings.simplefilter("ignore")
        M = torch.sparse_coo_tensor(idx, val, (V, V), is_coalesced=True, check_invariants=False)
    # the solver re-orders its private copy of M along a Morton curve of the positions (the public M is untouched)
    order = morton_order(verts, alloc) if V >= ORDER_MIN_V else None
    _remember_csr(M, rowptr, col, val.detach() if graph else val, order, val if graph else None)
    return M


class _CotValues(torch.autograd.Function):
    """The values of the cotangent M = shift I + scale L as a function of the positions: the forward is the assembly
    (_fill), the backward ls_laplacian_cot_bwd_f32.  The index tensors come out as non-differentiable outputs."""

    @staticmethod
    def forward(ctx, verts, faces, shift, scale, alloc):
        idx, val, rowptr, col = _fill(verts, faces, shift, scale, True, alloc)
        ctx.mark_non_differentiable(idx, rowptr, col)
        ctx.save_for_backward(verts.detach().to(torch.float32).contiguous(), rowptr, col)
        ctx.faces, ctx.scale, ctx.dtype = faces, scale, verts.dtype
        return val, idx, rowptr, col

    @staticmethod
    def backward(ctx, gval, *_):
        from .meshops import face_incidence
        vc, rowptr, col = ctx.saved_tensors
        faces = ctx.faces
        fc = faces.contiguous()
        V, F = vc.shape[0], fc.shape[0]
        dev = vc.device
        ptr, items = face_incidence(faces, V)
        g = gval.to(torch.float32).contiguous()
        gv = torch.empty((V, 3), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            nbytes = ctypes.c_size_t(0)
            N.check(N.lib().ls_laplacian_cot_bwd_scratch_bytes(F, ctypes.byref(nbytes)), "ls_laplacian_cot_bwd_scratch_bytes")
            scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
            N.check(N.lib().ls_laplacian_cot_bwd_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, ctx.scale, N.ptr(rowptr),
                                                     N.ptr(col), N.ptr(g), N.ptr(ptr), N.ptr(items), N.ptr(scratch),
                                                     nbytes.value, N.ptr(gv), N.stream_ptr(dev)), "ls_laplacian_cot_bwd_f32")
        return gv.to(ctx.dtype), None, None, None, None


def _fill(verts, faces, shift, scale, cotan, alloc):
    """Count and fill: the coalesced COO indices (2, nnz) int64 and values (nnz) float32, and the int32 CSR rowptr / col that
    shares those values."""
    V, F = verts.shape[0], faces.shape[0]
    dev = verts.device
    faces_c = faces.contiguous()
    verts_c = verts.detach().to(torch.float32).contiguous() if cotan else None
    lib = N.lib()
    with torch.cuda.device(dev):
        st = N.stream_ptr(dev)
        nbytes = ctypes.c_size_t(0)
        N.check(lib.ls_assemble_workspace_bytes(F, V, ctypes.byref(nbytes)), "ls_assemble_workspace_bytes")
        ws = alloc.take(nbytes.value, dev)
        nnz = ctypes.c_int64(0)
        N.check(lib.ls_assemble_count(N.ptr(faces_c), faces_c.element_size(), F, V, N.ptr(ws), nbytes.value,
                                      ctypes.byref(nnz), st), "ls_assemble_count")
        nnz = nnz.value
        idx = _view(alloc.take(16 * nnz, dev), torch.int64, 2 * nnz).view(2, nnz)
        val = _view(alloc.take(4 * (nnz + 8), dev), torch.float32, nnz + 8)[:nnz]
        rowptr = _view(alloc.take(4 * (V + 1 + 8), dev), torch.int32, V + 1 + 8)[: V + 1]
        col = _view(alloc.take(4 * (nnz + 8), dev), torch.int32, nnz + 8)[:nnz]
        # COO values and CSR values are the same array (same order): write it once
        N.check(lib.ls_assemble_fill(N.ptr(faces_c), faces_c.element_size(), N.ptr(verts_c), F, V, int(bool(cotan)),
                                     float(shift), float(scale), N.ptr(ws), nbytes.value, nnz,
                                     N.ptr(idx[0]), N.ptr(idx[1]), N.ptr(val),
                                     N.ptr(rowptr), N.ptr(col), N.ptr(val), st), "ls_assemble_fill")
    return idx, val, rowptr, col


def laplacian_uniform(verts, faces):
    """Combinatorial Laplacian L = D - A (geometry.py:65-94), coalesced float32 sparse COO on verts.device."""
    return _assemble(verts, faces, 0.0, 1.0, False)


def laplacian_cot(verts, faces):
    """Cotangent Laplacian, PSD, no 1/2 factor (geometry.py:3-63), returned coalesced."""
    return _assemble(verts, faces, 0.0, 1.0, True)


def compute_matrix(verts, faces, lambda_, alpha=None, cotan=False, alloc=None):
    """Build the parameterization matrix (geometry.py:96-133).

    If alpha is defined, M = (1-alpha)*I + alpha*L, otherwise M = I + lambda_*L (lambda_ is ignored when alpha is
    given, as in the reference).  Returns a coalesced float32 torch.sparse_coo_tensor with int64 indices.
    `alloc` (not in the reference): where the output and work buffers come from (largesteps_b200.remesh.Arena).
    """
    if alpha is None:
        shift, scale = 1.0, float(lambda_)
    else:
        if alpha < 0.0 or alpha >= 1.0:
            raise ValueError(f"Invalid value for alpha: {alpha} : it should take values between 0 (included) and 1 (excluded)")
        shift, scale = 1.0 - alpha, float(alpha)
    return _assemble(verts, faces, shift, scale, cotan, alloc if alloc is not None else _TorchAlloc)
