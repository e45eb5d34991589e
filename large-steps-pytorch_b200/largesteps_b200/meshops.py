"""Per-step glue either side of the solve, on the GPU -- same surface as the reference's scripts/geometry.py plus the two
one-liners of its optimisation loop (scripts/main.py:176-180, 192-195).

    remove_duplicates(v, f)                        scripts/geometry.py:3-11    (setup, once per mesh / remesh)
    average_edge_length(verts, faces)              scripts/geometry.py:13-35   (setup, once per remesh)
    massmatrix_voronoi(verts, faces)               scripts/geometry.py:35-89   -- (V,), differentiable; not in the reference loop
    safe_acos(x)                                   scripts/geometry.py:113-114
    gather_rows(v, idx)                            v[duplicate_idx], scripts/main.py:176,180 -- differentiable
    compute_face_normals(verts, faces)             scripts/geometry.py:91-110  -- (3,F), differentiable
    compute_vertex_normals(verts, faces, fn)       scripts/geometry.py:115-147 -- (V,3), differentiable
    compute_vertex_normals_batch(...)              the same per mesh of a packed batch (batch.pack_meshes), bitwise
    laplacian_regularizer(L, v, bilaplacian)       scripts/main.py:192-195     -- through the library's SpMM
    laplacian_cot_product(verts, faces, x)         laplacian_cot(verts, faces) @ x without the matrix -- differentiable

The reference spends ~40 eager kernels (index_select, cross, norms, acos, nine atomic index_add_ ...) per step on the
normals alone; here each operator is one kernel per direction (csrc/ls_glue.cu), gathers over an incidence list instead of
atomic scatter-adds, bit-reproducible.  The incidence list depends on the connectivity only and is cached per `faces`
tensor (weakly, like the solver cache of parameterize.py:5-17).
"""
import ctypes
import weakref

import torch

from . import _native as N
from .parameterize import spmm_autograd

_inc_cache = {}      # id(faces) -> (weakref, version, V, ptr, items)
_bucket_cache = {}   # id(idx)   -> (weakref, version, V, ptr, items)


def _check_mesh(verts, faces):
    N.require_cuda(verts, "verts")
    N.require_cuda(faces, "faces")
    if verts.dim() != 2 or verts.shape[1] != 3:
        raise ValueError(f"verts must have shape (V, 3), got {tuple(verts.shape)}")
    if faces.dim() != 2 or faces.shape[1] != 3:
        raise ValueError(f"faces must have shape (F, 3), got {tuple(faces.shape)}")
    if faces.dtype not in (torch.int32, torch.int64):
        raise TypeError(f"faces must be int32 or int64, got {faces.dtype}")
    if verts.dtype != torch.float32:
        raise TypeError(f"verts must be float32, got {verts.dtype}")
    if faces.device != verts.device:
        raise RuntimeError("verts and faces must live on the same device")


def _buckets(cache, key_tensor, nkeys, per_face):
    ent = cache.get(id(key_tensor))
    if ent is not None and ent[0]() is key_tensor and ent[1] == key_tensor._version and ent[2] == nkeys:
        return ent[3], ent[4]
    t = key_tensor.contiguous()
    n = t.numel()
    dev = t.device
    lib = N.lib()
    ptr = torch.empty(nkeys + 1, dtype=torch.int32, device=dev)
    items = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        nbytes = ctypes.c_size_t(0)
        N.check(lib.ls_bucket_workspace_bytes(nkeys, ctypes.byref(nbytes)), "ls_bucket_workspace_bytes")
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        if per_face:
            N.check(lib.ls_face_incidence(N.ptr(t), t.element_size(), n // 3, nkeys, N.ptr(ptr), N.ptr(items), N.ptr(ws),
                                          nbytes.value, N.stream_ptr(dev)), "ls_face_incidence")
        else:
            N.check(lib.ls_index_buckets(N.ptr(t), t.element_size(), n, nkeys, N.ptr(ptr), N.ptr(items), N.ptr(ws),
                                         nbytes.value, N.stream_ptr(dev)), "ls_index_buckets")
    key = id(key_tensor)

    def _drop(_wr, key=key):
        cache.pop(key, None)

    cache[key] = (weakref.ref(key_tensor, _drop), key_tensor._version, nkeys, ptr, items)
    return ptr, items


def face_incidence(faces, V):
    """(ptr, items): for vertex v the sorted codes 4 * face + corner of its incident face corners (cached per tensor)."""
    return _buckets(_inc_cache, faces, V, True)


def _scratch(dev):
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_glue_scratch_bytes(ctypes.byref(nb)), "ls_glue_scratch_bytes")
    return torch.empty(nb.value, dtype=torch.uint8, device=dev)


# ---- setup-time helpers (not on the per-step path) ---------------------------------------------------------------------
def remove_duplicates(v, f):
    """Mesh representation with no duplicate vertices + the mapping to the original layout (scripts/geometry.py:3-11).
    Runs once per mesh / remesh; the sort behind torch.unique(dim=0) is torch's (setup, not the per-step path)."""
    unique_verts, inverse = torch.unique(v, dim=0, return_inverse=True)
    new_faces = inverse[f.long()]
    return unique_verts, new_faces, inverse


def average_edge_length(verts, faces):
    """Average length of all (face) edges (scripts/geometry.py:13-35); used once per remesh (scripts/main.py:146)."""
    fv = verts[faces.long()]
    v0, v1, v2 = fv[:, 0], fv[:, 1], fv[:, 2]
    A = (v1 - v2).norm(dim=1)
    B = (v0 - v2).norm(dim=1)
    C = (v0 - v1).norm(dim=1)
    return (A + B + C).sum() / faces.shape[0] / 3


# ---- v[duplicate_idx] ----------------------------------------------------------------------------------------------------
class _GatherRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, v, idx):
        N.require_cuda(v, "v")
        N.require_cuda(idx, "idx")
        if v.dtype != torch.float32 or v.dim() != 2:
            raise TypeError("gather_rows: v must be a float32 (V, k) tensor")
        if idx.dtype not in (torch.int32, torch.int64) or idx.dim() != 1:
            raise TypeError("gather_rows: idx must be a 1-D int32 / int64 tensor")
        vc = v.detach().contiguous()
        ic = idx.contiguous()
        out = torch.empty((ic.shape[0], vc.shape[1]), dtype=torch.float32, device=v.device)
        with torch.cuda.device(v.device):
            N.check(N.lib().ls_gather_rows_f32(N.ptr(vc), N.ptr(ic), ic.element_size(), ic.shape[0], vc.shape[1], N.ptr(out),
                                               N.stream_ptr(v.device)), "ls_gather_rows_f32")
        ctx.idx = idx
        ctx.V = v.shape[0]
        return out

    @staticmethod
    def backward(ctx, g):
        if g.shape[0] == 0:
            # nothing was gathered, so nothing flows back; the empty g has no storage, and ls_gather_rows_bwd_f32 rejects
            # its NULL pointer because the C call cannot tell that every bucket is empty
            return torch.zeros((ctx.V, g.shape[1]), dtype=torch.float32, device=g.device), None
        ptr, items = _buckets(_bucket_cache, ctx.idx, ctx.V, False)
        gc = g.contiguous()
        out = torch.empty((ctx.V, gc.shape[1]), dtype=torch.float32, device=g.device)
        with torch.cuda.device(g.device):
            N.check(N.lib().ls_gather_rows_bwd_f32(N.ptr(gc), N.ptr(ptr), N.ptr(items), ctx.V, gc.shape[1], N.ptr(out),
                                                   N.stream_ptr(g.device)), "ls_gather_rows_bwd_f32")
        return out, None


def gather_rows(v, idx):
    """v[idx] (rows), differentiable w.r.t. v; the backward is a deterministic segmented sum (no atomics)."""
    return _GatherRows.apply(v, idx)


# ---- normals ---------------------------------------------------------------------------------------------------------------
class _FaceNormals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces):
        _check_mesh(verts, faces)
        vc = verts.detach().contiguous()
        fc = faces.contiguous()
        F = fc.shape[0]
        n = torch.empty((3, F), dtype=torch.float32, device=verts.device)
        with torch.cuda.device(verts.device):
            N.check(N.lib().ls_face_normals_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, N.ptr(n), N.stream_ptr(verts.device)),
                    "ls_face_normals_f32")
        ctx.save_for_backward(vc)
        ctx.faces = faces
        ctx.fc = fc
        return n

    @staticmethod
    def backward(ctx, gn):
        (vc,) = ctx.saved_tensors
        fc = ctx.fc
        V, F = vc.shape[0], fc.shape[0]
        ptr, items = face_incidence(ctx.faces, V)
        g = gn.contiguous()
        out = torch.empty((V, 3), dtype=torch.float32, device=vc.device)
        with torch.cuda.device(vc.device):
            N.check(N.lib().ls_face_normals_bwd_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items), N.ptr(g),
                                                    N.ptr(out), N.stream_ptr(vc.device)), "ls_face_normals_bwd_f32")
        return out, None


def compute_face_normals(verts, faces):
    """Per-face unit normals, shape (3, F) like the reference (scripts/geometry.py:91-110)."""
    return _FaceNormals.apply(verts, faces)


class _VertexNormals(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, face_normals):
        _check_mesh(verts, faces)
        vc = verts.detach().contiguous()
        fc = faces.contiguous()
        fn = face_normals.detach().contiguous()
        V, F = vc.shape[0], fc.shape[0]
        if tuple(fn.shape) != (3, F) or fn.dtype != torch.float32:
            raise ValueError(f"face_normals must be float32 of shape (3, {F}), got {tuple(fn.shape)} {fn.dtype}")
        ptr, items = face_incidence(faces, V)
        dev = verts.device
        out = torch.empty((V, 3), dtype=torch.float32, device=dev)
        raw = torch.empty(V, dtype=torch.float32, device=dev)
        norms = torch.empty(4, dtype=torch.float32, device=dev)
        scratch = _scratch(dev)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_vertex_normals_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items), N.ptr(fn),
                                                  N.ptr(out), N.ptr(raw), N.ptr(norms), N.ptr(scratch), N.stream_ptr(dev)),
                    "ls_vertex_normals_f32")
        ctx.save_for_backward(vc, fn, out, raw, norms, ptr, items)
        ctx.fc = fc
        return out

    @staticmethod
    def backward(ctx, gout):
        vc, fn, out, raw, norms, ptr, items = ctx.saved_tensors
        fc = ctx.fc
        V, F = vc.shape[0], fc.shape[0]
        dev = vc.device
        g = gout.contiguous()
        gv = torch.empty((V, 3), dtype=torch.float32, device=dev)
        gfn = torch.empty((3, F), dtype=torch.float32, device=dev)
        scratch = _scratch(dev)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_vertex_normals_bwd_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items),
                                                      N.ptr(fn), N.ptr(out), N.ptr(raw), N.ptr(norms), N.ptr(g), N.ptr(gv),
                                                      N.ptr(gfn), N.ptr(scratch), N.stream_ptr(dev)), "ls_vertex_normals_bwd_f32")
        return gv, None, gfn


def compute_vertex_normals(verts, faces, face_normals):
    """Angle-weighted per-vertex normals (V, 3) from face normals (scripts/geometry.py:115-147), including the reference's
    normalisation of the edge fields by their GLOBAL Frobenius norm (geometry.py:137-140)."""
    return _VertexNormals.apply(verts, faces, face_normals)


# ---- vertex normals of packed meshes ------------------------------------------------------------------------------------------
_offsets_cache = {}      # id(offset tensor) -> (weakref, version, host tuple)
_offsets_dev_cache = {}  # (device, host tuple) -> device int64 tensor
_batch_faces_cache = {}  # id(faces) -> (weakref, version, vert offsets) of a packing whose per-mesh ranges were checked


def _offsets(o, dev, what):
    """Host tuple and device int64 tensor of B + 1 offsets given as a sequence of ints or as an int64 tensor.  A tensor's
    values are read once (one synchronisation) and cached with the tensor; pack_meshes fills that cache."""
    if isinstance(o, torch.Tensor):
        ent = _offsets_cache.get(id(o))
        if ent is not None and ent[0]() is o and ent[1] == o._version:
            host = ent[2]
        else:
            if o.dim() != 1 or o.dtype not in (torch.int32, torch.int64):
                raise TypeError(f"{what} must be a 1-D int64 tensor or a sequence of ints")
            host = tuple(int(x) for x in o.tolist())
            _remember_offsets(o, host)
        if o.device == torch.device(dev) and o.dtype == torch.int64 and o.is_contiguous():
            return host, o
    else:
        host = tuple(int(x) for x in o)
    key = (str(dev), host)
    t = _offsets_dev_cache.get(key)
    if t is None:
        t = _offsets_dev_cache[key] = torch.tensor(host, dtype=torch.int64, device=dev)
    return host, t


def _remember_offsets(o, host):
    key = id(o)

    def _drop(_wr, key=key):
        _offsets_cache.pop(key, None)

    _offsets_cache[key] = (weakref.ref(o, _drop), o._version, host)


def _check_offsets(vo, fo, V, F, names=("vert_offsets", "face_offsets")):
    if len(vo) < 2 or len(vo) != len(fo):
        raise ValueError(f"{names[0]} and {names[1]} must both hold B + 1 >= 2 entries, got {len(vo)} and {len(fo)}")
    for name, o, end in ((names[0], vo, V), (names[1], fo, F)):
        if o[0] != 0 or o[-1] != end:
            raise ValueError(f"{name} must start at 0 and end at {end}, got {o[0]} .. {o[-1]}")
        if any(b < a for a, b in zip(o[:-1], o[1:])):
            raise ValueError(f"{name} must be non-decreasing")


def _check_face_ranges(faces, vo, vo_dev, fo):
    """IndexError unless every face of mesh i indexes vertices in [vo[i], vo[i+1]) (checked once per faces tensor)."""
    ent = _batch_faces_cache.get(id(faces))
    if ent is not None and ent[0]() is faces and ent[1] == faces._version and ent[2] == vo:
        return
    counts = torch.tensor([b - a for a, b in zip(fo[:-1], fo[1:])], dtype=torch.int64, device=faces.device)
    mesh = torch.repeat_interleave(torch.arange(len(counts), device=faces.device), counts)
    f = faces.long()
    bad = ((f < vo_dev[mesh, None]) | (f >= vo_dev[mesh + 1, None])).any(1)
    if bool(bad.any()):
        i = int(mesh[bad.nonzero()[0, 0]])
        raise IndexError(f"a face of mesh {i} indexes a vertex outside the mesh's range [{vo[i]}, {vo[i + 1]})")
    key = id(faces)

    def _drop(_wr, key=key):
        _batch_faces_cache.pop(key, None)

    _batch_faces_cache[key] = (weakref.ref(faces, _drop), faces._version, vo)


def _batch_scratch(dev, B):
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_vertex_normals_batch_scratch_bytes(B, ctypes.byref(nb)), "ls_vertex_normals_batch_scratch_bytes")
    return torch.empty(nb.value, dtype=torch.uint8, device=dev)


class _VertexNormalsBatch(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, face_normals, vert_offsets, face_offsets):
        _check_mesh(verts, faces)
        N.require_cuda(face_normals, "face_normals")
        vc = verts.detach().contiguous()
        fc = faces.contiguous()
        fn = face_normals.detach().contiguous()
        V, F = vc.shape[0], fc.shape[0]
        if tuple(fn.shape) != (3, F) or fn.dtype != torch.float32:
            raise ValueError(f"face_normals must be float32 of shape (3, {F}), got {tuple(fn.shape)} {fn.dtype}")
        dev = verts.device
        vo, vo_dev = _offsets(vert_offsets, dev, "vert_offsets")
        fo, fo_dev = _offsets(face_offsets, dev, "face_offsets")
        _check_offsets(vo, fo, V, F)
        B = len(vo) - 1
        ptr, items = face_incidence(faces, V)      # IndexError on an index outside [0, V)
        _check_face_ranges(faces, vo, vo_dev, fo)  # ... and outside the face's own mesh
        vo_h, fo_h = (ctypes.c_int64 * (B + 1))(*vo), (ctypes.c_int64 * (B + 1))(*fo)
        out = torch.empty((V, 3), dtype=torch.float32, device=dev)
        raw = torch.empty(V, dtype=torch.float32, device=dev)
        norms = torch.empty((B, 3), dtype=torch.float32, device=dev)
        scratch = _batch_scratch(dev, B)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_vertex_normals_batch_f32(
                N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, B, N.ptr(vo_dev), N.ptr(fo_dev), vo_h, fo_h, N.ptr(ptr),
                N.ptr(items), N.ptr(fn), N.ptr(out), N.ptr(raw), N.ptr(norms), N.ptr(scratch), scratch.numel(),
                N.stream_ptr(dev)), "ls_vertex_normals_batch_f32")
        ctx.save_for_backward(vc, fn, out, raw, norms, ptr, items, vo_dev, fo_dev)
        ctx.fc = fc
        ctx.host = (vo_h, fo_h)
        return out

    @staticmethod
    def backward(ctx, gout):
        vc, fn, out, raw, norms, ptr, items, vo_dev, fo_dev = ctx.saved_tensors
        fc = ctx.fc
        vo_h, fo_h = ctx.host
        V, F, B = vc.shape[0], fc.shape[0], norms.shape[0]
        dev = vc.device
        g = gout.contiguous()
        gv = torch.empty((V, 3), dtype=torch.float32, device=dev)
        gfn = torch.empty((3, F), dtype=torch.float32, device=dev)
        scratch = _batch_scratch(dev, B)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_vertex_normals_batch_bwd_f32(
                N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, B, N.ptr(vo_dev), N.ptr(fo_dev), vo_h, fo_h, N.ptr(ptr),
                N.ptr(items), N.ptr(fn), N.ptr(out), N.ptr(raw), N.ptr(norms), N.ptr(g), N.ptr(gv), N.ptr(gfn),
                N.ptr(scratch), scratch.numel(), N.stream_ptr(dev)), "ls_vertex_normals_batch_bwd_f32")
        return gv, None, gfn, None, None


def compute_vertex_normals_batch(verts, faces, face_normals, vert_offsets, face_offsets):
    """compute_vertex_normals of every mesh of a packed batch (batch.pack_meshes) in one call per direction.

    verts (sum V_i, 3), faces (sum F_i, 3) with each mesh's indices shifted by its first vertex, face_normals (3, sum F_i);
    vert_offsets / face_offsets: B + 1 offsets each, as int64 tensors or sequences of ints.  The reference's global edge-field
    norms (geometry.py:137-140) are taken per mesh, so the result, and its gradients w.r.t. verts and face_normals, are
    bitwise those of compute_vertex_normals called on each mesh alone.  Offset tensors are read on the host once and cached
    with the tensor (pack_meshes' tensors are cached from the start)."""
    return _VertexNormalsBatch.apply(verts, faces, face_normals, vert_offsets, face_offsets)


def safe_acos(x):
    """acos with its argument clamped to [-1, 1] (scripts/geometry.py:113-114)."""
    return torch.acos(x.clamp(min=-1, max=1))


# ---- Voronoi mass matrix ---------------------------------------------------------------------------------------------------
class _MassVoronoi(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces):
        _check_mesh(verts, faces)
        vc = verts.detach().contiguous()
        fc = faces.contiguous()
        V, F = vc.shape[0], fc.shape[0]
        ptr, items = face_incidence(faces, V)      # raises IndexError on a face index outside [0, V)
        dev = verts.device
        out = torch.empty(V, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_massmatrix_voronoi_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items),
                                                      N.ptr(out), N.stream_ptr(dev)), "ls_massmatrix_voronoi_f32")
        ctx.save_for_backward(vc, ptr, items)
        ctx.fc = fc
        return out

    @staticmethod
    def backward(ctx, gm):
        vc, ptr, items = ctx.saved_tensors
        fc = ctx.fc
        V, F = vc.shape[0], fc.shape[0]
        dev = vc.device
        g = gm.contiguous()
        gv = torch.empty((V, 3), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_massmatrix_voronoi_bwd_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items),
                                                          N.ptr(g), N.ptr(gv), N.stream_ptr(dev)), "ls_massmatrix_voronoi_bwd_f32")
        return gv, None


def massmatrix_voronoi(verts, faces):
    """Mixed Voronoi area of each vertex, (V,) float32 (scripts/geometry.py:35-89), differentiable w.r.t. verts.

    Same float32 operations as the reference, in the same order, with the same quirks: Heron's area is not clamped, the
    obtuse override is three sequential torch.where's, and a face with a zero-length edge makes its vertices NaN.  One
    gather per vertex over the cached incidence list instead of a scatter_add_, so results are bit-reproducible.  The
    reference's optimisation loop (scripts/main.py) does not call this function."""
    return _MassVoronoi.apply(verts, faces)


# ---- L_cot(verts) @ x without the matrix -------------------------------------------------------------------------------------
class _CotLaplacianProduct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, verts, faces, x):
        _check_mesh(verts, faces)
        N.require_cuda(x, "x")
        V, F = verts.shape[0], faces.shape[0]
        if x.dim() != 2 or x.shape[0] != V or x.shape[1] < 1:
            raise ValueError(f"x must have shape (V, k) with V = {V} and k >= 1, got {tuple(x.shape)}")
        if x.dtype != torch.float32:
            raise TypeError(f"x must be float32, got {x.dtype}")
        if x.device != verts.device:
            raise RuntimeError("x must live on the device of verts")
        ptr, items = face_incidence(faces, V)      # raises IndexError on a face index outside [0, V)
        vc = verts.detach().contiguous()
        xc = x.detach().contiguous()
        fc = faces.contiguous()
        dev = verts.device
        k = xc.shape[1]
        y = torch.empty((V, k), dtype=torch.float32, device=dev)
        w = torch.empty(max(3 * F, 1), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            N.check(N.lib().ls_cot_laplacian_product_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items),
                                                         N.ptr(xc), k, N.ptr(y), N.ptr(w), N.stream_ptr(dev)),
                    "ls_cot_laplacian_product_f32")
        ctx.save_for_backward(vc, xc, w, ptr, items)
        ctx.fc = fc
        return y

    @staticmethod
    def backward(ctx, gy):
        vc, xc, w, ptr, items = ctx.saved_tensors
        fc = ctx.fc
        V, F, k = vc.shape[0], fc.shape[0], xc.shape[1]
        dev = vc.device
        need_v, need_x = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        g = gy.contiguous()
        gx = torch.empty((V, k), dtype=torch.float32, device=dev) if need_x else None
        gv = torch.empty((V, 3), dtype=torch.float32, device=dev) if need_v else None
        nbytes = ctypes.c_size_t(0)
        scratch = None
        with torch.cuda.device(dev):
            if need_v:
                N.check(N.lib().ls_cot_laplacian_product_scratch_bytes(F, ctypes.byref(nbytes)),
                        "ls_cot_laplacian_product_scratch_bytes")
                scratch = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
            N.check(N.lib().ls_cot_laplacian_product_bwd_f32(N.ptr(vc), N.ptr(fc), fc.element_size(), F, V, N.ptr(ptr), N.ptr(items),
                                                             N.ptr(w), N.ptr(xc), k, N.ptr(g), N.ptr(gx), N.ptr(gv), N.ptr(scratch),
                                                             nbytes.value, N.stream_ptr(dev)), "ls_cot_laplacian_product_bwd_f32")
        return gv, None, gx


def laplacian_cot_product(verts, faces, x):
    """laplacian_cot(verts, faces) @ x as a (V, k) float32 tensor, without building the matrix; differentiable w.r.t. verts
    (through the cotangent weights) and x.

    y_i = sum over the edges (i, j) of the faces at i of w (x_i - x_j), w the face's cotangent weight as laplacian_cot computes
    it: a self-edge adds nothing, a duplicated face adds twice, an unused vertex gets 0.  Two kernels forward, one for the
    gradient w.r.t. x and two for the gradient w.r.t. verts, each only when asked for; no sort, no host synchronisation after
    the incidence list is cached, bit-reproducible.  The regulariser of scripts/main.py:192-195 on a cotangent L recomputed from
    the current shape is then `laplacian_cot_product(v, f, v).square().mean()` (or `(v * y).mean()`), and autograd adds the
    paths through the weights and through x.  On a packed mesh (batch.pack_meshes) each vertex gathers only its own mesh's
    faces, so every mesh gets what a call on it alone gives."""
    return _CotLaplacianProduct.apply(verts, faces, x)


# ---- regulariser -------------------------------------------------------------------------------------------------------------
def laplacian_regularizer(L, v, bilaplacian=True):
    """reg_loss of scripts/main.py:192-195: (L@v).square().mean() (bi-Laplacian) or (v * (L@v)).mean(), with L @ v through
    the library's SpMM (differentiable w.r.t. v, and w.r.t. L's values when L carries a graph, as for
    laplacian_cot(v, f) with v.requires_grad)."""
    Lv = spmm_autograd(L, v)
    return Lv.square().mean() if bilaplacian else (v * Lv).mean()
