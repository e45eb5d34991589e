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

The remesh itself (main.py:149) runs on the device too:

    v_unique, f_unique = remesh_botsch(v_unique, f_unique, 5, h, True)

Botsch and Kobbelt's isotropic remesher as parallel rounds (csrc/ls_remesh.cu, DESIGN 4.7): split the edges longer than
1.4 h, collapse those shorter than 0.7 h, flip edges to even the valences, relax every vertex tangentially and project
it onto the input surface, `iters` times.  Mesh data stays on the device; the host reads counts only.  `h` may also be a
per-vertex target edge length, and `feature=` pins vertices that are never split, collapsed, flipped or moved:

    v, f, feat = remesh_botsch(v, f, 5, t, True, feature=feat, return_feature=True)
"""
import ctypes
import math

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


_BAD = ((1, "an edge with one face: the mesh must be closed"), (2, "an edge with more than two faces"),
        (4, "a directed edge held by two faces: the faces are not consistently oriented"), (8, "a face repeats a vertex"))


class _Remesher:
    """Device buffers of one remesh_botsch call: vertices and int32 faces with room for a split, and the stages' workspace.
    With a per-vertex target t (V,), also the vertices' bounds high = 1.4 t and low = 0.7 t in float64 (remesh_botsch.cpp:19-20)
    and their feature flags (uint8; `feature` a (V,) bool mask, None for none); without, the stages take scalar bounds."""

    def __init__(self, verts, faces, t=None, feature=None):
        self.dev = verts.device
        self.V, self.F = int(verts.shape[0]), int(faces.shape[0])
        self.verts = verts.detach().to(torch.float32).contiguous().clone()
        self.faces = faces.to(torch.int32).contiguous().clone()
        self.high = self.low = self.feat = None
        if t is not None:
            t = t.detach().to(self.dev, torch.float64)
            self.high, self.low = (1.4 * t).contiguous(), (0.7 * t).contiguous()
            self.feat = torch.zeros(self.V, dtype=torch.uint8, device=self.dev)
            if feature is not None:
                self.feat[feature] = 1
        self.ws = torch.empty(0, dtype=torch.uint8, device=self.dev)
        self.ensure(self.V, self.F)

    def ensure(self, Vc, Fc):
        """Grow the buffers to Vc vertices and Fc faces (their contents kept) and the workspace to match."""
        if Vc > self.verts.shape[0]:
            self.verts = torch.cat([self.verts[:self.V], self.verts.new_empty(Vc - self.V, 3)])
            if self.high is not None:
                self.high, self.low, self.feat = (torch.cat([a[:self.V], a.new_empty(Vc - self.V)])
                                                  for a in (self.high, self.low, self.feat))
        if Fc > self.faces.shape[0]:
            self.faces = torch.cat([self.faces[:self.F], self.faces.new_empty(Fc - self.F, 3)])
        nb = ctypes.c_size_t(0)
        N.check(N.lib().ls_remesh_workspace_bytes(self.verts.shape[0], self.faces.shape[0], ctypes.byref(nb)), "ls_remesh_workspace_bytes")
        if nb.value > self.ws.numel():
            self.ws = torch.empty(nb.value, dtype=torch.uint8, device=self.dev)

    def args(self):
        return N.ptr(self.verts), N.ptr(self.faces)

    def attrs(self):
        return N.ptr(self.high), N.ptr(self.low), N.ptr(self.feat)

    def check(self):
        flags = ctypes.c_uint32(0)
        N.check(N.lib().ls_remesh_check(N.ptr(self.faces), self.F, self.V, N.ptr(self.ws), self.ws.numel(), ctypes.byref(flags),
                                        N.stream_ptr(self.dev)), "ls_remesh_check")
        bad = [msg for bit, msg in _BAD if flags.value & bit]
        if bad:
            raise ValueError("remesh_botsch needs a closed, edge-manifold, consistently oriented mesh: " + "; ".join(bad))

    def split(self, high):
        self.ensure(self.V + 3 * self.F // 2, 4 * self.F)
        n = ctypes.c_int64(0)
        N.check(N.lib().ls_remesh_split_v(*self.args(), self.V, self.F, self.verts.shape[0], self.faces.shape[0], high, *self.attrs(),
                                          N.ptr(self.ws), self.ws.numel(), ctypes.byref(n), N.stream_ptr(self.dev)), "ls_remesh_split_v")
        self.V += n.value
        self.F += 2 * n.value
        return n.value

    def collapse_round(self, low, high, live):
        n = ctypes.c_int64(0)
        N.check(N.lib().ls_remesh_collapse_round_v(*self.args(), self.V, self.F, live, low, high, *self.attrs(), N.ptr(self.ws),
                                                   self.ws.numel(), ctypes.byref(n), N.stream_ptr(self.dev)), "ls_remesh_collapse_round_v")
        return n.value

    def compact(self):
        nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
        N.check(N.lib().ls_remesh_compact_v(*self.args(), self.V, self.F, *self.attrs(), N.ptr(self.ws), self.ws.numel(),
                                            ctypes.byref(nv), ctypes.byref(nf), N.stream_ptr(self.dev)), "ls_remesh_compact_v")
        self.V, self.F = nv.value, nf.value

    def flip_round(self):
        n = ctypes.c_int64(0)
        N.check(N.lib().ls_remesh_flip_round_v(*self.args(), self.V, self.F, *self.attrs(), N.ptr(self.ws), self.ws.numel(),
                                               ctypes.byref(n), N.stream_ptr(self.dev)), "ls_remesh_flip_round_v")
        return n.value

    def relax(self, target):
        N.check(N.lib().ls_remesh_relax_v(*self.args(), self.V, self.F, N.ptr(target._bvh), target.F, *self.attrs(), N.ptr(self.ws),
                                          self.ws.numel(), N.stream_ptr(self.dev)), "ls_remesh_relax_v")

    def mesh(self):
        return self.verts[:self.V], self.faces[:self.F]

    def features(self):
        """The feature vertices' indices, ascending (int64)."""
        if self.feat is None:
            return torch.zeros(0, dtype=torch.int64, device=self.dev)
        return torch.nonzero(self.feat[:self.V]).flatten()


class _StageTimer:
    """CUDA events around each stage; `ms` adds up the device time per stage once the call has synchronised."""

    def __init__(self, ms):
        self.ms, self.marks = ms, []

    def __call__(self, name):
        if self.ms is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.marks.append((name, ev))

    def close(self):
        if self.ms is None:
            return
        self("end")
        self.marks[-1][1].synchronize()
        for (name, a), (_, b) in zip(self.marks, self.marks[1:]):
            self.ms[name] = self.ms.get(name, 0.0) + a.elapsed_time(b)


def _check_targets(h, V):
    """h: a positive finite number, or a (V,) float32 / float64 tensor of them.  True for a tensor."""
    if isinstance(h, torch.Tensor):
        if h.dtype not in (torch.float32, torch.float64) or tuple(h.shape) != (V,):
            raise ValueError(f"h must be a positive finite float or a ({V},) float32 / float64 tensor, got {h.dtype} {tuple(h.shape)}")
        if not bool((torch.isfinite(h) & (h > 0)).all()):
            raise ValueError("h must be positive and finite at every vertex")
        return True
    if isinstance(h, bool) or not isinstance(h, (int, float)) or not math.isfinite(h) or h <= 0:
        raise ValueError(f"h must be a positive finite float, got {h!r}")
    return False


def _feature_mask(feature, V):
    """feature: None, a 1-D integer tensor of vertex indices (any order, repeats allowed) or a (V,) bool mask -> a (V,) bool
    mask or None."""
    if feature is None:
        return None
    if not isinstance(feature, torch.Tensor) or feature.is_floating_point() or feature.is_complex():
        raise TypeError(f"feature must be an integer tensor of vertex indices or a ({V},) bool mask")
    if feature.dtype == torch.bool:
        if tuple(feature.shape) != (V,):
            raise ValueError(f"a bool feature mask must have shape ({V},), got {tuple(feature.shape)}")
        return feature
    if feature.dim() != 1:
        raise ValueError(f"feature indices must be 1-D, got shape {tuple(feature.shape)}")
    if bool(((feature < 0) | (feature >= V)).any()):
        raise IndexError(f"a feature index is outside [0, {V})")
    mask = torch.zeros(V, dtype=torch.bool, device=feature.device)
    mask[feature.long()] = True
    return mask


def remesh_botsch(v, f, iters, h, project=True, stage_ms=None, *, feature=None, return_feature=False):
    """The reference's remesh_botsch(v, f, iters, h, project) on the device: `iters` rounds of split (edges > 1.4 h),
    collapse (edges < 0.7 h), valence flips and tangential relaxation with projection onto the input surface (project=True)
    or onto the mesh before the relaxation (project=False).

    v: CUDA float32 (V, 3); f: int32 / int64 (F, 3) on the same device, a closed, edge-manifold, consistently oriented mesh.
    h: the target edge length, a positive finite float, or a (V,) CUDA float32 / float64 tensor of per-vertex targets t on
    v's device (the reference's remesh_botsch(V, F, target, iters, feature, project)): edge (a, b) is then split above
    (1.4 t_a + 1.4 t_b) / 2, collapsed below (0.7 t_a + 0.7 t_b) / 2, and a new vertex takes the mean of its edge's bounds.
    feature: vertices that are never split, collapsed, flipped or moved, as a 1-D integer tensor of indices into v (any
    order, repeats allowed) or a (V,) bool mask; a feature that no face references is dropped with its vertex.
    Returns (v_new float32, f_new with f's dtype): no duplicate or unreferenced vertices.  Bitwise reproducible; a constant
    tensor h with no feature gives the scalar call's result bit for bit.  return_feature=True adds a third output: the int64
    indices of the feature vertices in v_new, ascending.
    stage_ms: a dict to which each stage's device time in ms is added (split, collapse, flip, relax, and bvh for
    project=False); None to skip the timing."""
    from .distance import MeshDistance
    from .meshops import _check_mesh
    if isinstance(iters, bool) or not isinstance(iters, int) or iters < 0:
        raise ValueError(f"iters must be an int >= 0, got {iters!r}")
    V = int(v.shape[0]) if hasattr(v, "shape") and len(v.shape) > 0 else 0
    per_vertex = _check_targets(h, V)
    mask = _feature_mask(feature, V)
    _check_mesh(v, f)
    for name, t in (("h", h if per_vertex else None), ("feature", mask)):
        if t is not None:
            N.require_cuda(t, name)
            if t.device != v.device:
                raise RuntimeError(f"{name} and verts must live on the same device")
    if f.shape[0] == 0:
        raise ValueError("the mesh has no faces")
    if bool(((f < 0) | (f >= v.shape[0])).any()):
        raise IndexError(f"a face indexes a vertex outside [0, {v.shape[0]})")
    # per-vertex bounds when h is a tensor or a vertex is pinned; scalar bounds (which the stages then ignore) otherwise
    high, low = (0.0, 0.0) if per_vertex else (1.4 * float(h), 0.7 * float(h))
    t = h if per_vertex else (torch.full((V,), float(h), dtype=torch.float64, device=v.device) if mask is not None else None)
    timer = _StageTimer(stage_ms)
    with torch.cuda.device(v.device):
        r = _Remesher(v, f, t, mask)
        r.check()
        r.compact()                                           # drop vertices no face references
        target = MeshDistance(*r.mesh()) if project else None
        for _ in range(iters):
            timer("split")
            r.split(high)
            timer("collapse")
            live = r.V
            while True:
                n = r.collapse_round(low, high, live)
                live -= n
                if n == 0:
                    break
            r.compact()
            timer("flip")
            while r.flip_round():
                pass
            if not project:
                timer("bvh")
                target = MeshDistance(*r.mesh())
            timer("relax")
            r.relax(target)
        timer.close()
        vo, fo = r.mesh()
        out = vo.clone(), fo.to(f.dtype, copy=True)      # copies: the work buffers have room for a split
        return (*out, r.features()) if return_feature else out
