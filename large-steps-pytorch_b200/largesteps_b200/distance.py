"""Point-to-mesh distances and the mesh Hausdorff distance on the GPU: libigl's `point_mesh_squared_distance` and `hausdorff`,
which the reference's figure scripts rank their runs by (figures/comparison/generate_data.py:78-88).

    MeshDistance(verts, faces)                 one mesh's BVH, built on the device (csrc/ls_distance.cu)
      .squared_distance(P) -> (sqrD, I, C)     asynchronous, device tensors
      .hausdorff(VA, FA) -> float              another mesh scored against this one
    point_mesh_squared_distance(P, V, F)       igl.point_mesh_squared_distance
    hausdorff(VA, FA, VB, FB) -> float         igl.hausdorff

sqrD[q] (float64) is the squared distance from row q of P to the nearest point of the faces, I[q] (int64) that face (the lowest
index among faces at an equal float64 distance) and C[q] (float64, 3) the point.  The closest point on a face is computed in
float64 from the float32 corners.  hausdorff(A, B) = sqrt(max(max_a sqrD(a, B), max_b sqrD(b, A))) with a and b over every
row of VA and VB, unreferenced vertices included: symmetric, and NaN if any coordinate is.  A row of P with a NaN gives NaN
and -1.

    chamfer(VA, FA, VB, FB) -> 0-dim tensor    mean_a sqrD(a, B) + mean_b sqrD(b, A), differentiable w.r.t. VA and VB
    MeshDistance(VB, FB).chamfer(VA, FA)       the same against a fixed target, differentiable w.r.t. VA

Gradients.  sqrD is differentiable (I and C are not): w.r.t. P and V in point_mesh_squared_distance, w.r.t. P alone in
MeshDistance.squared_distance, whose BVH is a snapshot.  With C = C[q] on face I[q] = (a, b, c) and beta its weights on the
corners (from the same Voronoi region as the forward: face, edge, vertex, or the segment a degenerate face was reduced to),
    d sqrD[q] / d P[q] = 2 (P[q] - C),    d sqrD[q] / d V[k] = -2 beta_k (P[q] - C) for each corner k of face I[q]
(Danskin's theorem: only the face that attains the minimum counts).  A row answered with face -1 gets NaN in its row of the
gradient w.r.t. P and adds nothing w.r.t. V; its sqrD, and so any loss built on it, is NaN too.  The backward
(ls_distance_grad_f32) sums in float64 without atomics and rounds once to float32: bitwise reproducible.  Only the gradients
autograd asks for are computed.  The chamfer loss is the mean-square counterpart of the Hausdorff maximum; a loop that fits
a mesh to a fixed target calls MeshDistance(target_v, target_f).chamfer(v, f) every step and never synchronises.

Batches.  B meshes packed as by batch.pack_meshes (verts (sum V_b, 3), faces (sum F_b, 3) with mesh b's indices shifted by
vert_offsets[b], and vert_offsets / face_offsets of B + 1 entries as int64 tensors or sequences of ints) are scored in one
BVH build, one query launch per direction and one backward, whatever B:

    MeshDistanceBatch(verts, faces, vert_offsets, face_offsets)          the BVHs of B meshes, one forest
      .squared_distance(P, point_offsets) -> (sqrD, I, C)               rows point_offsets[b]:point_offsets[b+1] against mesh b
      .hausdorff(VA, FA, vo_A, fo_A) -> (B,) float64                    entry b: hausdorff(A_b, this_b)
      .chamfer(VA, FA, vo_A, fo_A) -> (B,) float64                      entry b: MeshDistance(this_b).chamfer(A_b)
    point_mesh_squared_distance_batch(P, point_offsets, V, F, vo, fo)
    hausdorff_batch(VA, FA, vo_A, fo_A, VB, FB, vo_B, fo_B) -> (B,) float64
    chamfer_batch(VA, FA, vo_A, fo_A, VB, FB, vo_B, fo_B) -> (B,) float64  differentiable w.r.t. VA and VB

Each entry is bitwise its single-mesh counterpart (sqrD, C, I minus the face offset, hausdorff), or, for the chamfer means,
the same sums in another fixed order; the chamfer gradients are bitwise the single-mesh ones.  A side holding one mesh is
paired with every mesh of the other side (T iterates of a run scored against one target: the target's BVH is built once).
The constructor and point_mesh_squared_distance_batch check the faces against their meshes' vertex ranges with one read-back
per faces tensor not seen before, and raise IndexError for a face outside its mesh's range.  The hausdorff and chamfer calls
never synchronise: such a face, on a side they build, makes that mesh's entry NaN, and check() raises IndexError.
"""
import ctypes
import math

import torch

from . import _native as N
from .meshops import _check_face_ranges, _check_mesh, _check_offsets, _offsets


def _workspace(n, dev):
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_distance_query_workspace_bytes(n, ctypes.byref(nb)), "ls_distance_query_workspace_bytes")
    return torch.empty(nb.value, dtype=torch.uint8, device=dev)


def _workspace_batch(n, S, dev):
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_distance_query_batch_workspace_bytes(n, S, ctypes.byref(nb)), "ls_distance_query_batch_workspace_bytes")
    return torch.empty(nb.value, dtype=torch.uint8, device=dev)


def _wants_grad(*ts):
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in ts)


class MeshDistance:
    """The BVH of one triangle mesh: float32 verts (V, 3) and int32 / int64 faces (F, 3), F >= 1, on one CUDA device.
    The BVH holds its own copy of the triangles and of verts, so later changes to verts or faces do not reach it."""

    def __init__(self, verts, faces, _defer_index_check=False):
        _check_mesh(verts, faces)
        F, V = faces.shape[0], verts.shape[0]
        if F == 0:
            raise ValueError("the mesh has no faces")
        fc = faces.contiguous()
        self._bad = None
        if _defer_index_check:
            # no read-back: out-of-range indices are replaced by 0 before anything reads through them, the losses built on
            # this mesh are NaN and check() raises IndexError
            out = (fc < 0) | (fc >= V)
            self._bad = out.any()
            fc = fc.masked_fill(out, 0)
        elif bool(((fc < 0) | (fc >= V)).any()):
            raise IndexError(f"a face indexes a vertex outside [0, {V})")
        self.device = verts.device
        self.verts = verts.detach().clone(memory_format=torch.contiguous_format)   # B's query points in hausdorff
        self.F = F
        self._faces = fc                                                            # the gradient w.r.t. the corners
        lib = N.lib()
        with torch.cuda.device(self.device):
            nb = ctypes.c_size_t(0)
            N.check(lib.ls_distance_bvh_bytes(F, ctypes.byref(nb)), "ls_distance_bvh_bytes")
            self._bvh = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
            N.check(lib.ls_distance_bvh_build(N.ptr(self.verts), V, N.ptr(fc), fc.element_size(), F, N.ptr(self._bvh), nb.value,
                                              N.stream_ptr(self.device)), "ls_distance_bvh_build")
        self._last = ()
        self._last_bad = ()

    def _points(self, P):
        N.require_cuda(P, "P")
        if P.dim() != 2 or P.shape[1] != 3:
            raise ValueError(f"P must have shape (n, 3), got {tuple(P.shape)}")
        if P.dtype != torch.float32:
            raise TypeError(f"P must be float32, got {P.dtype}")
        if P.device != self.device:
            raise RuntimeError("P and the mesh must live on the same device")
        return P.detach().contiguous()

    def _query(self, P, ws, max_mode, outputs=True):
        n = P.shape[0]
        dev = self.device
        sqrD = torch.empty(n, dtype=torch.float64, device=dev) if outputs else None
        I = torch.empty(n, dtype=torch.int64, device=dev) if outputs else None
        C = torch.empty((n, 3), dtype=torch.float64, device=dev) if outputs else None
        with torch.cuda.device(dev):
            N.check(N.lib().ls_distance_query(N.ptr(self._bvh), self.F, N.ptr(P), n, N.ptr(sqrD), N.ptr(I), N.ptr(C), max_mode,
                                              N.ptr(ws), ws.numel(), N.stream_ptr(dev)), "ls_distance_query")
        return sqrD, I, C

    def _distances(self, P, V, ws):
        """(sqrD, I, C) of the rows of P, with sqrD differentiable w.r.t. P and V (this mesh's vertices, or None) when
        autograd asks for it; otherwise the plain query."""
        Pd = self._points(P)
        if _wants_grad(P, V):
            return _SquaredDistance.apply(P, V, self, lambda Pc: self._query(Pc, ws, 0))
        return self._query(Pd, ws, 0)

    def squared_distance(self, P):
        """(sqrD (n,) float64, I (n,) int64, C (n, 3) float64) for the rows of P (n, 3) float32.  Asynchronous.  sqrD is
        differentiable w.r.t. P (the BVH is a snapshot, so its vertices get no gradient)."""
        ws = _workspace(self._points(P).shape[0], self.device)
        self._last, self._last_bad = (ws,), ()
        return self._distances(P, None, ws)

    def check(self):
        """Synchronises; raises RuntimeError if the last squared_distance or chamfer call overflowed its traversal stack, and
        IndexError if the mesh a chamfer call built indexes a vertex outside its range."""
        for bad in self._last_bad:
            if bool(bad):
                raise IndexError("a face of the chamfer call's mesh indexes a vertex outside its range")
        for ws in self._last:
            with torch.cuda.device(self.device):
                N.check(N.lib().ls_distance_result(N.ptr(ws), None, N.stream_ptr(self.device)), "ls_distance_result")

    def hausdorff(self, VA, FA):
        """igl.hausdorff(VA, FA, VB, FB) with (VB, FB) this mesh: builds the BVH of A, runs both directions on the device and
        reads the result back once."""
        A = MeshDistance(VA, FA)
        PA = self._points(A.verts)
        ws = _workspace(max(PA.shape[0], self.verts.shape[0]), self.device)
        self._query(PA, ws, 1, outputs=False)
        A._query(self.verts, ws, 2, outputs=False)
        out = ctypes.c_double(0.0)
        with torch.cuda.device(self.device):
            N.check(N.lib().ls_distance_result(N.ptr(ws), ctypes.byref(out), N.stream_ptr(self.device)), "ls_distance_result")
        return math.sqrt(out.value)

    def chamfer(self, VA, FA):
        """chamfer(VA, FA, VB, FB) with (VB, FB) this mesh, its BVH reused: mean_a sqrD(a, B) + mean_b sqrD(b, A) as a 0-dim
        float64 tensor, differentiable w.r.t. VA through both terms (B's vertices get no gradient).  Does not synchronise;
        check() covers both queries."""
        A = MeshDistance(VA, FA, _defer_index_check=True)
        wa, wb = _workspace(VA.shape[0], self.device), _workspace(self.verts.shape[0], self.device)
        self._last, self._last_bad = (wa, wb), (A._bad,)
        loss = self._distances(VA, None, wa)[0].mean() + A._distances(self.verts, VA, wb)[0].mean()
        return loss.masked_fill(A._bad, math.nan)


class _SquaredDistance(torch.autograd.Function):
    """sqrD of md's query of P (query(P) -> (sqrD, I, C)), differentiable w.r.t. P and V (md's vertices as a tensor of the
    graph, or None).  md is a MeshDistance or a MeshDistanceBatch: the backward runs on the packed rows as they are."""

    @staticmethod
    def forward(ctx, P, V, md, query):
        sqrD, I, C = query(P.detach().contiguous())
        ctx.mark_non_differentiable(I, C)
        ctx.save_for_backward(P, V, I, C)     # an in-place change to P or V before backward raises
        ctx.md = md
        return sqrD, I, C

    @staticmethod
    def backward(ctx, gsq, _gI, _gC):
        P, V, I, C = ctx.saved_tensors
        md = ctx.md
        need_p, need_v = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        dev, n = md.device, P.shape[0]
        Pc = P.detach().contiguous()
        g = gsq.to(torch.float64).contiguous()
        gP = torch.empty((n, 3), dtype=torch.float32, device=dev) if need_p else None
        gV = Vc = ws = None
        nb = ctypes.c_size_t(0)
        nV = md.verts.shape[0]
        fc = md._faces
        with torch.cuda.device(dev):
            if need_v:
                Vc = V.detach().contiguous()
                gV = torch.empty((nV, 3), dtype=torch.float32, device=dev)
                N.check(N.lib().ls_distance_grad_workspace_bytes(n, md.F, nV, ctypes.byref(nb)), "ls_distance_grad_workspace_bytes")
                ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
            if need_p or need_v:
                N.check(N.lib().ls_distance_grad_f32(N.ptr(Pc), n, N.ptr(Vc), nV, N.ptr(fc), fc.element_size(), md.F, N.ptr(I),
                                                     N.ptr(C), N.ptr(g), N.ptr(gP), N.ptr(gV), N.ptr(ws), nb.value,
                                                     N.stream_ptr(dev)), "ls_distance_grad_f32")
        return gP, gV, None, None


def point_mesh_squared_distance(P, V, F):
    """igl.point_mesh_squared_distance(P, V, F) -> (sqrD, I, C) as CUDA tensors (float64, int64, float64).  Synchronises.
    sqrD is differentiable w.r.t. P and V when either requires grad (I and C are not)."""
    md = MeshDistance(V, F)
    ws = _workspace(md._points(P).shape[0], md.device)
    md._last = (ws,)
    out = md._distances(P, V, ws)
    md.check()
    return out


def hausdorff(VA, FA, VB, FB):
    """igl.hausdorff(VA, FA, VB, FB): the Hausdorff distance between the vertex sets and the surfaces, as a Python float."""
    return MeshDistance(VB, FB).hausdorff(VA, FA)


def chamfer(VA, FA, VB, FB):
    """mean_a sqrD(a, B) + mean_b sqrD(b, A) over every row a of VA and b of VB (unreferenced vertices included, the sets
    hausdorff takes its maximum over) as a 0-dim float64 tensor, differentiable w.r.t. VA and VB: the first term reaches VA
    as query points and VB as mesh corners, the second the reverse.  Does not synchronise; NaN if a coordinate is NaN or a
    face indexes a vertex out of range."""
    A = MeshDistance(VA, FA, _defer_index_check=True)
    B = MeshDistance(VB, FB, _defer_index_check=True)
    wa, wb = _workspace(VA.shape[0], A.device), _workspace(VB.shape[0], A.device)
    loss = B._distances(VA, VB, wa)[0].mean() + A._distances(VB, VA, wb)[0].mean()
    return loss.masked_fill(A._bad | B._bad, math.nan)


# ---- packed batches -------------------------------------------------------------------------------------------------------
class MeshDistanceBatch:
    """The BVHs of B packed triangle meshes, built in one call: float32 verts (sum V_b, 3), int32 / int64 faces (sum F_b, 3)
    with mesh b's indices shifted by vert_offsets[b], and B + 1 vert_offsets / face_offsets (int64 tensors or sequences of
    ints; pack_meshes(...)[:4] fits).  Every mesh needs a face.  Like MeshDistance, it holds a snapshot of the triangles."""

    def __init__(self, verts, faces, vert_offsets, face_offsets, _defer_index_check=False):
        _check_mesh(verts, faces)
        dev = verts.device
        V, F = verts.shape[0], faces.shape[0]
        vo, vo_dev = _offsets(vert_offsets, dev, "vert_offsets")
        fo, fo_dev = _offsets(face_offsets, dev, "face_offsets")
        B = _check_batch(vo, fo, V, F)
        fc = faces.contiguous()
        self._bad = None
        if _defer_index_check:
            # no read-back: a face outside its mesh's vertex range is pointed at the mesh's first vertex (the last vertex of
            # the batch if the mesh has none, as the last mesh may), that mesh's results are NaN and check() raises IndexError
            mesh = torch.repeat_interleave(torch.arange(B, device=dev), fo_dev.diff(), output_size=F)
            lo, hi = vo_dev[mesh, None], vo_dev[mesh + 1, None]
            out = (fc < lo) | (fc >= hi)
            nbad = torch.nn.functional.pad(out.any(1).cumsum(0), (1, 0))
            self._bad = nbad[fo_dev[1:]] > nbad[fo_dev[:-1]]
            fc = torch.where(out, lo.clamp(max=V - 1).to(fc.dtype), fc)
        else:
            _check_face_ranges(faces, vo, vo_dev, fo)
        self.device, self.B, self.F = dev, B, F
        self.verts = verts.detach().clone(memory_format=torch.contiguous_format)
        self.vert_offsets, self.face_offsets = (vo, vo_dev), (fo, fo_dev)
        self._faces = fc
        lib = N.lib()
        with torch.cuda.device(dev):
            nb = ctypes.c_size_t(0)
            N.check(lib.ls_distance_bvh_batch_bytes(F, B, ctypes.byref(nb)), "ls_distance_bvh_batch_bytes")
            self._bvh = torch.empty(nb.value, dtype=torch.uint8, device=dev)
            N.check(lib.ls_distance_bvh_batch_build(N.ptr(self.verts), V, N.ptr(fc), fc.element_size(), F, B, N.ptr(fo_dev),
                                                    N.ptr(self._bvh), nb.value, N.stream_ptr(dev)), "ls_distance_bvh_batch_build")
        self._last = ()
        self._last_bad = ()

    def _points(self, P, point_offsets):
        MeshDistance._points(self, P)
        n = P.shape[0]
        po, po_dev = _offsets(point_offsets, self.device, "point_offsets")
        _check_points(po, n, self.B)
        return po_dev

    def _query(self, P, po_dev, ws, max_mode, maxout=None, outputs=True):
        n, S = P.shape[0], po_dev.shape[0] - 1
        dev = self.device
        sqrD = torch.empty(n, dtype=torch.float64, device=dev) if outputs else None
        I = torch.empty(n, dtype=torch.int64, device=dev) if outputs else None
        C = torch.empty((n, 3), dtype=torch.float64, device=dev) if outputs else None
        with torch.cuda.device(dev):
            N.check(N.lib().ls_distance_query_batch(N.ptr(self._bvh), self.F, self.B, N.ptr(P), n, S, N.ptr(po_dev), N.ptr(sqrD),
                                                    N.ptr(I), N.ptr(C), N.ptr(maxout), max_mode, N.ptr(ws), ws.numel(),
                                                    N.stream_ptr(dev)), "ls_distance_query_batch")
        return sqrD, I, C

    def _distances(self, P, po_dev, V, ws):
        Pd = P.detach().contiguous()
        if _wants_grad(P, V):
            return _SquaredDistance.apply(P, V, self, lambda Pc: self._query(Pc, po_dev, ws, 0))
        return self._query(Pd, po_dev, ws, 0)

    def squared_distance(self, P, point_offsets):
        """(sqrD (n,) float64, I (n,) int64 packed face index, C (n, 3) float64) for the rows of P (n, 3) float32, rows
        point_offsets[b]:point_offsets[b+1] against mesh b (against the one mesh, for any number of segments, when B == 1).
        Asynchronous; sqrD is differentiable w.r.t. P."""
        po_dev = self._points(P, point_offsets)
        ws = _workspace_batch(P.shape[0], po_dev.shape[0] - 1, self.device)
        self._last, self._last_bad = (ws,), ()
        return self._distances(P, po_dev, None, ws)

    check = MeshDistance.check

    def hausdorff(self, VA, FA, vert_offsets_A, face_offsets_A):
        """(B,) float64 CUDA tensor, entry b = hausdorff(A_b, this_b): one BVH build for A, one query launch per direction.
        Does not synchronise; a face of A_b outside its vertex range makes entry b NaN, and check() raises IndexError (as it
        does for a traversal stack overflow)."""
        A = MeshDistanceBatch(VA, FA, vert_offsets_A, face_offsets_A, _defer_index_check=True)
        T = _pair(A.B, self.B)
        PA, poA = _tiled(A.verts, A.vert_offsets, T)
        PB, poB = _tiled(self.verts, self.vert_offsets, T)
        self._points(PA, poA[0])
        out = torch.empty(T, dtype=torch.float64, device=self.device)
        ws = _workspace_batch(max(PA.shape[0], PB.shape[0]), T, self.device)
        self._query(PA, poA[1], ws, 1, out, outputs=False)
        A._query(PB, poB[1], ws, 2, out, outputs=False)
        bad = A._bad.expand(T) if self._bad is None else A._bad.expand(T) | self._bad.expand(T)
        self._last, self._last_bad = (ws,), (bad.any(),)
        return out.sqrt().masked_fill(bad, math.nan)

    def chamfer(self, VA, FA, vert_offsets_A, face_offsets_A):
        """(B,) float64, entry b = MeshDistance(this_b).chamfer(A_b), differentiable w.r.t. VA.  Does not synchronise; a face of
        A_b outside its vertex range makes entry b NaN, and check() raises IndexError."""
        A = MeshDistanceBatch(VA, FA, vert_offsets_A, face_offsets_A, _defer_index_check=True)
        T = _pair(A.B, self.B)
        PA, poA = _tiled(VA, A.vert_offsets, T)
        PB, poB = _tiled(self.verts, self.vert_offsets, T)
        self._points(PA, poA[0])
        wa, wb = _workspace_batch(PA.shape[0], T, self.device), _workspace_batch(PB.shape[0], T, self.device)
        self._last, self._last_bad = (wa, wb), (A._bad.any(),)
        loss = _SegmentMean.apply(self._distances(PA, poA[1], None, wa)[0], poA[1]) + \
            _SegmentMean.apply(A._distances(PB, poB[1], VA, wb)[0], poB[1])
        return loss.masked_fill(A._bad.expand(T), math.nan)


def _check_batch(vo, fo, V, F):
    """B, from the host offsets of a packed batch of V vertices and F faces; every mesh needs a face."""
    _check_offsets(vo, fo, V, F)
    empty = [b for b, (a, e) in enumerate(zip(fo[:-1], fo[1:])) if a == e]
    if empty:
        raise ValueError(f"mesh {empty[0]} of the batch has no faces")
    return len(fo) - 1


def _check_points(po, n, B):
    """point_offsets of n rows against a batch of B meshes: one segment per mesh, or any number against one mesh."""
    _check_offsets(po, po, n, n, names=("point_offsets", "point_offsets"))
    if len(po) - 1 != B and B != 1:
        raise ValueError(f"point_offsets holds {len(po) - 1} segments for a batch of {B} meshes")


def _pair(BA, BB):
    """The number of pairs of two sides of BA and BB meshes: equal counts, or one side holding one mesh."""
    if BA != BB and BA != 1 and BB != 1:
        raise ValueError(f"the two sides hold {BA} and {BB} meshes: they must hold as many, or one side a single mesh")
    return max(BA, BB)


def _tiled(V, offsets, T):
    """V's rows as T point segments, with their (host, device) offsets: V itself if it holds T meshes, or its one mesh T times."""
    if len(offsets[0]) - 1 == T:
        return V, offsets
    n = V.shape[0]
    return V.repeat(T, 1), _offsets(range(0, n * T + 1, n) if n else [0] * (T + 1), V.device, "offsets")


class _SegmentMean(torch.autograd.Function):
    """The mean of each segment [off[s], off[s+1]) of x (float64): a fixed-order sum on the device (ls_distance_segment_sum_f64)
    times 1 / count.  The backward hands each row g[s] * (1 / count): torch's mean backward divides by the count as a CPU
    scalar, which its CUDA division applies as a multiplication by the reciprocal, so each mesh's rows get bitwise the gradient
    the mean of that mesh alone gives them, for any upstream g."""

    @staticmethod
    def forward(ctx, x, off_dev):
        S, n = off_dev.shape[0] - 1, x.shape[0]
        xc = x.detach().contiguous()
        sums = torch.empty(S, dtype=torch.float64, device=x.device)
        with torch.cuda.device(x.device):
            N.check(N.lib().ls_distance_segment_sum_f64(N.ptr(xc), n, S, N.ptr(off_dev), N.ptr(sums), N.stream_ptr(x.device)),
                    "ls_distance_segment_sum_f64")
        counts = off_dev.diff()
        inv = 1.0 / counts.to(torch.float64)
        ctx.save_for_backward(counts, inv)
        ctx.n = n
        return sums * inv

    @staticmethod
    def backward(ctx, g):
        counts, inv = ctx.saved_tensors
        return torch.repeat_interleave(g * inv, counts, output_size=ctx.n), None


def point_mesh_squared_distance_batch(P, point_offsets, V, F, vert_offsets, face_offsets):
    """point_mesh_squared_distance of each mesh of a packed batch: rows point_offsets[b]:point_offsets[b+1] of P against mesh b.
    (sqrD, I, C) as CUDA tensors, I the packed face index.  Synchronises.  sqrD is differentiable w.r.t. P and V."""
    md = MeshDistanceBatch(V, F, vert_offsets, face_offsets)
    po_dev = md._points(P, point_offsets)
    ws = _workspace_batch(P.shape[0], po_dev.shape[0] - 1, md.device)
    md._last = (ws,)
    out = md._distances(P, po_dev, V, ws)
    md.check()
    return out


def hausdorff_batch(VA, FA, vert_offsets_A, face_offsets_A, VB, FB, vert_offsets_B, face_offsets_B):
    """(B,) float64 CUDA tensor, entry b = hausdorff(A_b, B_b), a side of one mesh paired with every mesh of the other.
    Does not synchronise; NaN in entry b if a coordinate of the pair is NaN or a face indexes outside its mesh."""
    return MeshDistanceBatch(VB, FB, vert_offsets_B, face_offsets_B, _defer_index_check=True).hausdorff(
        VA, FA, vert_offsets_A, face_offsets_A)


def chamfer_batch(VA, FA, vert_offsets_A, face_offsets_A, VB, FB, vert_offsets_B, face_offsets_B):
    """(B,) float64, entry b = chamfer(A_b, B_b), a side of one mesh paired with every mesh of the other; differentiable w.r.t.
    VA and VB.  Does not synchronise; NaN in entry b if a coordinate of the pair is NaN or a face indexes outside its mesh."""
    A = MeshDistanceBatch(VA, FA, vert_offsets_A, face_offsets_A, _defer_index_check=True)
    B = MeshDistanceBatch(VB, FB, vert_offsets_B, face_offsets_B, _defer_index_check=True)
    T = _pair(A.B, B.B)
    PA, poA = _tiled(VA, A.vert_offsets, T)
    PB, poB = _tiled(VB, B.vert_offsets, T)
    B._points(PA, poA[0])
    A._points(PB, poB[0])
    wa, wb = _workspace_batch(PA.shape[0], T, A.device), _workspace_batch(PB.shape[0], T, A.device)
    loss = _SegmentMean.apply(B._distances(PA, poA[1], VB, wa)[0], poA[1]) + \
        _SegmentMean.apply(A._distances(PB, poB[1], VA, wb)[0], poB[1])
    return loss.masked_fill(A._bad.expand(T) | B._bad.expand(T), math.nan)
