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
"""
import ctypes
import math

import torch

from . import _native as N
from .meshops import _check_mesh


def _workspace(n, dev):
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_distance_query_workspace_bytes(n, ctypes.byref(nb)), "ls_distance_query_workspace_bytes")
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
            return _SquaredDistance.apply(P, V, self, ws)
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
    """sqrD of md's query of P, differentiable w.r.t. P and V (md's vertices as a tensor of the graph, or None)."""

    @staticmethod
    def forward(ctx, P, V, md, ws):
        sqrD, I, C = md._query(P.detach().contiguous(), ws, 0)
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
