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


class MeshDistance:
    """The BVH of one triangle mesh: float32 verts (V, 3) and int32 / int64 faces (F, 3), F >= 1, on one CUDA device.
    The BVH holds its own copy of the triangles and of verts, so later changes to verts or faces do not reach it."""

    def __init__(self, verts, faces):
        _check_mesh(verts, faces)
        F, V = faces.shape[0], verts.shape[0]
        if F == 0:
            raise ValueError("the mesh has no faces")
        fc = faces.contiguous()
        if bool(((fc < 0) | (fc >= V)).any()):
            raise IndexError(f"a face indexes a vertex outside [0, {V})")
        self.device = verts.device
        self.verts = verts.detach().clone(memory_format=torch.contiguous_format)   # B's query points in hausdorff
        self.F = F
        lib = N.lib()
        with torch.cuda.device(self.device):
            nb = ctypes.c_size_t(0)
            N.check(lib.ls_distance_bvh_bytes(F, ctypes.byref(nb)), "ls_distance_bvh_bytes")
            self._bvh = torch.empty(nb.value, dtype=torch.uint8, device=self.device)
            N.check(lib.ls_distance_bvh_build(N.ptr(self.verts), V, N.ptr(fc), fc.element_size(), F, N.ptr(self._bvh), nb.value,
                                              N.stream_ptr(self.device)), "ls_distance_bvh_build")
        self._last = None

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

    def squared_distance(self, P):
        """(sqrD (n,) float64, I (n,) int64, C (n, 3) float64) for the rows of P (n, 3) float32.  Asynchronous."""
        P = self._points(P)
        ws = _workspace(P.shape[0], self.device)
        self._last = ws
        return self._query(P, ws, 0)

    def check(self):
        """Synchronises; raises RuntimeError if the last squared_distance call overflowed its traversal stack."""
        if self._last is not None:
            with torch.cuda.device(self.device):
                N.check(N.lib().ls_distance_result(N.ptr(self._last), None, N.stream_ptr(self.device)), "ls_distance_result")

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


def point_mesh_squared_distance(P, V, F):
    """igl.point_mesh_squared_distance(P, V, F) -> (sqrD, I, C) as CUDA tensors (float64, int64, float64).  Synchronises."""
    md = MeshDistance(V, F)
    out = md.squared_distance(P)
    md.check()
    return out


def hausdorff(VA, FA, VB, FB):
    """igl.hausdorff(VA, FA, VB, FB): the Hausdorff distance between the vertex sets and the surfaces, as a Python float."""
    return MeshDistance(VB, FB).hausdorff(VA, FA)
