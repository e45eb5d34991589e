"""CPU: packing meshes (batch.pack_meshes), the offset checks of the packed vertex normals, and the host-side argument checks
of the multi-tensor AdamUniform step and the packed vertex-normal entry points."""
import ctypes

import numpy as np
import pytest
import torch

import largesteps_b200._native as N
from largesteps_b200 import batch, meshops, workloads


def mesh(level, idx_dtype=torch.int64):
    v, f = workloads.icosphere(level)
    return torch.from_numpy(v), torch.from_numpy(f).to(idx_dtype)


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64])
def test_pack_meshes_offsets_and_shifts(idx_dtype):
    ms = [mesh(1, idx_dtype), mesh(2, idx_dtype), mesh(1, idx_dtype)]
    p = batch.pack_meshes([v for v, _ in ms], [f for _, f in ms])
    V = [v.shape[0] for v, _ in ms]
    F = [f.shape[0] for _, f in ms]
    assert p.vert_offsets_host == (0, V[0], V[0] + V[1], sum(V))
    assert p.face_offsets_host == (0, F[0], F[0] + F[1], sum(F))
    assert p.vert_offsets.dtype == torch.int64 and p.vert_offsets.tolist() == list(p.vert_offsets_host)
    assert p.face_offsets.dtype == torch.int64 and p.face_offsets.tolist() == list(p.face_offsets_host)
    assert p.faces.dtype == idx_dtype and p.faces.shape == (sum(F), 3)
    assert torch.equal(p.verts, torch.cat([v for v, _ in ms]))
    for i, (v, f) in enumerate(ms):
        fo, vo = p.face_offsets_host, p.vert_offsets_host
        assert torch.equal(p.faces[fo[i]:fo[i + 1]], f + vo[i])
    # verts stay differentiable through the packing
    vs = [v.clone().requires_grad_(True) for v, _ in ms]
    batch.pack_meshes(vs, [f for _, f in ms]).verts.sum().backward()
    assert all(torch.equal(v.grad, torch.ones_like(v)) for v in vs)


def test_pack_meshes_rejects_bad_input():
    (v1, f1), (v2, f2) = mesh(1), mesh(1)
    with pytest.raises(ValueError, match="at least one"):
        batch.pack_meshes([], [])
    with pytest.raises(ValueError, match="face arrays"):
        batch.pack_meshes([v1, v2], [f1])
    with pytest.raises(TypeError, match="int32"):
        batch.pack_meshes([v1, v2], [f1, f2.to(torch.int32)])
    with pytest.raises(ValueError, match=r"\(V, 3\)"):
        batch.pack_meshes([v1[:, :2]], [f1])


def test_offset_tensors_are_read_once_and_cached():
    (v1, f1), (v2, f2) = mesh(1), mesh(2)
    p = batch.pack_meshes([v1, v2], [f1, f2])
    host, dev_t = meshops._offsets(p.vert_offsets, "cpu", "vert_offsets")
    assert host == p.vert_offsets_host and dev_t is p.vert_offsets
    host, _ = meshops._offsets([0, 3, 5], "cpu", "vert_offsets")
    assert host == (0, 3, 5)


def test_offset_validation():
    meshops._check_offsets((0, 4, 9), (0, 2, 6), 9, 6)
    meshops._check_offsets((0, 4, 4, 9), (0, 2, 2, 6), 9, 6)          # an empty mesh is fine
    with pytest.raises(ValueError, match="non-decreasing"):
        meshops._check_offsets((0, 5, 4, 9), (0, 2, 3, 6), 9, 6)
    with pytest.raises(ValueError, match="end at 9"):
        meshops._check_offsets((0, 4, 8), (0, 2, 6), 9, 6)
    with pytest.raises(ValueError, match="end at 6"):
        meshops._check_offsets((0, 4, 9), (0, 2, 7), 9, 6)
    with pytest.raises(ValueError, match="start at 0"):
        meshops._check_offsets((1, 4, 9), (0, 2, 6), 9, 6)
    with pytest.raises(ValueError, match="B \\+ 1"):
        meshops._check_offsets((0, 4, 9), (0, 6), 9, 6)
    with pytest.raises(ValueError, match="B \\+ 1"):
        meshops._check_offsets((0,), (0,), 0, 0)


def test_vertex_normals_cpu_tensors_raise():
    v, f = mesh(1)
    p = batch.pack_meshes([v], [f])
    fn = torch.zeros((3, f.shape[0]))
    with pytest.raises(RuntimeError, match="CUDA"):
        meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, p.vert_offsets, p.face_offsets)


def i64(*xs):
    return (ctypes.c_int64 * len(xs))(*xs)


def test_vertex_normals_batch_entry_points_validate_on_the_host():
    lib = N.lib()
    nb = ctypes.c_size_t(0)
    assert lib.ls_vertex_normals_batch_scratch_bytes(1, ctypes.byref(nb)) == N.LS_OK
    one = nb.value
    assert lib.ls_vertex_normals_batch_scratch_bytes(64, ctypes.byref(nb)) == N.LS_OK and nb.value > 32 * one
    assert lib.ls_vertex_normals_batch_scratch_bytes(0, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    assert lib.ls_vertex_normals_batch_scratch_bytes(65536, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    assert lib.ls_vertex_normals_batch_scratch_bytes(4, None) == N.LS_ERR_BAD_ARG
    lib.ls_vertex_normals_batch_scratch_bytes(2, ctypes.byref(nb))
    need = nb.value

    def fwd(vo, fo, V=9, F=6, B=2, scratch_bytes=need, idx_bytes=4):
        return lib.ls_vertex_normals_batch_f32(None, None, idx_bytes, F, V, B, None, None, vo, fo, None, None, None, None,
                                               None, None, None, scratch_bytes, None)

    def bwd(vo, fo, V=9, F=6, B=2, scratch_bytes=need):
        return lib.ls_vertex_normals_batch_bwd_f32(None, None, 4, F, V, B, None, None, vo, fo, None, None, None, None, None,
                                                   None, None, None, None, None, scratch_bytes, None)

    for call in (fwd, bwd):
        assert call(i64(0, 4, 9), i64(0, 2, 6)) == N.LS_ERR_BAD_ARG and "NULL pointer" in N.last_error()
        assert call(i64(0, 5, 4), i64(0, 2, 6), V=4) == N.LS_ERR_BAD_ARG and "non-decreasing" in N.last_error()
        assert call(i64(0, 4, 8), i64(0, 2, 6)) == N.LS_ERR_BAD_ARG and "end at V and F" in N.last_error()
        assert call(i64(0, 4, 9), i64(0, 2, 5)) == N.LS_ERR_BAD_ARG and "end at V and F" in N.last_error()
        assert call(i64(1, 4, 9), i64(0, 2, 6)) == N.LS_ERR_BAD_ARG and "start at 0" in N.last_error()
        assert call(None, i64(0, 2, 6)) == N.LS_ERR_BAD_ARG and "host offsets" in N.last_error()
        assert call(i64(0, 4, 9), i64(0, 2, 6), scratch_bytes=need - 1) == N.LS_ERR_BAD_ARG and "scratch" in N.last_error()
        assert call(i64(0, 9), i64(0, 6), B=0) == N.LS_ERR_BAD_ARG
    assert fwd(i64(0, 4, 9), i64(0, 2, 6), idx_bytes=2) == N.LS_ERR_BAD_ARG


def test_adam_tensor_table_layout():
    class T(ctypes.Structure):      # ls_adam_tensor of include/largesteps_b200.h
        _fields_ = [("param", ctypes.c_void_p), ("grad", ctypes.c_void_p), ("g1", ctypes.c_void_p), ("g2", ctypes.c_void_p),
                    ("n", ctypes.c_int64)] + [(k, ctypes.c_float) for k in
                                              ("lr", "beta1", "beta2", "one_minus_beta1", "one_minus_beta2", "c1", "c2")]
    assert N.ADAM_TENSOR.itemsize == ctypes.sizeof(T) == 72
    for name, (_, off) in N.ADAM_TENSOR.fields.items():
        assert getattr(T, name).offset == off, name


def test_adam_multi_entry_point_validates_on_the_host():
    lib = N.lib()
    tab = np.zeros(3, dtype=N.ADAM_TENSOR)
    p = ctypes.c_void_p(tab.ctypes.data)
    dummy = ctypes.c_void_p(16)      # never dereferenced: the checks fail first
    assert lib.ls_adam_uniform_step_multi(None, 0, None, 0, None) == N.LS_OK          # nothing to do
    assert lib.ls_adam_uniform_step_multi(p, -1, dummy, 64, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_adam_uniform_step_multi(None, 3, dummy, 64, None) == N.LS_ERR_BAD_ARG and "NULL" in N.last_error()
    assert lib.ls_adam_uniform_step_multi(p, 3, None, 64, None) == N.LS_ERR_BAD_ARG and "NULL" in N.last_error()
    assert lib.ls_adam_uniform_step_multi(p, 3, dummy, 23, None) == N.LS_ERR_BAD_ARG and "8 n" in N.last_error()
    tab["n"] = [0, 5, 0]
    assert lib.ls_adam_uniform_step_multi(p, 3, dummy, 24, None) == N.LS_ERR_BAD_ARG and "NULL tensor" in N.last_error()
    tab["n"] = [0, -5, 0]
    assert lib.ls_adam_uniform_step_multi(p, 3, dummy, 24, None) == N.LS_ERR_BAD_ARG and "negative" in N.last_error()
