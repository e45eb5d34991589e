"""CPU: the argument handling of the batched distances (largesteps_b200.distance, csrc/ls_distance.cu) without a GPU: the
offsets' length, start, end and order, a mesh without faces, mismatched batch sizes and the one broadcast rule, CPU tensors,
and the C entry points' host-side checks, which fail before any launch."""
import ctypes

import pytest
import torch

import largesteps_b200._native as N
from largesteps_b200 import distance as D


def test_batch_offsets():
    assert D._check_batch((0, 3, 7), (0, 2, 5), 7, 5) == 2
    assert D._check_batch([0, 7], [0, 5], 7, 5) == 1
    for vo, fo, msg in (((0, 7), (0, 2, 5), "B \\+ 1"), ((0,), (0,), "B \\+ 1"), ((1, 7), (0, 5), "start at 0"),
                        ((0, 6), (0, 5), "end at 7"), ((0, 3, 7), (0, 4, 6), "end at 5"), ((0, 5, 3, 7), (0, 1, 2, 5), "non-decreasing")):
        with pytest.raises(ValueError, match=msg):
            D._check_batch(vo, fo, 7, 5)
    with pytest.raises(ValueError, match="mesh 1 of the batch has no faces"):
        D._check_batch((0, 3, 5, 7), (0, 2, 2, 5), 7, 5)


def test_point_offsets():
    D._check_points((0, 4, 9), 9, 2)
    D._check_points((0, 4, 9, 9), 9, 1)          # any number of segments against one mesh
    with pytest.raises(ValueError, match="3 segments for a batch of 2"):
        D._check_points((0, 4, 9, 9), 9, 2)
    for po, msg in (((0, 4), "end at 9"), ((2, 9), "start at 0"), ((0, 5, 4, 9), "non-decreasing"), ((0,), "B \\+ 1")):
        with pytest.raises(ValueError, match=f"point_offsets.*{msg}|{msg}"):
            D._check_points(po, 9, 3 if len(po) == 4 else 1)


def test_broadcast_rule():
    assert D._pair(4, 4) == 4 and D._pair(1, 4) == 4 and D._pair(4, 1) == 4 and D._pair(1, 1) == 1
    with pytest.raises(ValueError, match="2 and 3 meshes"):
        D._pair(2, 3)


def test_offset_types():
    with pytest.raises(TypeError, match="face_offsets"):
        D._offsets(torch.zeros(3, dtype=torch.float32), "cpu", "face_offsets")
    with pytest.raises(TypeError):
        D._offsets(torch.zeros((2, 2), dtype=torch.int64), "cpu", "vert_offsets")


def test_cpu_tensors_raise():
    v, f = torch.zeros(3, 3), torch.tensor([[0, 1, 2]])
    with pytest.raises(RuntimeError, match="CUDA"):
        D.MeshDistanceBatch(v, f, [0, 3], [0, 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        D.hausdorff_batch(v, f, [0, 3], [0, 1], v, f, [0, 3], [0, 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        D.chamfer_batch(v, f, [0, 3], [0, 1], v, f, [0, 3], [0, 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        D.point_mesh_squared_distance_batch(v, [0, 3], v, f, [0, 3], [0, 1])


def test_c_entry_points_validate_on_the_host():
    lib = N.lib()
    nb = ctypes.c_size_t(0)
    one = ctypes.c_size_t(0)
    assert lib.ls_distance_bvh_bytes(1000, ctypes.byref(one)) == N.LS_OK
    assert lib.ls_distance_bvh_batch_bytes(1000, 1, ctypes.byref(nb)) == N.LS_OK and nb.value == one.value
    assert lib.ls_distance_bvh_batch_bytes(1000, 10, ctypes.byref(nb)) == N.LS_OK
    assert nb.value >= 256 + 48 * 1000 + 64 * 990
    for F, B in ((1000, 0), (1000, 1001), (0, 1), (1 << 31, 2)):
        assert lib.ls_distance_bvh_batch_bytes(F, B, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG, (F, B)
    assert lib.ls_distance_query_workspace_bytes(500, ctypes.byref(one)) == N.LS_OK
    assert lib.ls_distance_query_batch_workspace_bytes(500, 1, ctypes.byref(nb)) == N.LS_OK and nb.value == one.value
    assert lib.ls_distance_query_batch_workspace_bytes(500, 0, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    assert lib.ls_distance_query_batch_workspace_bytes(-1, 3, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    fake = ctypes.c_void_p(1 << 20)                  # never dereferenced: every check below fails before a launch
    null = ctypes.c_void_p(0)
    stream = ctypes.c_void_p(0)
    assert lib.ls_distance_bvh_batch_build(fake, 10, fake, 4, 8, 2, null, fake, 1 << 30, stream) == N.LS_ERR_BAD_ARG
    assert lib.ls_distance_bvh_batch_build(fake, 10, fake, 2, 8, 2, fake, fake, 1 << 30, stream) == N.LS_ERR_BAD_ARG
    assert lib.ls_distance_bvh_batch_build(fake, 10, fake, 4, 8, 9, fake, fake, 1 << 30, stream) == N.LS_ERR_BAD_ARG
    assert lib.ls_distance_bvh_batch_build(fake, 10, fake, 4, 8, 2, fake, fake, 1, stream) == N.LS_ERR_WORKSPACE

    def query(B=2, S=2, po=fake, mx=null, mode=0, ws=fake, nbytes=1 << 30):
        return lib.ls_distance_query_batch(fake, 8, B, fake, 10, S, po, fake, fake, fake, mx, mode, ws, nbytes, stream)

    assert query(S=3) == N.LS_ERR_BAD_ARG and "segment" in N.last_error()
    assert query(po=null) == N.LS_ERR_BAD_ARG
    assert query(mode=1) == N.LS_ERR_BAD_ARG and "max_out" in N.last_error()
    assert query(mx=fake) == N.LS_ERR_BAD_ARG
    assert query(mx=fake, mode=3) == N.LS_ERR_BAD_ARG
    assert query(ws=ctypes.c_void_p((1 << 20) + 16)) == N.LS_ERR_BAD_ARG and "aligned" in N.last_error()
    assert query(nbytes=1) == N.LS_ERR_WORKSPACE
    assert lib.ls_distance_segment_sum_f64(fake, 10, 0, fake, fake, stream) == N.LS_ERR_BAD_ARG
    assert lib.ls_distance_segment_sum_f64(fake, 10, 2, null, fake, stream) == N.LS_ERR_BAD_ARG
