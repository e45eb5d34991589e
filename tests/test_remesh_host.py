"""CPU: remesh_botsch's argument checks and the remesher's C entry points that answer without a GPU (workspace sizes,
rejected arguments)."""
import ctypes

import numpy as np
import pytest
import torch

import largesteps_b200._native as N
from largesteps_b200.remesh import remesh_botsch


def ws_bytes(V, F):
    nb = ctypes.c_size_t(0)
    rc = N.lib().ls_remesh_workspace_bytes(V, F, ctypes.byref(nb))
    return rc, nb.value


def test_workspace_bytes_grow_with_the_mesh():
    sizes = [ws_bytes(V, F) for V, F in ((0, 0), (4, 4), (12, 20), (1000, 1996), (2_600_000, 5_200_000))]
    assert all(rc == N.LS_OK for rc, _ in sizes)
    b = [n for _, n in sizes]
    assert b == sorted(b) and b[0] > 0
    # per vertex slot: buckets, edge pointers, maps, claims, positions and the float64 closest points (~100 bytes); per face
    # slot: corners, edges, face edges and copies (~100 bytes)
    assert b[-1] < 400 * (2_600_000 + 5_200_000)


@pytest.mark.parametrize("V,F", [(-1, 4), (4, -1), (1 << 30, 4), (4, 1 << 29)])
def test_workspace_bytes_reject_sizes(V, F):
    assert ws_bytes(V, F)[0] == N.LS_ERR_BAD_ARG
    assert N.lib().ls_remesh_workspace_bytes(4, 4, None) == N.LS_ERR_BAD_ARG


def test_stages_reject_null_and_small_workspaces():
    lib = N.lib()
    n = ctypes.c_int64(0)
    flags = ctypes.c_uint32(0)
    buf = ctypes.create_string_buffer(4096)
    ws = ctypes.c_void_p((ctypes.addressof(buf) + 255) // 256 * 256)
    fake = ctypes.c_void_p(256)
    assert lib.ls_remesh_check(None, 4, 4, ws, 1024, ctypes.byref(flags), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_check(fake, 0, 4, ws, 1024, ctypes.byref(flags), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_check(fake, 4, 4, ws, 16, ctypes.byref(flags), None) == N.LS_ERR_WORKSPACE
    assert lib.ls_remesh_check(fake, 4, 4, ctypes.c_void_p(ws.value + 8), 1 << 20, ctypes.byref(flags), None) == N.LS_ERR_BAD_ARG
    # split needs room for V + 3F/2 vertices and 4F faces
    assert lib.ls_remesh_split(fake, fake, 4, 4, 9, 16, 1.0, ws, 1 << 20, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_split(fake, fake, 4, 4, 10, 16, 0.0, ws, 1 << 20, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_collapse_round(fake, fake, 4, 4, 4, 1.0, 0.5, ws, 1 << 20, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_collapse_round(None, fake, 4, 4, 4, 0.5, 1.0, ws, 1 << 20, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_flip_round(fake, fake, 4, 4, ws, 16, ctypes.byref(n), None) == N.LS_ERR_WORKSPACE
    assert lib.ls_remesh_compact(fake, fake, 4, 4, ws, 1 << 20, None, None, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_relax(fake, fake, 4, 4, None, 4, ws, 1 << 20, None) == N.LS_ERR_BAD_ARG


def cpu_mesh():
    return torch.zeros(4, 3), torch.tensor([[0, 1, 2], [0, 2, 3], [0, 3, 1], [1, 3, 2]])


@pytest.mark.parametrize("h", [0.0, -1.0, float("nan"), float("inf"), "1", True])
def test_bad_h_is_a_value_error(h):
    v, f = cpu_mesh()
    with pytest.raises(ValueError, match="h must be"):
        remesh_botsch(v, f, 1, h)


@pytest.mark.parametrize("iters", [-1, 1.0, True, None])
def test_bad_iters_is_a_value_error(iters):
    v, f = cpu_mesh()
    with pytest.raises(ValueError, match="iters must be"):
        remesh_botsch(v, f, iters, 0.5)


def test_cpu_tensors_are_refused():
    v, f = cpu_mesh()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        remesh_botsch(v, f, 1, 0.5)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        remesh_botsch(v.numpy(), f, 1, 0.5)


def test_empty_sizes_launch_nothing():
    lib = N.lib()
    n, nv, nf = ctypes.c_int64(-1), ctypes.c_int64(-1), ctypes.c_int64(-1)
    flags = ctypes.c_uint32(0)
    buf = ctypes.create_string_buffer(1 << 16)
    ws = ctypes.c_void_p((ctypes.addressof(buf) + 255) // 256 * 256)
    fake = ctypes.c_void_p(256)
    assert lib.ls_remesh_check(fake, 4, 0, ws, 1 << 15, ctypes.byref(flags), None) == N.LS_ERR_INDEX_RANGE
    assert lib.ls_remesh_split(fake, fake, 5, 0, 5, 0, 1.0, ws, 1 << 15, ctypes.byref(n), None) == N.LS_OK and n.value == 0
    n.value = -1
    assert lib.ls_remesh_collapse_round(fake, fake, 5, 0, 5, 0.5, 1.0, ws, 1 << 15, ctypes.byref(n), None) == N.LS_OK
    assert n.value == 0
    n.value = -1
    assert lib.ls_remesh_flip_round(fake, fake, 5, 0, ws, 1 << 15, ctypes.byref(n), None) == N.LS_OK and n.value == 0
    assert lib.ls_remesh_compact(fake, fake, 5, 0, ws, 1 << 15, ctypes.byref(nv), ctypes.byref(nf), None) == N.LS_OK
    assert nv.value == 0 and nf.value == 0
    # faces without vertices
    assert lib.ls_remesh_split(fake, fake, 0, 4, 6, 16, 1.0, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_flip_round(fake, fake, 0, 4, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
