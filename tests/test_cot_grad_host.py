"""CPU: the per-face and per-vertex bodies of the cotangent assembly's backward (csrc/ls_assemble.cu, __host__ __device__)
compiled for the host by nvcc and run against tests/golden/cot_grad.npz, with the bars of tests/test_gpu_cot_grad.py: the
gradient of (M.values() * W).sum() w.r.t. verts, for M = I + 19 L and M = 0.05 I + 0.95 L, lies within max(5e-6, 20x the
reference's own float32 error) of the reference's float64 gradient."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, rel_l2
import largesteps_b200._native as N
from cot_grad_model import golden_mesh, golden_weights
from test_massmatrix_host import incidence

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HARNESS = r"""
#include "ls_assemble.cu"
extern "C" void host_cot_bwd(const float *verts, const int64_t *faces, int64_t F, int64_t V, float scale, const int *rowptr,
                             const int *col, const float *gval, const int *ptr, const int *inc, float *wbar, float *gverts) {
    for (int64_t f = 0; f < F; ++f) {
        float w[3];
        cot_face_wbar(faces, f, scale, rowptr, col, gval, w);
        for (int e = 0; e < 3; ++e) wbar[3 * f + e] = w[e];
    }
    for (int64_t v = 0; v < V; ++v) {
        float acc[3];
        cot_vertex_grad(verts, faces, ptr, inc, wbar, v, acc);
        for (int d = 0; d < 3; ++d) gverts[3 * v + d] = acc[d];
    }
}
"""


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    d = tmp_path_factory.mktemp("cot_host")
    src, lib = d / "harness.cu", d / "libcot_host.so"
    src.write_text(HARNESS)
    libdir = os.path.dirname(N.LIB_PATH)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I", os.path.join(ROOT, "large-steps-pytorch_b200", "csrc"), str(src), "-o", str(lib),
                        "-L", libdir, "-l:libls_b200.so", "-Xlinker", "-rpath=" + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    h = ctypes.CDLL(str(lib))
    h.host_cot_bwd.restype = None
    return h


def host_grad(host_lib, g, mesh, W, scale):
    v, f = golden_mesh(g, mesh)
    idx = g[f"{mesh}.idx"]
    V, F = len(v), len(f)
    rowptr = np.searchsorted(idx[0], np.arange(V + 1)).astype(np.int32)
    col = np.ascontiguousarray(idx[1], dtype=np.int32)
    ptr, inc = incidence(f, V)
    wbar, grad = np.zeros(3 * F, np.float32), np.zeros((V, 3), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    W = np.ascontiguousarray(W, dtype=np.float32)
    host_lib.host_cot_bwd(p(v), p(f), ctypes.c_int64(F), ctypes.c_int64(V), ctypes.c_float(scale), p(rowptr), p(col), p(W),
                          p(ptr), p(inc), p(wbar), p(grad))
    return wbar, grad


@pytest.mark.parametrize("case,scale", [("l19", 19.0), ("a095", 0.95)])
@pytest.mark.parametrize("mesh", ["ico2", "bunny", "grid", "plane", "degen"])
def test_kernel_math_matches_reference(host_lib, mesh, case, scale):
    g = np.load(os.path.join(GOLDEN, "cot_grad.npz"))
    _, grad = host_grad(host_lib, g, mesh, golden_weights(g, mesh, case), scale)
    assert np.isfinite(grad).all()                      # as the reference's: the area clamp keeps degenerate faces finite
    err, ref_err = rel_l2(grad, g[f"{mesh}.{case}.grad"]), float(g[f"{mesh}.{case}.f32_err"])
    assert err < max(5e-6, 20 * ref_err), (err, ref_err)


def test_self_edge_and_duplicate_face_weights(host_lib):
    """The degenerate mesh's repeated-vertex face [0, 0, 2] gets no gradient on its self-edge (0, 0); its duplicated face
    [0, 1, 2] reads the same coalesced entries as the original, so both get the same weight gradients."""
    g = np.load(os.path.join(GOLDEN, "cot_grad.npz"))
    f = g["degen.faces"]
    wbar, _ = host_grad(host_lib, g, "degen", golden_weights(g, "degen", "l19"), 19.0)
    wbar = wbar.reshape(-1, 3)
    rep = int(np.flatnonzero((f[:, 0] == f[:, 1]) & (f[:, 1] != f[:, 2]))[0])
    assert wbar[rep, 2] == 0.0 and wbar[rep, 0] != 0.0 and wbar[rep, 1] != 0.0
    np.testing.assert_array_equal(wbar[0], wbar[len(f) - 1])
    assert (f[0] == f[-1]).all()
