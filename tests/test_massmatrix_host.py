"""CPU: the per-vertex bodies of the massmatrix_voronoi kernels (csrc/ls_glue.cu, __host__ __device__) compiled for the host
by nvcc and run against tests/golden/mass.npz with the same bars as tests/test_gpu_massmatrix.py, so the float32 operation
order and the NaN behaviour of degenerate faces are checked without a GPU."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, rel_l2
import largesteps_b200._native as N

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HARNESS = r"""
#include "ls_glue.cu"
extern "C" void host_massmatrix_voronoi(const float *verts, const int64_t *faces, int64_t V, const int *ptr, const int *inc,
                                        const float *gout, float *out, float *gverts) {
    for (int64_t v = 0; v < V; ++v) {
        out[v] = mass_vertex(verts, faces, ptr, inc, v);
        float acc[3];
        mass_vertex_grad(verts, faces, ptr, inc, gout, v, acc);
        for (int d = 0; d < 3; ++d) gverts[3 * v + d] = acc[d];
    }
}
"""


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    d = tmp_path_factory.mktemp("mass_host")
    src, lib = d / "harness.cu", d / "libmass_host.so"
    src.write_text(HARNESS)
    libdir = os.path.dirname(N.LIB_PATH)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I", os.path.join(ROOT, "large-steps-pytorch_b200", "csrc"), str(src), "-o", str(lib),
                        "-L", libdir, "-l:libls_b200.so", "-Xlinker", "-rpath=" + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    h = ctypes.CDLL(str(lib))
    h.host_massmatrix_voronoi.restype = None
    return h


def incidence(f, V):
    """What ls_face_incidence builds: per vertex the sorted codes 4 * face + corner."""
    codes = 4 * np.repeat(np.arange(len(f)), 3) + np.tile(np.arange(3), len(f))
    order = np.lexsort((codes, f.ravel()))
    ptr = np.zeros(V + 1, np.int32)
    ptr[1:] = np.cumsum(np.bincount(f.ravel(), minlength=V))
    return ptr, np.ascontiguousarray(codes[order], dtype=np.int32)


@pytest.mark.parametrize("mesh", ["ico2", "bunny", "grid", "plane", "degen"])
def test_kernel_math_matches_reference(host_lib, mesh):
    g = np.load(os.path.join(GOLDEN, "mass.npz"))
    v, f, W = g[f"{mesh}.verts"], g[f"{mesh}.faces"], g[f"{mesh}.W"]
    V = len(v)
    ptr, inc = incidence(f, V)
    m, grad = np.zeros(V, np.float32), np.zeros((V, 3), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    host_lib.host_massmatrix_voronoi(p(v), p(f), ctypes.c_int64(V), p(ptr), p(inc), p(W), p(m), p(grad))
    ref = g[f"{mesh}.f32.mass"]
    np.testing.assert_array_equal(np.isnan(m), np.isnan(ref))
    fin = ~np.isnan(ref)
    np.testing.assert_allclose(m[fin], ref[fin], rtol=0, atol=2e-6 * np.abs(ref[fin]).max())
    g64, g32 = g[f"{mesh}.f64.grad"], g[f"{mesh}.f32.grad"]
    bad = ~np.isfinite(g64).all(axis=1)
    np.testing.assert_array_equal(~np.isfinite(grad).all(axis=1), bad)
    assert rel_l2(grad[~bad], g64[~bad]) < max(5e-6, 20 * rel_l2(g32[~bad], g64[~bad]))
