"""CPU: the per-vertex gather and the per-face weight gradient of the matrix-free cotangent product (csrc/ls_assemble.cu,
laplacian_cot_product; __host__ __device__) compiled for the host by nvcc and run on the meshes of tests/golden/cot_grad.npz,
with the bars of tests/test_gpu_cot_product.py: y = L x against the float64 model, and the gradients of the two regularisers
built on y = L v against the reference's float64 gradients."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, ROOT, rel_l2
import largesteps_b200._native as N
import cot_grad_model as model
from test_massmatrix_host import incidence

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HARNESS = r"""
#include "ls_assemble.cu"
static void gather(const int64_t *faces, int64_t V, const int *ptr, const int *inc, const float *w, const float *x, int k,
                   float *y) {
    for (int64_t v = 0; v < V; ++v)
        for (int c0 = 0; c0 < k; c0 += 4) {
            float acc[4];
            cot_product_row(faces, ptr, inc, w, x, k, c0, v, acc);
            for (int q = 0; q < 4 && c0 + q < k; ++q) y[v * k + c0 + q] = acc[q];
        }
}
// forward (w as k_cot computes it, then y = L x) and, for the gradient gy of y, gx = L gy and gverts through the weights
extern "C" void host_cot_product(const float *verts, const int64_t *faces, int64_t F, int64_t V, const int *ptr, const int *inc,
                                 const float *x, const float *gy, int k, float *w, float *y, float *gx, float *wbar,
                                 float *gverts) {
    for (int64_t f = 0; f < F; ++f) {
        float p[3][3];
        for (int a = 0; a < 3; ++a)
            for (int d = 0; d < 3; ++d) p[a][d] = verts[3 * faces[3 * f + a] + d];
        CotFace c;
        cot_face(p, c);
        for (int e = 0; e < 3; ++e) w[3 * f + e] = (c.num[e] / c.area) / 4.0f;
    }
    gather(faces, V, ptr, inc, w, x, k, y);
    gather(faces, V, ptr, inc, w, gy, k, gx);
    for (int64_t f = 0; f < F; ++f) {
        float wb[3];
        cot_product_face_wbar(faces, f, x, gy, k, wb);
        for (int e = 0; e < 3; ++e) wbar[3 * f + e] = wb[e];
    }
    for (int64_t v = 0; v < V; ++v) {
        float acc[3];
        cot_vertex_grad(verts, faces, ptr, inc, wbar, v, acc);
        for (int d = 0; d < 3; ++d) gverts[3 * v + d] = acc[d];
    }
}
"""
MESHES = ["ico2", "bunny", "grid", "plane", "degen"]


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    d = tmp_path_factory.mktemp("cot_product_host")
    src, lib = d / "harness.cu", d / "libcot_product_host.so"
    src.write_text(HARNESS)
    libdir = os.path.dirname(N.LIB_PATH)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I", os.path.join(ROOT, "large-steps-pytorch_b200", "csrc"), str(src), "-o", str(lib),
                        "-L", libdir, "-l:libls_b200.so", "-Xlinker", "-rpath=" + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    h = ctypes.CDLL(str(lib))
    h.host_cot_product.restype = None
    return h


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "cot_grad.npz"))


def host_product(host_lib, v, f, x, gy):
    """(y, gx, gverts) of the host bodies: y = L x, and for the gradient gy of y, L gy and the gradient through the weights."""
    V, F, k = len(v), len(f), x.shape[1]
    ptr, inc = incidence(f, V)
    v, f = np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int64)
    x, gy = np.ascontiguousarray(x, np.float32), np.ascontiguousarray(gy, np.float32)
    w, wbar = np.zeros(3 * F, np.float32), np.zeros(3 * F, np.float32)
    y, gx, gv = np.zeros((V, k), np.float32), np.zeros((V, k), np.float32), np.zeros((V, 3), np.float32)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    host_lib.host_cot_product(p(v), p(f), ctypes.c_int64(F), ctypes.c_int64(V), p(ptr), p(inc), p(x), p(gy), ctypes.c_int(k),
                              p(w), p(y), p(gx), p(wbar), p(gv))
    return y, gx, gv


def forward_bound(v, f, x):
    """1e-5 max_i sum_j |W_ij| |x_i - x_j|, per column, W the off-diagonal of the float64 model's L."""
    rows, cols, vals = model.laplacian(v, f)
    off = rows != cols
    r, c, a = rows[off], cols[off], np.abs(vals[off])
    x = np.asarray(x, np.float64)
    s = np.zeros_like(x)
    np.add.at(s, r, a[:, None] * np.abs(x[r] - x[c]))
    return 1e-5 * s.max()


def model_product(v, f, x):
    rows, cols, vals = model.laplacian(v, f)
    y = np.zeros((len(v), x.shape[1]))
    np.add.at(y, rows, vals[:, None] * np.asarray(x, np.float64)[cols])
    return y


@pytest.mark.parametrize("k", [1, 3, 4])
@pytest.mark.parametrize("mesh", MESHES)
def test_forward_matches_float64_model(host_lib, golden, mesh, k):
    v, f = model.golden_mesh(golden, mesh)
    x = np.random.default_rng(k).normal(size=(len(v), k)).astype(np.float32)
    y, _, _ = host_product(host_lib, v, f, x, np.zeros_like(x))
    err, bound = np.abs(y - model_product(v, f, x)).max(), forward_bound(v, f, x)
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("loss", ["reg_bi", "reg_lap"])
@pytest.mark.parametrize("mesh", MESHES)
def test_regulariser_gradient_matches_reference(host_lib, golden, mesh, loss):
    """y = L v; reg_bi = mean(y^2), reg_lap = mean(v * y): the gradient is the x path L gy, the weights path, and for reg_lap
    the direct y / n, combined in float32 as autograd combines them."""
    v, f = model.golden_mesh(golden, mesh)
    y, _, _ = host_product(host_lib, v, f, v, np.zeros_like(v))
    n = np.float32(v.size)
    gy = (np.float32(2) * y / n if loss == "reg_bi" else v / n).astype(np.float32)
    _, gx, gv = host_product(host_lib, v, f, v, gy)
    grad = gv + gx if loss == "reg_bi" else gv + gx + y / n
    assert np.isfinite(grad).all()
    err, ref_err = rel_l2(grad, golden[f"{mesh}.{loss}.grad"]), float(golden[f"{mesh}.{loss}.f32_err"])
    assert err < max(5e-6, 20 * ref_err), (err, ref_err)


def test_corner_cases_of_the_degenerate_mesh(host_lib, golden):
    """The isolated vertex gets 0 in y and in both gradients, and a duplicated face adds its weights twice."""
    v, f = model.golden_mesh(golden, "degen")
    used = np.zeros(len(v), bool)
    used[f.ravel()] = True
    rng = np.random.default_rng(0)
    x, gy = rng.normal(size=(len(v), 3)).astype(np.float32), rng.normal(size=(len(v), 3)).astype(np.float32)
    y, gx, gv = host_product(host_lib, v, f, x, gy)
    assert (~used).any()
    assert (y[~used] == 0).all() and (gx[~used] == 0).all() and (gv[~used] == 0).all()
    # without the duplicated face and the self-edge face, vertex 1 sees the proper face [0, 1, 2] once
    y1, _, _ = host_product(host_lib, v, f[[0, 2, 3]], x, gy)
    y2, _, _ = host_product(host_lib, v, f[[0, 0, 2, 3]], x, gy)
    np.testing.assert_allclose(y2[1], 2 * y1[1], rtol=1e-5, atol=1e-6 * np.abs(y1[1]).max())
