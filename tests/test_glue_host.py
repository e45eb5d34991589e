"""CPU: the per-face and per-vertex bodies of the normals kernels (csrc/ls_glue.cu, __host__ __device__) compiled for the
host by nvcc and run against the float64 model of tests/glue_model.py, one gradient path at a time, so that a sign, corner
or index error in them shows up without a GPU.  Host and device contract products into FMAs differently, so the bars are
tolerances: rel-L2 below max(5e-6, 20 x the float32 model's own error), the convention of tests/test_gpu_meshops.py."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, rel_l2
from gpu_util import fan_mesh
import glue_model as M
import largesteps_b200._native as N

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HARNESS = r"""
#include <cmath>
#include "ls_glue.cu"
// the normals' two directions on the host, pass by pass as the kernels run them; fn is an input (the face normals)
extern "C" void host_glue(const float *verts, const int64_t *faces, int64_t F, int64_t V, const int *ptr, const int *inc,
                          const float *fn, const float *gn, const float *gout, float *gverts_fn, float *norms, float *out,
                          float *raw_len, float *gfn, float *T, float *gverts) {
    for (int64_t v = 0; v < V; ++v) face_normals_vertex_grad(verts, faces, F, ptr, inc, gn, v, gverts_fn);
    double sq[3] = {0.0, 0.0, 0.0};        // k_edge_norms_batch: float squares summed in double
    for (int64_t f = 0; f < F; ++f)
        for (int d = 0; d < 3; ++d) {
            const float a = verts[3 * faces[3 * f] + d], b = verts[3 * faces[3 * f + 1] + d], c = verts[3 * faces[3 * f + 2] + d];
            const float e01 = b - a, e02 = c - a, e12 = c - b;
            sq[0] += (double)(e01 * e01);
            sq[1] += (double)(e02 * e02);
            sq[2] += (double)(e12 * e12);
        }
    for (int k = 0; k < 3; ++k) norms[k] = (float)std::sqrt(sq[k]);
    const float nm[3] = {norms[0], norms[1], norms[2]};
    for (int64_t v = 0; v < V; ++v) vertex_normal(verts, faces, F, ptr, inc, fn, nm, v, out, raw_len);
    double t[3] = {0.0, 0.0, 0.0};
    for (int64_t f = 0; f < F; ++f) {
        float gf[3];
        vertex_normals_face_grad(verts, faces, F, fn, nm, out, gout, raw_len, f, gf, t);
        for (int d = 0; d < 3; ++d) gfn[d * F + f] = gf[d];
    }
    for (int k = 0; k < 3; ++k) T[k] = (float)t[k];
    const float Tg[3] = {T[0], T[1], T[2]};
    for (int64_t v = 0; v < V; ++v) vertex_normals_vertex_grad(verts, faces, F, ptr, inc, fn, nm, Tg, out, gout, raw_len, v, gverts);
}
"""


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    d = tmp_path_factory.mktemp("glue_host")
    src, lib = d / "harness.cu", d / "libglue_host.so"
    src.write_text(HARNESS)
    libdir = os.path.dirname(N.LIB_PATH)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I", os.path.join(ROOT, "large-steps-pytorch_b200", "csrc"), str(src), "-o", str(lib),
                        "-L", libdir, "-l:libls_b200.so", "-Xlinker", "-rpath=" + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    h = ctypes.CDLL(str(lib))
    h.host_glue.restype = None
    return h


def incidence(f, V):
    """What ls_face_incidence builds: per vertex the sorted codes 4 * face + corner."""
    codes = 4 * np.repeat(np.arange(len(f)), 3) + np.tile(np.arange(3), len(f))
    order = np.lexsort((codes, f.ravel()))
    ptr = np.zeros(V + 1, np.int32)
    ptr[1:] = np.cumsum(np.bincount(f.ravel(), minlength=V))
    return ptr, np.ascontiguousarray(codes[order], dtype=np.int32)


def run_host(h, v, f, fn, gn, gout):
    V, F = len(v), len(f)
    ptr, inc = incidence(f, V)
    o = dict(gverts_fn=np.zeros((V, 3), np.float32), norms=np.zeros(3, np.float32), n=np.zeros((V, 3), np.float32),
             raw_len=np.zeros(V, np.float32), g_fn=np.zeros((3, F), np.float32), T=np.zeros(3, np.float32),
             g_angle=np.zeros((V, 3), np.float32))
    a = [np.ascontiguousarray(x) for x in (v, f, fn, gn, gout)]
    p = lambda x: x.ctypes.data_as(ctypes.c_void_p)
    h.host_glue(p(a[0]), p(a[1]), ctypes.c_int64(F), ctypes.c_int64(V), p(ptr), p(inc), p(a[2]), p(a[3]), p(a[4]),
                p(o["gverts_fn"]), p(o["norms"]), p(o["n"]), p(o["raw_len"]), p(o["g_fn"]), p(o["T"]), p(o["g_angle"]))
    return o


def meshes():
    ms = M.small_meshes()
    d = np.load(os.path.join(GOLDEN, "bunny_mesh.npz"))
    ms["bunny"] = (d["verts"].astype(np.float32), d["faces"].astype(np.int64))
    ms["fan3000"] = fan_mesh(3000)
    return ms


def bound(got, want64, want32):
    return rel_l2(got, want64), max(5e-6, 20 * rel_l2(want32, want64))


@pytest.mark.parametrize("mesh", list(meshes()))
def test_normals_paths_match_the_model(host_lib, mesh):
    v, f = meshes()[mesh]
    rng = np.random.default_rng(7)
    gn = rng.normal(size=(3, len(f))).astype(np.float32)
    gout = rng.normal(size=(len(v), 3)).astype(np.float32)
    fn64, gfn64 = M.face_normal_vjp(v, f, gn)
    fn = fn64.astype(np.float32)
    _, gfn32 = M.face_normal_vjp(v, f, gn, dtype=torch.float32)
    m64 = M.vertex_normal_paths(v, f, fn, gout)
    m32 = M.vertex_normal_paths(v, f, fn, gout, dtype=torch.float32)
    h = run_host(host_lib, v, f, fn, gn, gout)
    err, bar = bound(h["gverts_fn"], gfn64, gfn32)
    assert err < bar, ("face normal backward", err, bar)
    np.testing.assert_allclose(h["norms"], m64["norms"], rtol=2e-7)
    nan = np.isnan(m64["n"]).any(1)
    np.testing.assert_array_equal(np.isnan(h["n"]).any(1), nan)
    assert nan.any() == (mesh == "isolated")
    for path in ("n", "g_fn", "g_angle"):
        got, w64, w32 = h[path], m64[path], m32[path]
        if path == "n":
            got, w64, w32 = got[~nan], w64[~nan], w32[~nan]
        if mesh == "triangle" and path == "g_angle":
            # every vertex normal is the face normal whatever the angles: the path is zero up to rounding
            assert np.abs(w64).max() < 1e-12
            assert np.linalg.norm(got) < 64 * np.finfo(np.float32).eps * np.linalg.norm(gout)
            continue
        err, bar = bound(got, w64, w32)
        assert err < bar, (path, err, bar)
    # T_i: each within the rounding of its terms' magnitudes
    err, bar = bound(h["T"], m64["T"], m32["T"])
    assert err < bar, ("T", h["T"], m64["T"])
