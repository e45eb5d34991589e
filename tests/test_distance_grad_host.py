"""CPU: the weights body of the distance backward (ls_closest_on_triangle_w, csrc/ls_distance.cu, __host__ __device__) compiled
for the host by nvcc.  On 10^5 seeded pairs, degenerate triangles included, its point is ls_closest_on_triangle's bit for bit,
its weights sum to 1 to float64 rounding and match the float64 model of tests/distance_grad_model.py.  The new C entry points
reject bad arguments before touching a device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import largesteps_b200._native as N
import distance_grad_model as gm
from test_distance_host import seeded_pairs

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
HARNESS = r"""
#include "ls_distance.cu"
extern "C" void host_closest_w(const float *p, const float *tri, int64_t m, double *sqrD, double *C, double *sqrD_w,
                               double *C_w, double *beta) {
    for (int64_t i = 0; i < m; ++i) {
        const double q[3] = {p[3 * i], p[3 * i + 1], p[3 * i + 2]};
        double a[3], b[3], c[3];
        for (int d = 0; d < 3; ++d) {
            a[d] = tri[9 * i + d];
            b[d] = tri[9 * i + 3 + d];
            c[d] = tri[9 * i + 6 + d];
        }
        sqrD[i] = ls_closest_on_triangle(q, a, b, c, C + 3 * i);
        sqrD_w[i] = ls_closest_on_triangle_w(q, a, b, c, C_w + 3 * i, beta + 3 * i);
    }
}
"""


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    if shutil.which(NVCC) is None and not os.path.exists(NVCC):
        pytest.skip("nvcc is not available")
    d = tmp_path_factory.mktemp("distance_grad_host")
    src, lib = d / "harness.cu", d / "libdistance_grad_host.so"
    src.write_text(HARNESS)
    libdir = os.path.dirname(N.LIB_PATH)
    r = subprocess.run([NVCC, "-std=c++17", "-O2", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                        "-I", os.path.join(ROOT, "large-steps-pytorch_b200", "csrc"), str(src), "-o", str(lib),
                        "-L", libdir, "-l:libls_b200.so", "-Xlinker", "-rpath=" + libdir], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    h = ctypes.CDLL(str(lib))
    h.host_closest_w.restype = None
    return h


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def test_weights_body_against_the_closest_point_and_the_model(host_lib):
    q, tri = seeded_pairs()
    m = len(q)
    s, c, sw, cw, beta = np.zeros(m), np.zeros((m, 3)), np.zeros(m), np.zeros((m, 3)), np.zeros((m, 3))
    host_lib.host_closest_w(_p(q), _p(np.ascontiguousarray(tri.reshape(m, 9))), ctypes.c_int64(m), _p(s), _p(c), _p(sw), _p(cw),
                            _p(beta))
    np.testing.assert_array_equal(sw.view(np.uint64), s.view(np.uint64))          # the same point, bit for bit
    np.testing.assert_array_equal(cw.view(np.uint64), c.view(np.uint64))
    assert np.abs(beta.sum(1) - 1.0).max() <= 4 * 2.0 ** -53
    t = tri.astype(np.float64)
    want = gm.weights(q.astype(np.float64), t[:, 0], t[:, 1], t[:, 2])
    err = np.abs(beta - want).max(1)
    assert err.max() <= 1e-12, (err.max(), int(err.argmax()))
    # the weights give back the point, to rounding in the corners' scale
    scale = np.abs(t).max((1, 2))
    assert (np.abs((beta[:, :, None] * t).sum(1) - c).max(1) <= 1e-12 * scale + 1e-300).all()


def test_grad_entry_points_validate_on_the_host():
    lib = N.lib()
    nb = ctypes.c_size_t(0)
    assert lib.ls_distance_grad_workspace_bytes(1000, 2000, 1002, ctypes.byref(nb)) == N.LS_OK
    small = nb.value
    # queries by face (F + 1, n), corners by vertex (V + 1, 3F), and one bucket workspace
    assert 4 * (2001 + 1000 + 1003 + 6000) <= small
    # the plane(1000) pair: 10^6 queries on 1,996,002 faces and 10^6 vertices, about 56 MB
    assert lib.ls_distance_grad_workspace_bytes(1_000_000, 1_996_002, 1_000_000, ctypes.byref(nb)) == N.LS_OK
    assert small < nb.value < 64e6
    print(f"gradient workspace at the plane(1000) pair: {nb.value} bytes")
    for n, F, V in ((-1, 10, 10), (10, 0, 10), (10, 10, 0), (10, 0x1ffffff0 // 3 + 1, 10), (0x7ffffff0, 10, 10)):
        assert lib.ls_distance_grad_workspace_bytes(n, F, V, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG, (n, F, V)
    assert lib.ls_distance_grad_workspace_bytes(10, 10, 10, None) == N.LS_ERR_BAD_ARG
    fake = ctypes.c_void_p(1 << 20)                  # never dereferenced: every check below fails before a launch
    null = ctypes.c_void_p(0)
    stream = ctypes.c_void_p(0)

    def call(n=4, F=2, V=4, idx_bytes=4, pts=fake, verts=fake, faces=fake, face=fake, closest=fake, g=fake, gp=fake, gv=fake,
             ws=fake, nbytes=1 << 30):
        return lib.ls_distance_grad_f32(pts, n, verts, V, faces, idx_bytes, F, face, closest, g, gp, gv, ws, nbytes, stream)

    assert call(idx_bytes=2) == N.LS_ERR_BAD_ARG
    assert call(n=-1) == N.LS_ERR_BAD_ARG
    assert call(F=0) == N.LS_ERR_BAD_ARG
    assert call(V=0) == N.LS_ERR_BAD_ARG
    for k in ("pts", "face", "closest", "g"):
        assert call(**{k: null}) == N.LS_ERR_BAD_ARG, k
    assert call(verts=null) == N.LS_ERR_BAD_ARG and "verts" in N.last_error()
    assert call(faces=null) == N.LS_ERR_BAD_ARG
    assert call(ws=null) == N.LS_ERR_BAD_ARG
    assert call(ws=ctypes.c_void_p((1 << 20) + 16)) == N.LS_ERR_BAD_ARG and "aligned" in N.last_error()
    assert call(nbytes=1) == N.LS_ERR_WORKSPACE
    with pytest.raises(RuntimeError):
        N.check(call(nbytes=1))
