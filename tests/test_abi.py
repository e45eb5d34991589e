"""CPU: the C-ABI library loads and exports every symbol include/largesteps_b200.h declares; host-only entry
points validate their arguments without touching a GPU."""
import ctypes
import os
import re

import pytest

from conftest import ROOT
import largesteps_b200._native as N

HEADERS = [os.path.join(ROOT, "include", "largesteps_b200.h"), os.path.join(ROOT, "include", "largesteps_b200_diag.h")]


def declared_symbols(headers=HEADERS):
    names = set()
    for h in headers:
        src = open(h).read()
        src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
        names |= set(re.findall(r"\b(ls_[a-z0-9_]+)\s*\(", src))
    return sorted(names)


def test_diagnostics_are_not_in_the_product_header():
    prod = declared_symbols(HEADERS[:1])
    for n in ("ls_pcg_bench", "ls_pcg_bench_spmm", "ls_pcg_phase_cycles", "ls_pcg_spmv_put", "ls_pcg_spmv_get"):
        assert n not in prod and n in declared_symbols(HEADERS[1:])


def test_library_is_built_and_loads():
    assert os.path.exists(N.LIB_PATH), "libls_b200.so missing: run __graft_entry__.build()"
    lib = N.lib()
    assert lib.ls_version() >= 100
    assert isinstance(N.last_error(), str)


def test_every_declared_symbol_is_exported_and_bound():
    names = declared_symbols()
    assert len(names) == len(N.SYMBOLS) >= 16
    raw = ctypes.CDLL(N.LIB_PATH)
    for n in names:
        assert hasattr(raw, n), f"{n} declared in the header but not exported"
        assert n in N.SYMBOLS, f"{n} declared in the header but not bound in _native.SYMBOLS"
    for n in N.SYMBOLS:
        assert n in names, f"{n} bound in Python but not declared in the header"


def test_status_strings():
    lib = N.lib()
    assert lib.ls_status_string(0) == b"ok"
    for s in range(1, 8):
        assert len(lib.ls_status_string(s)) > 0


def test_host_side_argument_validation():
    lib = N.lib()
    nb = ctypes.c_size_t(0)
    assert lib.ls_assemble_workspace_bytes(10, 8, ctypes.byref(nb)) == N.LS_OK and nb.value > 0
    assert lib.ls_assemble_workspace_bytes(-1, 8, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    assert "negative" in N.last_error()
    assert lib.ls_assemble_workspace_bytes(400_000_000, 8, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG   # int32 bucket limit
    assert lib.ls_pcg_workspace_bytes(1000, 7000, 3, ctypes.byref(nb)) == N.LS_OK
    small = nb.value
    assert lib.ls_pcg_workspace_bytes(1_000_000, 6_992_002, 4, ctypes.byref(nb)) == N.LS_OK
    # 1M verts: CSR copy (60 MB) + 4x4 planes + dinv  ~ 0.33 GB
    assert small < nb.value < 400e6
    assert lib.ls_pcg_workspace_bytes(1000, 7000, 5, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    assert lib.ls_pcg_workspace_bytes(0, 0, 3, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    with pytest.raises(ValueError):
        N.check(lib.ls_pcg_workspace_bytes(1000, 7000, 0, ctypes.byref(nb)))
    assert lib.ls_pcg_destroy(None) == N.LS_OK
    assert lib.ls_pcg_spmm_bytes(None, 3) == 0
    assert lib.ls_launch_count() >= 0


def test_round2_entry_points_validate_on_the_host():
    lib = N.lib()
    nb = ctypes.c_size_t(0)
    assert lib.ls_glue_scratch_bytes(ctypes.byref(nb)) == N.LS_OK and nb.value >= 3 * 148 * 8
    assert lib.ls_bucket_workspace_bytes(1000, ctypes.byref(nb)) == N.LS_OK and nb.value > 8000
    assert lib.ls_bucket_workspace_bytes(-1, ctypes.byref(nb)) == N.LS_ERR_BAD_ARG
    assert lib.ls_pcg_set_refinement(None, 1, 3.0) == N.LS_ERR_BAD_ARG and "handle" in N.last_error()
    # the workspace size is a function of (V, nnz, k_max) only: no environment variable may change it (VERDICT r1)
    import os
    sizes = []
    for env in ({}, {"LS_PCG_PATTERN": "0"}, {"LS_PCG_MODE": "graph", "LS_PCG_CLUSTER": "16"}):
        old = {k: os.environ.get(k) for k in env}
        os.environ.update(env)
        try:
            assert lib.ls_pcg_workspace_bytes(250000, 1746002, 4, ctypes.byref(nb)) == N.LS_OK
            sizes.append(nb.value)
        finally:
            for k, v in old.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
    assert len(set(sizes)) == 1


def test_check_maps_status_to_exceptions():
    with pytest.raises(IndexError):
        N.check(N.LS_ERR_INDEX_RANGE)
    with pytest.raises(N.NotConverged):
        N.check(N.LS_ERR_NOT_CONVERGED)
    with pytest.raises(N.Breakdown):
        N.check(N.LS_ERR_BREAKDOWN)
    with pytest.raises(RuntimeError):
        N.check(N.LS_ERR_CUDA)
    N.check(N.LS_OK)


def test_header_is_plain_c_and_the_c_host_example_links(tmp_path):
    """include/largesteps_b200.h must be usable from C (the drop-in boundary is a C ABI, not a C++ or torch one):
    the pure-C host example is compiled as strict C99 with -Wall -Wextra -Werror and linked against the library.
    Nothing is executed here (no GPU); tests/test_gpu_integration_snippet.py runs it on the device."""
    import shutil
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if shutil.which("gcc") is None or not os.path.exists("/usr/local/cuda/include/cuda_runtime_api.h"):
        pytest.skip("gcc or the CUDA headers are not available")
    hdr = os.path.join(root, "include", "largesteps_b200.h")
    for std, lang in (("c99", "c"), ("c++17", "c++")):
        r = subprocess.run(["gcc", "-std=" + std, "-x", lang, "-Wall", "-Wextra", "-Werror", "-fsyntax-only", hdr],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
    out = str(tmp_path / "roundtrip")
    libdir = os.path.join(root, "large-steps-pytorch_b200", "largesteps_b200")
    r = subprocess.run(["gcc", "-std=c99", "-O1", "-Wall", "-Wextra", "-Werror", "-I", os.path.join(root, "include"),
                        "-I", "/usr/local/cuda/include", os.path.join(root, "examples", "c_host", "roundtrip.c"), "-o", out,
                        "-L", libdir, "-l:libls_b200.so", "-L", "/usr/local/cuda/lib64", "-lcudart", "-lm"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert os.path.getsize(out) > 0
