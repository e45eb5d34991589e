"""CPU: libls_b200.so holds one copy of each kernel.  A non-template `static __global__` kernel defined in a header is compiled
and registered again by every translation unit that includes the header, whether it launches the kernel or not, so such a
kernel lives in the .cu file that launches it.  The kernel entries are read with cuobjdump -symbols."""
import collections
import os
import shutil
import subprocess

import pytest

import largesteps_b200._native as N

CUOBJDUMP = os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")


def kernel_entries():
    tool = CUOBJDUMP if os.path.exists(CUOBJDUMP) else shutil.which("cuobjdump")
    if tool is None:
        pytest.skip("cuobjdump is not available")
    if not os.path.exists(N.LIB_PATH):
        pytest.skip("libls_b200.so is not built")
    out = subprocess.run([tool, "-symbols", N.LIB_PATH], capture_output=True, text=True, check=True).stdout
    return [line.split()[-1] for line in out.splitlines() if "STO_ENTRY" in line]


def test_every_kernel_is_compiled_once():
    names = kernel_entries()
    assert names, "no kernel entries found"
    dup = sorted((n, c) for n, c in collections.Counter(names).items() if c > 1)
    assert not dup, f"{len(dup)} kernels compiled more than once: " + ", ".join(f"{n} x{c}" for n, c in dup)
