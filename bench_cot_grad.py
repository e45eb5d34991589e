#!/usr/bin/env python
"""Timing of the cotangent matrix's gradient path on one GPU: the assembly forward (compute_matrix(v, f, 19, cotan=True), the
whole call), the values gradient of L @ v (ls_spmm_csr_grad_val_f32, k = 3) and the backward of the assembly
(ls_laplacian_cot_bwd_f32, both passes), at workloads.plane(1000) (V = 10^6) and the bunny subdivided twice (V = 52,786).

    python bench_cot_grad.py [--reps 200] [--rounds 5]

CUDA events around `reps` back-to-back calls after a warm-up, `rounds` times; prints the card name and power limit, then per
workload and operation the median and range of the per-call times in microseconds, and for the values gradient its bytes/s
from the byte model 8 nnz + 4 (V+1) + 8 k V against the H100 SXM data sheet's 3.35 TB/s.  Writes nothing.
"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "large-steps-pytorch_b200"))
from largesteps_b200 import _native as N, workloads  # noqa: E402
from largesteps_b200.geometry import compute_matrix, csr_of  # noqa: E402
from largesteps_b200.meshops import face_incidence  # noqa: E402
from largesteps_b200.parameterize import spmm_grad_values  # noqa: E402

DEV = "cuda:0"
HBM_PEAK = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def workload(name):
    if name == "plane1000":
        v, f = workloads.plane(1000)
    else:
        d = np.load(os.path.join(ROOT, "tests", "golden", "bunny_mesh.npz"))
        v, f = workloads.subdivide(*workloads.subdivide(d["verts"], d["faces"].astype(np.int64)))
    return (torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(DEV),
            torch.from_numpy(np.ascontiguousarray(f, dtype=np.int64)).to(DEV))


def timed(fn, reps, rounds):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    per = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        per.append(1e3 * e0.elapsed_time(e1) / reps)
    return float(np.median(per)), min(per), max(per)


def run(name, reps, rounds):
    v, f = workload(name)
    V, F = v.shape[0], f.shape[0]
    M = compute_matrix(v, f, 19.0, cotan=True)
    rowptr, col, _ = csr_of(M)
    nnz = col.shape[0]
    k = 3
    gen = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(V, k, device=DEV, generator=gen)
    gy = torch.randn(V, k, device=DEV, generator=gen)
    gval = torch.randn(nnz, device=DEV, generator=gen)
    ptr, items = face_incidence(f, V)
    gv = torch.empty(V, 3, device=DEV)
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_laplacian_cot_bwd_scratch_bytes(F, ctypes.byref(nb)))
    scratch = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    st = N.stream_ptr(DEV)

    def cot_bwd():
        N.check(N.lib().ls_laplacian_cot_bwd_f32(N.ptr(v), N.ptr(f), 8, F, V, 19.0, N.ptr(rowptr), N.ptr(col), N.ptr(gval),
                                                 N.ptr(ptr), N.ptr(items), N.ptr(scratch), nb.value, N.ptr(gv), st))

    rows = [("assembly forward (compute_matrix, cotan)", timed(lambda: compute_matrix(v, f, 19.0, cotan=True), max(reps // 10, 5),
                                                               rounds), None),
            ("values gradient of L @ v (k = 3)", timed(lambda: spmm_grad_values(M, gy, x), reps, rounds),
             8 * nnz + 4 * (V + 1) + 8 * k * V),
            ("assembly backward (both passes)", timed(cot_bwd, reps, rounds), None)]
    print(f"{name}: V = {V}, F = {F}, nnz = {nnz}")
    for what, (med, lo, hi), nbytes in rows:
        line = f"  {what:44s} {med:9.1f} us  [{lo:.1f} .. {hi:.1f}]"
        if nbytes:
            bw = nbytes / (med * 1e-6)
            line += f"  {nbytes / 1e6:.1f} MB -> {bw / 1e12:.2f} TB/s = {bw / HBM_PEAK:.2f} of 3.35 TB/s"
        print(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_cot_grad.py needs a GPU"
    print("card:", card())
    for name in ("plane1000", "bunny_x2"):
        run(name, a.reps, a.rounds)


if __name__ == "__main__":
    main()
