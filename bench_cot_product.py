#!/usr/bin/env python
"""Timing of the cotangent regulariser recomputed from the current shape, forward + backward, two ways, at workloads.plane(1000)
(V = 10^6) and the bunny subdivided twice (V = 52,786), int64 faces:

    (a) meshops.laplacian_regularizer(laplacian_cot(v, f), v)           assembly, SpMM, values gradient, assembly backward
    (b) y = meshops.laplacian_cot_product(v, f, v); y.square().mean()  matrix-free: k_cot + gather, gather + w-bar + vertex chain

    python bench_cot_product.py [--reps 200] [--rounds 5]

The harness of bench_cot_grad.py: CUDA events around `reps` back-to-back steps after a warm-up, `rounds` times; prints the card
name and power limit, then the median and range of the per-step times in microseconds.  Then, in a separate profiled run of
(b), each of its kernels' median and range from torch.profiler, with bytes/s from a compulsory-traffic byte model (every array
read or written once) against the H100 SXM data sheet's 3.35 TB/s.  Last, the rel-L2 between (a) and (b) of the loss and of
the gradient.  Writes nothing.
"""
import argparse
import os
import re
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "large-steps-pytorch_b200"))
from bench_cot_grad import DEV, HBM_PEAK, card, timed, workload  # noqa: E402
from largesteps_b200.geometry import laplacian_cot  # noqa: E402
from largesteps_b200.meshops import face_incidence, laplacian_cot_product, laplacian_regularizer  # noqa: E402


def kernel_bytes(V, F, s, k):
    """Compulsory bytes of each kernel of (b): faces (3 s F, s the index size), inc_ptr 4 (V + 1), inc 12 F, the weights and
    their gradient 12 F each, positions 12 V, k-column operands 4 k V."""
    return {"k_cot": 3 * s * F + 12 * V + 12 * F,
            "k_cot_product": 4 * (V + 1) + 12 * F + 3 * s * F + 12 * F + 8 * k * V,
            "k_cot_product_wbar": 3 * s * F + 8 * k * V + 12 * F,
            "k_cot_vertex_grad": 4 * (V + 1) + 12 * F + 3 * s * F + 12 * F + 24 * V}


def step_a(v, f):
    x = v.detach().requires_grad_(True)
    loss = laplacian_regularizer(laplacian_cot(x, f), x)
    loss.backward()
    return loss.detach(), x.grad


def step_b(v, f):
    x = v.detach().requires_grad_(True)
    loss = laplacian_cot_product(x, f, x).square().mean()
    loss.backward()
    return loss.detach(), x.grad


def kernel_times(v, f, reps):
    """Per-kernel device times of (b) in microseconds: {name: [duration per launch]}."""
    act = torch.profiler.ProfilerActivity
    with torch.profiler.profile(activities=[act.CUDA]) as prof:
        for _ in range(reps):
            step_b(v, f)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        m = re.search(r"\b(k_cot\w*)<", e.name)
        out.setdefault(m.group(1) if m else "other (torch)", []).append(e.time_range.elapsed_us())
    return out


def run(name, reps, rounds):
    v, f = workload(name)
    V, F = v.shape[0], f.shape[0]
    face_incidence(f, V)                    # cached per faces tensor, as in a training loop
    print(f"{name}: V = {V}, F = {F}, int64 faces, k = 3")
    for what, fn in (("(a) laplacian_regularizer(laplacian_cot(v, f), v)", lambda: step_a(v, f)),
                     ("(b) laplacian_cot_product(v, f, v).square().mean()", lambda: step_b(v, f))):
        med, lo, hi = timed(fn, reps, rounds)
        print(f"  {what:52s} fwd + bwd {med:9.1f} us  [{lo:.1f} .. {hi:.1f}]")
    times = kernel_times(v, f, reps)
    nbytes = kernel_bytes(V, F, f.element_size(), 3)
    print(f"  kernels of (b), torch.profiler over {reps} steps (per launch):")
    for kname in ("k_cot", "k_cot_product", "k_cot_product_wbar", "k_cot_vertex_grad", "other (torch)"):
        d = times.get(kname, [])
        if not d:
            continue
        med = float(np.median(d))
        line = f"    {kname:20s} x{len(d) // reps} per step  {med:8.1f} us  [{min(d):.1f} .. {max(d):.1f}]"
        if kname in nbytes:
            bw = nbytes[kname] / (med * 1e-6)
            line += f"  {nbytes[kname] / 1e6:6.1f} MB -> {bw / 1e12:.2f} TB/s = {bw / HBM_PEAK:.2f} of 3.35 TB/s"
        print(line)
    la, ga = step_a(v, f)
    lb, gb = step_b(v, f)
    rel = lambda x, y: float(torch.linalg.norm((x - y).double()) / torch.linalg.norm(y.double()))
    print(f"  agreement (b) vs (a): loss rel {rel(lb, la):.2e}, gradient rel-L2 {rel(gb, ga):.2e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_cot_product.py needs a GPU"
    print("card:", card())
    for name in ("plane1000", "bunny_x2"):
        run(name, a.reps, a.rounds)


if __name__ == "__main__":
    main()
