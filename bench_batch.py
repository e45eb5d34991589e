"""Batched solve vs a loop of single solves: from_differential_batch(Ms, us) against [from_differential(M_i, u_i)] on the same
meshes, the same stream, asynchronous solves (check=False), timed with CUDA events after warm-up.

    python bench_batch.py [--reps R] [--json]

Prints the card name and power limit, then per workload meshes x solves per second for both arms and the worst per-mesh
rel-L2 error of each arm against the fp64 direct solve.  Writes nothing to disk.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "large-steps-pytorch_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

import oracle
from largesteps_b200 import workloads
from largesteps_b200.batch import from_differential_batch
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.parameterize import from_differential

DEV = "cuda:0"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0)


def noisy(v, sigma, seed):
    return (v + np.random.default_rng(seed).normal(0, sigma, size=v.shape)).astype(np.float32)


def bunny():
    d = np.load(os.path.join(ROOT, "tests", "golden", "bunny_mesh.npz"))
    return d["verts"].astype(np.float32), d["faces"].astype(np.int64)


def workload(name):
    """'<base>_x<n>' -> n (verts, faces, compute_matrix kwargs) with distinct matrices"""
    base, n = name.rsplit("_x", 1)
    n = int(n)
    if base == "ico4":          # noisy icospheres, cotan weights
        v, f = workloads.icosphere(4)
        return [(noisy(v, 0.01, s), f, dict(lambda_=19.0, cotan=True)) for s in range(n)]
    if base == "plane150_alpha":  # an alpha sweep on one plane
        v, f = workloads.plane(150, seed=0)
        alphas = (0.5, 0.7, 0.8, 0.9, 0.95, 0.98, 0.99, 0.995)
        return [(v, f, dict(lambda_=1.0, alpha=alphas[s % len(alphas)])) for s in range(n)]
    if base == "bunny":
        v, f = bunny()
        return [(noisy(v, 1e-4, s), f, dict(lambda_=19.0, cotan=True)) for s in range(n)]
    if base == "bunny2":        # the bunny subdivided twice, 52,786 vertices
        v, f = bunny()
        v, f = workloads.subdivide(*workloads.subdivide(v, f))
        return [(noisy(v.astype(np.float32), 1e-4, s), f, dict(lambda_=19.0, cotan=True)) for s in range(n)]
    raise ValueError(name)


def rel_l2(x, y):
    return float(np.linalg.norm(x - y) / max(np.linalg.norm(y), 1e-300))


def run(name, reps):
    cases = workload(name)
    Ms, us, direct = [], [], []
    for i, (v, f, kw) in enumerate(cases):
        tv = torch.from_numpy(v).to(DEV)
        tf = torch.from_numpy(f).to(DEV)
        Ms.append(compute_matrix(tv, tf, **kw))
        r, c, val, V = oracle.compute_matrix(v, f, **kw)
        A = oracle.coo_to_scipy(r, c, val, V)
        b = workloads.rhs_recipe(lambda x: A @ x, v, seed0=3 * i, seed1=3 * i + 1, seed2=3 * i + 2)[1]
        us.append(torch.from_numpy(b).to(DEV))
        direct.append(oracle.DirectSolver(r, c, val, V))

    def loop():
        return [from_differential(M, u) for M, u in zip(Ms, us)]

    def batched():
        return from_differential_batch(Ms, us)

    out = {}
    for arm, fn in (("loop", loop), ("batch", batched)):
        for _ in range(3):
            xs = fn()
        torch.cuda.synchronize()
        err = max(rel_l2(x.cpu().numpy().astype(np.float64), d.solve(u.cpu().numpy())) for x, u, d in zip(xs, us, direct))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        ms = e0.elapsed_time(e1) / reps
        out[arm] = dict(ms_per_call=ms, mesh_solves_per_s=len(Ms) * 1000.0 / ms, worst_rel_l2=err)
    V = [M.shape[0] for M in Ms]
    return dict(workload=name, meshes=len(Ms), V_min=min(V), V_max=max(V), **out,
                speedup=out["loop"]["ms_per_call"] / out["batch"]["ms_per_call"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", action="store_true")
    ap.add_argument("--workloads", default="ico4_x64,plane150_alpha_x8,bunny_x16,bunny2_x4",
                    help="comma-separated <base>_x<meshes>, base in ico4, plane150_alpha, bunny, bunny2")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch.py needs a GPU")
    print(f"card: {card()}", flush=True)
    for w in a.workloads.split(","):
        r = run(w, a.reps)
        if a.json:
            print(json.dumps(r), flush=True)
        else:
            print(f"{r['workload']:>18}: {r['meshes']:3d} meshes, V {r['V_min']}..{r['V_max']}:  "
                  f"loop {r['loop']['mesh_solves_per_s']:9.0f} mesh-solves/s ({r['loop']['ms_per_call']:.3f} ms, worst err {r['loop']['worst_rel_l2']:.1e})   "
                  f"batch {r['batch']['mesh_solves_per_s']:9.0f} mesh-solves/s ({r['batch']['ms_per_call']:.3f} ms, worst err {r['batch']['worst_rel_l2']:.1e})   "
                  f"batch/loop {r['speedup']:.2f}x", flush=True)


if __name__ == "__main__":
    main()
