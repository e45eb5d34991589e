"""Batched solve vs a loop of single solves: from_differential_batch(Ms, us) against [from_differential(M_i, u_i)] on the same
meshes, the same stream, asynchronous solves (check=False), timed with CUDA events after warm-up.

    python bench_batch.py [--reps R] [--rounds N] [--json] [--precond jacobi,chebyshev,mixed]

Prints the card name, power limit and clocks, then per workload meshes x solves per second for both arms and the worst
per-mesh rel-L2 error of each arm against the fp64 direct solve.  --precond picks the batch's preconditioner: 'jacobi',
'chebyshev', or 'mixed' (Chebyshev for the alpha >= 0.99 members of an alpha sweep, Jacobi elsewhere); a comma-separated
list times each in turn, alternating them for --rounds rounds in the same session, and prints each batch arm's per-mesh
outer-iteration counts.  Writes nothing to disk.
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
from largesteps_b200 import batch as B
from largesteps_b200.batch import from_differential_batch
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.parameterize import from_differential

DEV = "cuda:0"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
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


def preconds(cases, mode):
    """the batch's per-mesh preconditioners for --precond mode"""
    if mode == "mixed":
        return ["chebyshev" if kw.get("alpha", 0.0) >= 0.99 else "jacobi" for _, _, kw in cases]
    return [mode] * len(cases)


def run(name, reps, modes=("jacobi",), rounds=1):
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

    def batched(mode):
        return lambda: from_differential_batch(Ms, us, precond=preconds(cases, mode))

    def worst(xs):
        return max(rel_l2(x.cpu().numpy().astype(np.float64), d.solve(u.cpu().numpy())) for x, u, d in zip(xs, us, direct))

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / reps

    arms = {"loop": loop}
    arms.update({"batch" if modes == ("jacobi",) else f"batch_{m}": batched(m) for m in modes})
    out, times = {}, {a: [] for a in arms}
    for a, fn in list(arms.items()):   # warm-up (and, for the batch, the solver build), accuracy
        try:
            for _ in range(3):
                xs = fn()
        except ValueError as e:   # a mesh larger than one cluster with this preconditioner
            out[a] = dict(rejected=str(e))
            del arms[a]
            continue
        torch.cuda.synchronize()
        out[a] = dict(worst_rel_l2=worst(xs))
        if a != "loop":
            out[a]["iterations"] = B._cache[_key(Ms, preconds(cases, a.split("_", 1)[1] if "_" in a else "jacobi"))][0].iterations
    for _ in range(rounds):      # the arms alternate, round after round
        for a, fn in arms.items():
            times[a].append(timed(fn))
    for a in arms:
        ms = float(np.median(times[a]))
        out[a].update(ms_per_call=ms, mesh_solves_per_s=len(Ms) * 1000.0 / ms, ms_rounds=times[a])
    V = [M.shape[0] for M in Ms]
    res = dict(workload=name, meshes=len(Ms), V_min=min(V), V_max=max(V), **out)
    for a in arms:
        if a != "loop":
            res["speedup" if a == "batch" else f"speedup_{a}"] = out["loop"]["ms_per_call"] / out[a]["ms_per_call"]
    return res


def _key(Ms, ps):
    key = (tuple(id(M) for M in Ms), "Cholesky")
    return key + (tuple(ps),) if any(p != "jacobi" for p in ps) else key


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=1, help="timed rounds per arm, the arms alternating (median reported)")
    ap.add_argument("--json", action="store_true")
    ap.add_argument("--workloads", default="ico4_x64,plane150_alpha_x8,bunny_x16,bunny2_x4",
                    help="comma-separated <base>_x<meshes>, base in ico4, plane150_alpha, bunny, bunny2")
    ap.add_argument("--precond", default="jacobi",
                    help="comma-separated batch preconditioners: jacobi, chebyshev, mixed (Chebyshev for alpha >= 0.99)")
    a = ap.parse_args()
    modes = tuple(a.precond.split(","))
    for m in modes:
        if m not in ("jacobi", "chebyshev", "mixed"):
            ap.error(f"unknown --precond {m!r}")
    if not torch.cuda.is_available():
        sys.exit("bench_batch.py needs a GPU")
    print(f"card: {card()}", flush=True)
    for w in a.workloads.split(","):
        r = run(w, a.reps, modes, a.rounds)
        if a.json:
            print(json.dumps(r), flush=True)
            continue
        line = (f"{r['workload']:>18}: {r['meshes']:3d} meshes, V {r['V_min']}..{r['V_max']}:  "
                f"loop {r['loop']['mesh_solves_per_s']:9.0f} mesh-solves/s ({r['loop']['ms_per_call']:.3f} ms, worst err {r['loop']['worst_rel_l2']:.1e})")
        for k, v in r.items():
            if k.startswith("batch") and "rejected" in v:
                line += f"   {k} rejected ({v['rejected']})"
            elif k.startswith("batch"):
                s = r["speedup" if k == "batch" else "speedup_" + k]
                line += (f"   {k} {v['mesh_solves_per_s']:9.0f} mesh-solves/s ({v['ms_per_call']:.3f} ms, worst err {v['worst_rel_l2']:.1e}) "
                         f"{k}/loop {s:.2f}x")
        print(line, flush=True)
        if modes != ("jacobi",):
            for k, v in r.items():
                if k.startswith("batch") and "iterations" in v:
                    print(f"{'':>20}{k} iterations per mesh: {v['iterations']}", flush=True)


if __name__ == "__main__":
    main()
