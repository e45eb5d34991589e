"""A/B of builds of the fused solver on bench.py's figure of record (plane 1000x1000, V = 1e6, 3 columns, Jacobi-PCG) and on
the 4e6 plane and config 4's 250K mesh beside it.

    python bench_phase_a.py [--rounds 4] [--steps 100] [--warmup 5] [--workloads plane1000,...] [--out FILE] [NAME=LIB.so ...]

Every build is loaded into the same process (each library is a separate copy of the native code, solver handles are
created by the build that runs them) and the builds are timed alternately, round after round, on the same matrix and
right-hand sides, so that clock and neighbour drift spreads over all of them.  Without NAME=LIB arguments the builds are
libls_b200.so ("base") and every libls_b200_<name>.so next to it (csrc/build_variant.sh).  Reports per build: solves/s
(median and range over the rounds), CG iterations, whether the solution is bit-identical to the first build's, and the
per-phase SM cycles per iteration of the profiling instantiation (LS_PCG_PROFILE=1), on CTA 0 and over all CTAs.
Prints one JSON object; --out also writes it to a file.
"""
import argparse
import glob
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(ROOT, "large-steps-pytorch_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

PHASES = ("phaseA", "sync_ps", "phaseB", "sync_rz")


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return dict(zip(q.split(","), [s.strip() for s in out.split(",")]))
    except Exception as e:   # the timing itself does not depend on nvidia-smi
        return {"error": str(e)}


def load(N, path):
    """Load one build; returns its ctypes handle (N.lib() of that build)."""
    N._lib = None
    N.LIB_PATH = path
    return N.lib()


def per_cta_split(pc, it):
    """Per-CTA phase cycles per iteration: min / median / max over CTAs, and for each all-reduce the part every CTA pays
    (its minimum over CTAs: the fixed cost) against the part the CTAs wait for the slowest one (median - minimum: skew)."""
    rows = pc["per_cta"]
    out = {}
    for j, nm in enumerate(PHASES):
        v = sorted(r[j] / max(r[7], 1) for r in rows)
        out[nm] = {"min": round(v[0]), "median": round(statistics.median(v)), "max": round(v[-1])}
    work = sorted((r[0] + r[2]) / max(r[7], 1) for r in rows)
    out["work_A_plus_B"] = {"min": round(work[0]), "median": round(statistics.median(work)), "max": round(work[-1])}
    for nm in ("sync_ps", "sync_rz"):
        out[nm]["fixed"] = out[nm]["min"]
        out[nm]["skew"] = out[nm]["median"] - out[nm]["min"]
    out["ctas"] = len(rows)
    out["distinct_sms"] = len({r[6] for r in rows})
    return out


def run_workload(args, bench, N, torch, libs, names, builds, wl, dev):
    from largesteps_b200.geometry import compute_matrix
    from largesteps_b200.parameterize import to_differential
    from largesteps_b200.solvers import CholeskySolver

    steps = {"plane2000": max(args.steps // 10, 5)}.get(wl, args.steps)
    v, f, kw = bench.build_mesh(bench.WORKLOADS[wl], seed=0)
    V = v.shape[0]
    N._lib = libs[names[0]]
    tv, tf = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    M = compute_matrix(tv, tf, **kw)
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    us = []
    for i in range(4):
        vv = tv + 0.01 * torch.randn(V, 3, device=dev, generator=gen)
        us.append((to_differential(M, vv) + 0.01 * torch.randn(V, 3, device=dev, generator=gen)).contiguous())

    solvers = {}
    for name in names:
        N._lib = libs[name]
        solvers[name] = CholeskySolver(M)

    res = {name: {"path": os.path.relpath(path, ROOT), "solves_per_s": []} for name, path in builds}
    ref_x = None
    for name in names:                # bits and iterations, before any timing
        N._lib = libs[name]
        with torch.no_grad():
            x = solvers[name].solve(us[0])
        res[name]["iterations"] = solvers[name].iterations
        solvers[name].raise_for_status()
        if ref_x is None:
            ref_x = x
        res[name]["bitwise_equal_to_" + names[0]] = bool(torch.equal(x.view(torch.int32), ref_x.view(torch.int32)))

    for rnd in range(args.rounds):
        order = names[rnd % len(names):] + names[:rnd % len(names)]     # rotate who goes first
        for name in order:
            N._lib = libs[name]
            s = solvers[name]
            with torch.no_grad():
                for i in range(args.warmup):
                    s.solve(us[i % 4])
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(steps):
                    s.solve(us[i % 4])
                e1.record()
                torch.cuda.synchronize()
            res[name]["solves_per_s"].append(steps / (e0.elapsed_time(e1) * 1e-3))

    desc = solvers[names[0]].describe()
    if desc.get("algo") == "fused" and desc.get("precond") == "jacobi" and desc.get("residency") in (1, 2):
        os.environ["LS_PCG_PROFILE"] = "1"      # (the profiling instantiations: Jacobi, RES 1 and 2)
        try:
            for name in names:
                N._lib = libs[name]
                s = solvers[name]
                with torch.no_grad():
                    s.solve(us[0])
                pc = s.phase_cycles(per_cta=True)
                it = max(pc["iterations"], 1)
                res[name]["phase_cycles_per_iteration_cta0"] = {k: round(pc[k] / it) for k in PHASES}
                res[name]["phase_cycles_per_iteration_per_cta"] = per_cta_split(pc, it)
        finally:
            del os.environ["LS_PCG_PROFILE"]

    for name in names:
        sps = res[name]["solves_per_s"]
        res[name]["median"] = statistics.median(sps)
        res[name]["range"] = [min(sps), max(sps)]
    s = None
    for name in names:                # each handle is destroyed by the build that created it
        N._lib = libs[name]
        del solvers[name]
    return {"workload": bench.WORKLOADS[wl]["desc"], "steps": steps, "solver": desc, "builds": res}

def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("builds", nargs="*", help="NAME=path/to/libls_b200*.so (default: the in-tree build and its variants)")
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--workloads", default="plane1000,plane2000,plane500",
                    help="bench.py workloads, comma-separated (default: the figure of record, the 4e6 plane, config 4's mesh)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from largesteps_b200 import _native as N
    import bench

    if not torch.cuda.is_available():
        raise SystemExit("bench_phase_a.py needs a GPU")
    if args.builds:
        builds = [tuple(b.split("=", 1)) for b in args.builds]
    else:
        here = os.path.join(PKG, "largesteps_b200")
        builds = [("base", os.path.join(here, "libls_b200.so"))]
        builds += [(os.path.basename(p)[len("libls_b200_"):-3], p) for p in sorted(glob.glob(os.path.join(here, "libls_b200_*.so")))]
    dev = torch.device("cuda", 0)
    libs = {name: load(N, path) for name, path in builds}

    names = [n for n, _ in builds]
    info_before = gpu_info()
    sampler = bench.ClockSampler(0)
    sampler.start()
    per_wl = {}
    for wl in args.workloads.split(","):
        per_wl[wl] = run_workload(args, bench, N, torch, libs, names, builds, wl, dev)
    clocks = sampler.stop()
    out = {"rounds": args.rounds, "warmup": args.warmup, "gpu": info_before, "clocks_during_timing": clocks,
           "workloads": per_wl,
           "how": "all builds loaded in one process, timed alternately (rotated order per round), CUDA events around "
                  "back-to-back asynchronous solves; phase cycles from the profiling instantiation, one solve"}
    s = json.dumps(out, indent=1)
    print(s)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(s)


if __name__ == "__main__":
    main()
