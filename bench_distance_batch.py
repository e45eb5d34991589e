"""Times the batched distances (largesteps_b200.distance: MeshDistanceBatch, hausdorff_batch) with CUDA events against the
per-mesh loops they replace, on three workloads:

    trajectory   100 iterates of the bunny subdivided twice (52,786 vertices, seeded noise) scored against one target:
                 hausdorff_batch in its broadcast form vs the comparison figure's loop of 200 hausdorff calls
                 (hausdorff(it, target) + hausdorff(target, it) per iterate, each synchronising)
    chamfer      MeshDistanceBatch(targets).chamfer forward + backward vs a loop of MeshDistance(target_b).chamfer, for 64
                 icosphere(4) against 64 targets and for 16 bunnies against 16 targets
    step         a whole fitting step (from_differential_batch, the chamfer, backward, AdamUniform) vs the same step with a
                 per-mesh loop for the solve and the loss, at the two chamfer sizes

plus the forest build and one query direction alone.  Each figure is the median (min - max) of --repeats timed runs after
--warmup untimed ones.  The byte model counts what a build and a query must move at least (bench_mesh_distance.py's
model): neither is bandwidth-bound, so the GB/s figures only show how far from the 3.35 TB/s of HBM3 each runs.
    python bench_distance_batch.py [--repeats R] [--warmup W]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "large-steps-pytorch_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from largesteps_b200 import workloads  # noqa: E402
from largesteps_b200.batch import from_differential_batch, pack_meshes  # noqa: E402
from largesteps_b200.distance import MeshDistance, MeshDistanceBatch, hausdorff, hausdorff_batch  # noqa: E402
from largesteps_b200.geometry import compute_matrix  # noqa: E402
from largesteps_b200.optimize import AdamUniform  # noqa: E402
from largesteps_b200.parameterize import from_differential, to_differential  # noqa: E402

DEV = "cuda"


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def timed(fn, repeats, warmup):
    """median, min and max in ms of fn() between CUDA events"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(repeats)]
    for a, b in ev:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = sorted(a.elapsed_time(b) for a, b in ev)
    return {"median": round(ms[len(ms) // 2], 3), "min": round(ms[0], 3), "max": round(ms[-1], 3)}


def build_bytes(F, idx_bytes):
    # bench_mesh_distance.py's model: faces and corners twice, centroids and fine codes, the leaves and nodes written and read
    return F * (2 * 3 * idx_bytes + 2 * 36 + 36 + 8 + 48 + 64 + 2 * 48)


def query_bytes(n):
    return n * (12 + 8 + 8 + 24)


def t(x, dtype=None):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV) if dtype is None else torch.from_numpy(np.ascontiguousarray(x)).to(DEV, dtype)


def noisy(v, sigma, seed):
    return (v + np.random.default_rng(seed).normal(0, sigma, size=v.shape)).astype(np.float32)


def bunny():
    d = np.load(os.path.join(ROOT, "tests", "golden", "bunny_mesh.npz"))
    return d["verts"].astype(np.float32), d["faces"].astype(np.int64)


def trajectory(args):
    v, f = workloads.subdivide(*workloads.subdivide(*bunny()))
    v = v.astype(np.float32)
    vt, ft = t(v), t(f)
    its = [t(noisy(v, 1e-3 * (1 + k % 5), 100 + k)) for k in range(100)]
    p = pack_meshes(its, [ft] * 100)
    to, fo = [0, len(v)], [0, len(f)]

    def batch():
        return hausdorff_batch(*p[:4], vt, ft, to, fo)

    def loop():
        return [hausdorff(x, ft, vt, ft) + hausdorff(vt, ft, x, ft) for x in its]

    got, want = batch().tolist(), loop()
    assert [2 * g for g in got] == want, "the batch must give the loop's scores"
    q = MeshDistance(vt, ft)
    forest, tiled = MeshDistanceBatch(*p[:4]), vt.repeat(100, 1)   # built outside the timed query
    return {"workload": "trajectory", "iterates": 100, "V": len(v), "F": len(f),
            "batch_ms": timed(batch, args.repeats, args.warmup), "loop_ms": timed(loop, max(3, args.repeats // 4), 1),
            "build_forest_ms": timed(lambda: MeshDistanceBatch(*p[:4]), args.repeats, args.warmup),
            "query_forest_ms": timed(lambda: forest.squared_distance(tiled, p.vert_offsets), args.repeats, args.warmup),
            "query_target_ms": timed(lambda: q.squared_distance(p.verts), args.repeats, args.warmup), "F_forest": 100 * len(f)}


def chamfer_case(name, B, mesh, target):
    vs = [noisy(mesh[0], 1e-3, k) for k in range(B)]
    ts = [(noisy(target[0] * np.float32(1.0 + 0.01 * (k % 7)), 2e-3, 1000 + k), target[1]) for k in range(B)]
    return name, [(v, mesh[1]) for v in vs], ts


def chamfer_cases():
    v4, f4 = workloads.icosphere(4)
    yield chamfer_case("ico4_x64", 64, (v4, f4), (v4 * np.float32(1.1), f4))
    b = bunny()
    yield chamfer_case("bunny_x16", 16, b, (b[0] * np.float32(1.05), b[1]))


def chamfer_bench(args, name, meshes, targets):
    pA = pack_meshes([t(v) for v, _ in meshes], [t(f) for _, f in meshes])
    pT = pack_meshes([t(v) for v, _ in targets], [t(f) for _, f in targets])
    target = MeshDistanceBatch(*pT[:4])
    singles = [MeshDistance(t(v), t(f)) for v, f in targets]
    VA = pA.verts.clone().requires_grad_(True)
    parts = [t(v).requires_grad_(True) for v, _ in meshes]
    fs = [t(f) for _, f in meshes]

    def batch():
        VA.grad = None
        target.chamfer(VA, *pA[1:4]).sum().backward()

    def loop():
        for x in parts:
            x.grad = None
        sum(s.chamfer(x, f) for s, x, f in zip(singles, parts, fs)).backward()

    F = pT.face_offsets_host[-1]
    n = pA.vert_offsets_host[-1]
    rec = {"workload": "chamfer", "case": name, "B": len(meshes), "V_each": len(meshes[0][0]), "F_target_each": len(targets[0][1]),
           "batch_ms": timed(batch, args.repeats, args.warmup), "loop_ms": timed(loop, args.repeats, args.warmup),
           "build_forest_ms": timed(lambda: MeshDistanceBatch(*pT[:4]), args.repeats, args.warmup),
           "query_forest_ms": timed(lambda: target.squared_distance(pA.verts, pA.vert_offsets), args.repeats, args.warmup)}
    rec["build_forest_GBps_model"] = round(build_bytes(F, 8) / rec["build_forest_ms"]["median"] / 1e6, 1)
    rec["query_forest_GBps_model"] = round(query_bytes(n) / rec["query_forest_ms"]["median"] / 1e6, 1)
    return rec


def step_bench(args, name, meshes, targets):
    pA = pack_meshes([t(v) for v, _ in meshes], [t(f) for _, f in meshes])
    pT = pack_meshes([t(v) for v, _ in targets], [t(f) for _, f in targets])
    target = MeshDistanceBatch(*pT[:4])
    singles = [MeshDistance(t(v), t(f)) for v, f in targets]
    vs = [t(v) for v, _ in meshes]
    fs = [t(f) for _, f in meshes]
    Ms = [compute_matrix(v, f, 19.0) for v, f in zip(vs, fs)]
    ub = [to_differential(M, v).clone().requires_grad_(True) for M, v in zip(Ms, vs)]
    ul = [u.detach().clone().requires_grad_(True) for u in ub]
    ob, ol = AdamUniform(ub, lr=1e-3), AdamUniform(ul, lr=1e-3)

    def batch():
        ob.zero_grad()
        x = from_differential_batch(Ms, ub, packed=True)
        target.chamfer(x, *pA[1:4]).sum().backward()
        ob.step()

    def loop():
        ol.zero_grad()
        sum(s.chamfer(from_differential(M, u), f) for s, M, u, f in zip(singles, Ms, ul, fs)).backward()
        ol.step()

    return {"workload": "step", "case": name, "B": len(meshes),
            "batch_ms": timed(batch, args.repeats, args.warmup), "loop_ms": timed(loop, args.repeats, args.warmup)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_distance_batch.py needs a GPU"
    print(json.dumps({"card": card()}))
    rec = trajectory(args)
    rec["build_forest_GBps_model"] = round(build_bytes(rec["F_forest"], 8) / rec["build_forest_ms"]["median"] / 1e6, 1)
    print(json.dumps(rec))
    for name, meshes, targets in chamfer_cases():
        print(json.dumps(chamfer_bench(args, name, meshes, targets)))
        print(json.dumps(step_bench(args, name, meshes, targets)))


if __name__ == "__main__":
    main()
