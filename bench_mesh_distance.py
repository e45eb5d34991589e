"""Times the point-to-mesh distance path (largesteps_b200.distance) with CUDA events: the BVH build, each query direction and
the whole hausdorff call, on four workload pairs:

    plane      workloads.plane(1000) vs plane(1000, seed=1)         V = 1e6, F = 1,996,002 each
    plane_shuffled  the same with both meshes' faces in a seeded random order (as a remesher may number them)
    bunny2     bunny subdivided twice (52,786 vertices) vs a noisy copy (sigma = 1e-3 of its unit scale)
    ico        icosphere(6) vs 1.01 x icosphere(4)

The byte model counts what each step must move at least: a build reads the faces and their corners and writes the BVH; a
query reads its points and writes sqrD, I and C (52 bytes per point).  Neither is bandwidth-bound: a query walks the tree with
one thread per point and does its leaf tests in fp64, so the rates below are set by that latency and fp64 work, and
the bytes/s figures only show how far from the 3.35 TB/s of HBM3 each step runs.
    python bench_mesh_distance.py [--repeats R] [--warmup W] [--numpy-model]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "large-steps-pytorch_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from largesteps_b200 import workloads  # noqa: E402
from largesteps_b200.distance import MeshDistance, hausdorff  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def pairs():
    va, fa = workloads.plane(1000)
    vb, fb = workloads.plane(1000, seed=1)
    yield "plane", (va, fa), (vb, fb)
    rng = np.random.default_rng(7)
    yield "plane_shuffled", (va, fa[rng.permutation(len(fa))]), (vb, fb[rng.permutation(len(fb))])
    d = np.load(os.path.join(ROOT, "tests", "golden", "bunny_mesh.npz"))
    v, f = workloads.subdivide(*workloads.subdivide(d["verts"], d["faces"]))
    v = v.astype(np.float32)
    yield "bunny2", (v, f), ((v + np.random.default_rng(1).normal(0, 1e-3, v.shape)).astype(np.float32), f)
    (va, fa), (vb, fb) = workloads.icosphere(6), workloads.icosphere(4)
    yield "ico", (va, fa), ((vb * np.float32(1.01)).astype(np.float32), fb)


def timed(fn, repeats, warmup):
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
    return ms[len(ms) // 2], ms[0]


def build_bytes(V, F, idx_bytes):
    # faces twice (centroids, leaves), corners twice, centroids written and read twice (ordering, fine codes), fine codes
    # written and read, the BVH's leaves and nodes written and its leaves read by the tree and refit passes
    return F * (2 * 3 * idx_bytes + 2 * 36 + 36 + 8 + 48 + 64 + 2 * 48)


def query_bytes(n):
    return n * (12 + 8 + 8 + 24)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--numpy-model", action="store_true", help="also time the tests' float64 numpy model on 4096 queries")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_mesh_distance.py needs a GPU"
    print(f"card: {card()}")
    dev = "cuda"
    for name, (va, fa), (vb, fb) in pairs():
        VA, FA = torch.from_numpy(va).to(dev), torch.from_numpy(fa).to(dev)
        VB, FB = torch.from_numpy(vb).to(dev), torch.from_numpy(fb).to(dev)
        mb = MeshDistance(VB, FB)
        ma = MeshDistance(VA, FA)
        t_build, _ = timed(lambda: MeshDistance(VB, FB), args.repeats, args.warmup)
        t_ab, _ = timed(lambda: mb.squared_distance(VA), args.repeats, args.warmup)
        t_ba, _ = timed(lambda: ma.squared_distance(VB), args.repeats, args.warmup)
        t_h, _ = timed(lambda: mb.hausdorff(VA, FA), args.repeats, args.warmup)
        t_h2, _ = timed(lambda: hausdorff(VA, FA, VB, FB), args.repeats, args.warmup)
        t0 = time.perf_counter()
        h = mb.hausdorff(VA, FA)
        t_h_host = (time.perf_counter() - t0) * 1e3
        rec = {"workload": name, "VA": len(va), "FA": len(fa), "VB": len(vb), "FB": len(fb), "hausdorff": h,
               "build_ms": round(t_build, 3), "query_AB_ms": round(t_ab, 3), "query_BA_ms": round(t_ba, 3),
               "hausdorff_B_prebuilt_ms": round(t_h, 3), "hausdorff_B_prebuilt_host_ms": round(t_h_host, 3),
               "hausdorff_both_builds_ms": round(t_h2, 3),
               "query_AB_Mpts_per_s": round(len(va) / t_ab / 1e3, 1),
               "build_GBps_model": round(build_bytes(len(vb), len(fb), 8) / t_build / 1e6, 1),
               "query_AB_GBps_model": round(query_bytes(len(va)) / t_ab / 1e6, 1)}
        if args.numpy_model:
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            import distance_model
            sel = np.random.default_rng(0).choice(len(va), min(4096, len(va)), replace=False)
            t0 = time.perf_counter()
            distance_model.point_mesh(va[sel], vb, fb)
            rec["numpy_model_ms_per_4096_queries"] = round((time.perf_counter() - t0) * 1e3, 1)
        print(json.dumps(rec))


if __name__ == "__main__":
    main()
