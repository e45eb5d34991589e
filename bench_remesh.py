"""Times largesteps_b200.remesh.remesh_botsch(v, f, 5, h, True), the reference loop's remesh call (scripts/main.py:149), on
the device at h = 0.5 x the mean edge length (the mesh roughly quadruples), on:

    bunny      the golden bunny (3,301 vertices)
    ico6/7/8   icosphere level 6, 7, 8 (41K, 164K, 655K vertices) with seeded Gaussian noise of 0.1 x the mean edge length

Two arms per case:
    uniform    the scalar h above
    adaptive   a graded per-vertex target t_i = h (0.5 + 1.5 s_i), s_i the vertex's normalised x coordinate (a 4x ratio
               across the mesh), and feature vertices: a seeded 2 % of them plus the band |y - median y| < 0.4 x the mean
               edge, a pinned crease

Each call is timed with a host clock around the call and a device synchronise (the call itself reads counts back once per
stage and round, so it synchronises anyway); the per-stage split comes from CUDA events recorded between the stages.
    python bench_remesh.py [--repeats R] [--warmup W] [--cases bunny,ico6,...] [--arms uniform,adaptive]
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
from largesteps_b200.remesh import remesh_botsch  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or f"{torch.cuda.get_device_name(0)}, power limit unknown"


def workload(name):
    if name == "bunny":
        d = np.load(os.path.join(ROOT, "tests", "golden", "bunny_mesh.npz"))
        return d["verts"].astype(np.float32), d["faces"].astype(np.int64)
    v, f = workloads.icosphere(int(name[3:]))
    v, f = np.asarray(v, np.float32), np.asarray(f, np.int64)
    mean = float(np.linalg.norm(v[f[:, 1]] - v[f[:, 0]], axis=1).mean())
    return (v + np.random.default_rng(0).normal(size=v.shape) * 0.1 * mean).astype(np.float32), f


def adaptive_arguments(v, f, h, dev):
    """The adaptive arm's per-vertex target (float64) and feature mask."""
    x = v[:, 0].astype(np.float64)
    t = h * (0.5 + 1.5 * (x - x.min()) / (x.max() - x.min()))
    mean = float(np.linalg.norm(v[f[:, 1]] - v[f[:, 0]], axis=1).mean())
    feat = np.zeros(len(v), bool)
    feat[np.random.default_rng(0).choice(len(v), max(1, len(v) // 50), replace=False)] = True
    feat |= np.abs(v[:, 1] - np.median(v[:, 1])) < 0.4 * mean
    return torch.from_numpy(t).to(dev), torch.from_numpy(feat).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--cases", default="bunny,ico6,ico7,ico8")
    ap.add_argument("--arms", default="uniform,adaptive")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_remesh.py needs a GPU")
    dev = "cuda:0"
    print(json.dumps({"card": card()}))
    for name in a.cases.split(","):
        v, f = workload(name)
        h = 0.5 * float(np.linalg.norm(v[f[:, 1]] - v[f[:, 0]], axis=1).mean())
        tv, tf = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
        for arm in a.arms.split(","):
            if arm == "uniform":
                call = lambda **kw: remesh_botsch(tv, tf, 5, h, True, **kw)
            elif arm == "adaptive":
                t, feat = adaptive_arguments(v, f, h, dev)
                call = lambda **kw: remesh_botsch(tv, tf, 5, t, True, feature=feat, **kw)
            else:
                sys.exit(f"unknown arm {arm!r}")
            for _ in range(a.warmup):
                call()
            torch.cuda.synchronize()
            times, stages = [], {}
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                vo, fo = call()
                torch.cuda.synchronize()
                times.append(1e3 * (time.perf_counter() - t0))
            call(stage_ms=stages)
            print(json.dumps({"case": name, "arm": arm, "V_in": int(v.shape[0]), "V_out": int(vo.shape[0]), "F_out": int(fo.shape[0]),
                              "ms_median": round(float(np.median(times)), 2), "ms_min": round(min(times), 2),
                              "ms_max": round(max(times), 2), "stage_ms": {k: round(x, 2) for k, x in stages.items()}}))


if __name__ == "__main__":
    main()
