"""Times the backward of point-to-mesh squared distances (ls_distance_grad_f32, largesteps_b200.distance) and the chamfer loss with
CUDA events, on bench_mesh_distance.py's four workload pairs (A's vertices queried against B):

    query_ms            the forward query (sqrD, I, C), B's BVH prebuilt
    bwd_P_ms            the backward with grad P only: one streaming kernel
    bwd_PV_ms           the backward with grad P and grad V: grad P, the queries bucketed by face, B's corners bucketed by
                        vertex, and one gather per vertex
    chamfer_fwd_bwd_ms  MeshDistance(VB, FB).chamfer(VA, FA) forward + backward w.r.t. VA (A's BVH built inside)

and one whole fitting step at bunny x2 (52,786 vertices, a noisy copy as the target): from_differential, chamfer, backward,
AdamUniform.  The byte model counts what each backward must move at least: grad P reads P, C, I and g and writes grad P
(60 bytes per query); grad V adds the bucket builds (I read twice and the query positions written and sorted: ~24 bytes per
query; the faces read twice and the corners written and sorted: ~2 x 3 x idx_bytes + 24 bytes per face) and the gather
(per query once per corner: P, C, g and its position, 56 bytes, times 3; per vertex its corners and grad V: ~6 x 4 + 12).
    python bench_distance_grad.py [--repeats R] [--warmup W]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "large-steps-pytorch_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import largesteps_b200._native as N  # noqa: E402
from largesteps_b200 import workloads  # noqa: E402
from largesteps_b200.distance import MeshDistance  # noqa: E402
from largesteps_b200.geometry import compute_matrix  # noqa: E402
from largesteps_b200.optimize import AdamUniform  # noqa: E402
from largesteps_b200.parameterize import from_differential, to_differential  # noqa: E402
from bench_mesh_distance import card, pairs, timed  # noqa: E402


def bwd_bytes(n, F, V, idx_bytes, with_v):
    b = n * (12 + 24 + 8 + 8 + 12)
    if with_v:
        b += n * 24 + F * (2 * 3 * idx_bytes + 24) + 3 * n * 56 + V * (6 * 4 + 12)
    return b


def backward(VB, FB, P, I, C, g, with_v):
    n, V, F = P.shape[0], VB.shape[0], FB.shape[0]
    dev = P.device
    gP = torch.empty((n, 3), dtype=torch.float32, device=dev)
    gV = torch.empty((V, 3), dtype=torch.float32, device=dev) if with_v else None
    nb = ctypes.c_size_t(0)
    N.check(N.lib().ls_distance_grad_workspace_bytes(n, F, V, ctypes.byref(nb)))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev) if with_v else None
    args = (N.ptr(P), n, N.ptr(VB), V, N.ptr(FB), FB.element_size(), F, N.ptr(I), N.ptr(C), N.ptr(g), N.ptr(gP), N.ptr(gV),
            N.ptr(ws), nb.value if with_v else 0, N.stream_ptr(dev))
    return lambda: N.check(N.lib().ls_distance_grad_f32(*args), "ls_distance_grad_f32")


def fit_step_ms(repeats, warmup):
    d = np.load(os.path.join(ROOT, "tests", "golden", "bunny_mesh.npz"))
    v, f = workloads.subdivide(*workloads.subdivide(d["verts"], d["faces"]))
    v = v.astype(np.float32)
    dev = "cuda"
    target = MeshDistance(torch.from_numpy((v + np.random.default_rng(1).normal(0, 1e-3, v.shape)).astype(np.float32)).to(dev),
                          torch.from_numpy(f).to(dev))
    tv, tf = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    M = compute_matrix(tv, tf, 19.0)
    u = to_differential(M, tv).clone().requires_grad_(True)
    opt = AdamUniform([u], lr=1e-2)

    def step():
        x = from_differential(M, u, "Cholesky")
        loss = target.chamfer(x, tf)
        opt.zero_grad()
        loss.backward()
        opt.step()

    return timed(step, repeats, warmup)[0], len(v)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_distance_grad.py needs a GPU"
    print(f"card: {card()}")
    dev = "cuda"
    for name, (va, fa), (vb, fb) in pairs():
        VA, FA = torch.from_numpy(va).to(dev), torch.from_numpy(fa).to(dev)
        VB, FB = torch.from_numpy(vb).to(dev), torch.from_numpy(fb).to(dev)
        mb = MeshDistance(VB, FB)
        _, I, C = mb.squared_distance(VA)
        g = torch.full((len(va),), 1.0 / len(va), dtype=torch.float64, device=dev)
        t_q, _ = timed(lambda: mb.squared_distance(VA), args.repeats, args.warmup)
        t_p, _ = timed(backward(VB, FB, VA, I, C, g, False), args.repeats, args.warmup)
        t_pv, _ = timed(backward(VB, FB, VA, I, C, g, True), args.repeats, args.warmup)
        VAg = VA.clone().requires_grad_(True)

        def cham():
            VAg.grad = None
            mb.chamfer(VAg, FA).backward()

        t_c, _ = timed(cham, args.repeats, args.warmup)
        rec = {"workload": name, "VA": len(va), "FA": len(fa), "VB": len(vb), "FB": len(fb),
               "query_ms": round(t_q, 3), "bwd_P_ms": round(t_p, 3), "bwd_PV_ms": round(t_pv, 3),
               "chamfer_fwd_bwd_ms": round(t_c, 3),
               "bwd_P_GBps_model": round(bwd_bytes(len(va), len(fb), len(vb), 8, False) / t_p / 1e6, 1),
               "bwd_PV_GBps_model": round(bwd_bytes(len(va), len(fb), len(vb), 8, True) / t_pv / 1e6, 1)}
        print(json.dumps(rec))
    t_fit, V = fit_step_ms(args.repeats, args.warmup)
    print(json.dumps({"workload": "fit_step_bunny2", "V": V, "step_ms": round(t_fit, 3)}))


if __name__ == "__main__":
    main()
