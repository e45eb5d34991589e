"""Whole optimisation steps for B meshes: the per-mesh loop against the batched step, in steps per second.

    python bench_batch_loop.py [--reps R] [--warmup W] [--workloads ico4_x1,ico4_x4,...] [--json]

loop   per mesh: from_differential -> compute_face_normals -> compute_vertex_normals, one loss over all meshes, backward, then
       the per-parameter AdamUniform step (one ls_adam_uniform_step call, i.e. a ctypes call, a memset and two kernels, per mesh)
batch  from_differential_batch(packed=True) -> compute_face_normals and compute_vertex_normals_batch on the packed meshes,
       backward, then AdamUniform.step() (ls_adam_uniform_step_multi: two kernels for all meshes)

Both arms use the same stand-in loss, squared distances of the vertex normals and positions to fixed targets (there is no
renderer here), and the same meshes (bench_batch.py's recipes).  Steps are timed with CUDA events after warm-up.  A second,
separate run puts events around each part of the step (forward solve / forward normals and loss / backward / optimiser) to
split the time, and a third times the optimiser step alone.  Prints the card name and power limit; writes nothing to disk.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "large-steps-pytorch_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

from bench_batch import card, workload
from largesteps_b200 import meshops, _native as N
from largesteps_b200.batch import from_differential_batch, pack_meshes
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.optimize import AdamUniform
from largesteps_b200.parameterize import from_differential, to_differential

DEV = "cuda:0"


class PerParameterAdamUniform(torch.optim.Optimizer):
    """AdamUniform as one ls_adam_uniform_step call per parameter: the optimiser step of the per-mesh loop."""

    def __init__(self, params, lr=0.1, betas=(0.9, 0.999)):
        super().__init__(params, dict(lr=lr, betas=betas))

    @torch.no_grad()
    def step(self):
        lib = N.lib()
        for group in self.param_groups:
            lr, (b1, b2) = group["lr"], group["betas"]
            for p in group["params"]:
                state = self.state[p]
                if len(state) == 0:
                    state["step"] = 0
                    state["g1"] = torch.zeros_like(p.data)
                    state["g2"] = torch.zeros_like(p.data)
                    state["scratch"] = torch.zeros(4, dtype=torch.int32, device=p.device)
                state["step"] += 1
                s = state["step"]
                grad = p.grad.data.contiguous()
                with torch.cuda.device(p.device):
                    N.check(lib.ls_adam_uniform_step(
                        N.ptr(p.data), N.ptr(grad), N.ptr(state["g1"]), N.ptr(state["g2"]), p.numel(), float(lr), float(b1),
                        float(b2), float(1 - b1), float(1 - b2), float(1 - b1 ** s), float(1 - b2 ** s), N.ptr(state["scratch"]),
                        N.stream_ptr(p.device)), "ls_adam_uniform_step")


def setup(name):
    Ms, us, faces, tx, tn = [], [], [], [], []
    for v, f, kw in workload(name):
        tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
        M = compute_matrix(tv, tf, **kw)
        Ms.append(M)
        faces.append(tf)
        us.append(to_differential(M, tv))
        tx.append(1.05 * tv)
        tn.append(meshops.compute_vertex_normals(tv, tf, meshops.compute_face_normals(tv, tf)).detach())
    return Ms, us, faces, tx, tn


class Loop:
    def __init__(self, Ms, us, faces, tx, tn):
        self.Ms, self.faces, self.tx, self.tn = Ms, faces, tx, tn
        self.us = [u.clone().requires_grad_(True) for u in us]
        self.opt = PerParameterAdamUniform(self.us, lr=0.01)

    def solve(self):
        return [from_differential(M, u) for M, u in zip(self.Ms, self.us)]

    def loss(self, xs):
        out = 0
        for x, f, tx, tn in zip(xs, self.faces, self.tx, self.tn):
            n = meshops.compute_vertex_normals(x, f, meshops.compute_face_normals(x, f))
            out = out + ((n - tn) ** 2).sum() + 0.1 * ((x - tx) ** 2).sum()
        return out


class Batch:
    def __init__(self, Ms, us, faces, tx, tn):
        self.Ms = Ms
        self.us = [u.clone().requires_grad_(True) for u in us]
        self.opt = AdamUniform(self.us, lr=0.01)
        self.p = pack_meshes(tx, faces)             # the position targets, packed with the faces and offsets
        self.tx, self.tn = self.p.verts, torch.cat(tn)

    def solve(self):
        return from_differential_batch(self.Ms, self.us, packed=True)

    def loss(self, x):
        p = self.p
        n = meshops.compute_vertex_normals_batch(x, p.faces, meshops.compute_face_normals(x, p.faces), p.vert_offsets,
                                                 p.face_offsets)
        return ((n - self.tn) ** 2).sum() + 0.1 * ((x - self.tx) ** 2).sum()


def step(arm, ev=None):
    rec = (lambda i: ev[i].record()) if ev else (lambda i: None)
    rec(0)
    arm.opt.zero_grad()
    x = arm.solve()
    rec(1)
    loss = arm.loss(x)
    rec(2)
    loss.backward()
    rec(3)
    arm.opt.step()
    rec(4)


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


PARTS = ("solve_fwd", "normals_loss_fwd", "backward", "optimiser")


def run(name, reps, warmup):
    data = setup(name)
    arms = {"loop": Loop(*data), "batch": Batch(*data)}
    out = {}
    for key, arm in arms.items():
        for _ in range(warmup):
            step(arm)
        torch.cuda.synchronize()
        ms = timed(lambda: step(arm), reps)
        # the split, in a run of its own: events between the parts of each step, summed over the steps
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        split = dict.fromkeys(PARTS, 0.0)
        for _ in range(reps):
            step(arm, ev)
            ev[4].synchronize()
            for i, k in enumerate(PARTS):
                split[k] += ev[i].elapsed_time(ev[i + 1]) / reps
        opt_ms = timed(arm.opt.step, reps)          # the optimiser step alone, back to back
        out[key] = dict(ms_per_step=ms, steps_per_s=1000.0 / ms, split_ms=split, optimiser_alone_ms=opt_ms)
    # both arms ran the same steps from the same start: their parameters agree to solver precision
    err = max(float(np.linalg.norm((a.detach() - b.detach()).double().cpu().numpy()) /
                    max(np.linalg.norm(b.detach().double().cpu().numpy()), 1e-300))
              for a, b in zip(arms["batch"].us, arms["loop"].us))
    V = [u.shape[0] for u in data[1]]
    return dict(workload=name, meshes=len(V), V_min=min(V), V_max=max(V), **out,
                speedup=out["loop"]["ms_per_step"] / out["batch"]["ms_per_step"], worst_rel_l2_between_arms=err)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", action="store_true")
    ap.add_argument("--workloads", default="ico4_x1,ico4_x4,ico4_x16,ico4_x64,bunny_x16",
                    help="comma-separated <base>_x<meshes> as in bench_batch.py")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch_loop.py needs a GPU")
    print(f"card: {card()}", flush=True)
    for w in a.workloads.split(","):
        r = run(w, a.reps, a.warmup)
        if a.json:
            print(json.dumps(r), flush=True)
            continue
        print(f"{r['workload']:>10}: {r['meshes']:3d} meshes, V {r['V_min']}..{r['V_max']}:  "
              f"loop {r['loop']['steps_per_s']:8.1f} steps/s ({r['loop']['ms_per_step']:.3f} ms)   "
              f"batch {r['batch']['steps_per_s']:8.1f} steps/s ({r['batch']['ms_per_step']:.3f} ms)   "
              f"batch/loop {r['speedup']:.2f}x   arms agree to {r['worst_rel_l2_between_arms']:.1e}", flush=True)
        for arm in ("loop", "batch"):
            s = r[arm]["split_ms"]
            print(f"{'':>12}{arm:>5} split (ms): " + "  ".join(f"{k} {s[k]:.3f}" for k in PARTS) +
                  f"   optimiser alone {r[arm]['optimiser_alone_ms']:.3f} ms "
                  f"({1000 * r[arm]['optimiser_alone_ms'] / r['meshes']:.1f} us per parameter)", flush=True)


if __name__ == "__main__":
    main()
