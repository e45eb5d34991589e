#!/usr/bin/env python
"""Generate tests/golden/cot_grad.npz: values and vertex gradients of the reference's cotangent matrices
(largesteps/geometry.py:3-63 laplacian_cot, 96-133 compute_matrix) and of the products the reference loop takes with them
(parameterize.py:30 to_differential, scripts/main.py:192-195 regulariser), run on the CPU.

Run where a checkout of the reference is available (make_golden.REF):   python tests/golden/make_golden_cot.py

The reference's modules are loaded by make_golden.load_reference, and its geometry.py is then exec'd again from its source
text with two in-memory rewrites (nothing is copied into this repository):
  * "device='cuda'" -> "device='cpu'", as make_golden.py does;
  * "L += L.t()" (geometry.py:56) -> "L = L + L.t()".  The in-place sparse add gives the same forward values, but autograd
    rejects it ("modified by an inplace operation"), so the reference's matrices cannot be differentiated without it.

Gradients w.r.t. verts are taken in float64 (a tight reference) and in float32 (to measure the reference's own error).
Stored, to keep the fixture small:
  {mesh}.verts, .faces     the mesh (not for the bunny: it is tests/golden/bunny_mesh.npz, faces as int64)
  {mesh}.idx               int32 (2, nnz): the coalesced pattern of the cotangent compute_matrix (the same for both cases)
  {mesh}.l19.W, .a095.W    int8 (nnz): seeded integer weights in [-4, 4];   {mesh}.G  int8 (V, 3): the same for td
  {mesh}.{loss}.grad       the float64 gradient, rounded to float32 (a relative change of at most 2^-24 per entry)
  {mesh}.{loss}.f32_err    float64 scalar: rel-L2 of the reference's float32 gradient against its float64 one
The forward values are not stored again: assembly.npz holds the reference's cotangent matrices.  Losses:
  l19     (compute_matrix(v, f, 19, cotan=True).values() * W19).sum()
  a095    (compute_matrix(v, f, 1, alpha=0.95, cotan=True).values() * W095).sum()
  td      (to_differential(compute_matrix(v, f, 19, cotan=True), v) * G).sum()     -- v reaches the loss through M and directly
  reg_bi  (laplacian_cot(v, f) @ v).square().mean()
  reg_lap (v * (laplacian_cot(v, f) @ v)).mean()
Meshes: the five of make_golden_mass.py; the degenerate one also gets a duplicated face (a repeated-vertex face, [0, 0, 2], is
already part of it).
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, load_reference, workloads  # noqa: E402
from make_golden_mass import degenerate, grid  # noqa: E402

warnings.filterwarnings("ignore")
torch.set_num_threads(4)


def reference():
    mods = load_reference()
    geo = mods["geometry"]
    path = os.path.join(REF, "largesteps", "geometry.py")
    src = open(path).read().replace("device='cuda'", "device='cpu'")
    assert src.count("L += L.t()") == 1
    src = src.replace("L += L.t()", "L = L + L.t()")
    exec(compile(src, path, "exec"), geo.__dict__)
    return geo, mods["parameterize"]


def meshes():
    d = np.load(os.path.join(HERE, "bunny_mesh.npz"))
    dv, df = degenerate()
    return {"ico2": workloads.icosphere(2), "bunny": (d["verts"], d["faces"].astype(np.int64)), "grid": grid(),
            "plane": workloads.plane(16, seed=5), "degen": (dv, np.concatenate([df, df[:1]]))}


def main():
    geo, par = reference()
    out = {}
    for name, (v, f) in meshes().items():
        v = np.ascontiguousarray(v, dtype=np.float32)
        f = np.ascontiguousarray(f, dtype=np.int64)
        tf = torch.from_numpy(f)
        if name != "bunny":
            out[f"{name}.verts"], out[f"{name}.faces"] = v, f
        rng = np.random.default_rng(11)
        for case, kw in (("l19", dict(lambda_=19.0)), ("a095", dict(lambda_=1.0, alpha=0.95))):
            M = geo.compute_matrix(torch.from_numpy(v), tf, cotan=True, **kw)
            idx = M.indices().numpy().astype(np.int32)           # the same pattern for both cases: stored once
            assert np.array_equal(out.setdefault(f"{name}.idx", idx), idx)
            out[f"{name}.{case}.W"] = rng.integers(-4, 5, size=M._nnz()).astype(np.int8)
        out[f"{name}.G"] = rng.integers(-4, 5, size=v.shape).astype(np.int8)
        W = {c: torch.from_numpy(out[f"{name}.{c}.W"].astype(np.float64)) for c in ("l19", "a095")}
        G = torch.from_numpy(out[f"{name}.G"].astype(np.float64))
        grads = {}
        for dt in (torch.float32, torch.float64):
            losses = {
                "l19": lambda x: (geo.compute_matrix(x, tf, 19.0, cotan=True).values() * W["l19"].to(dt)).sum(),
                "a095": lambda x: (geo.compute_matrix(x, tf, 1.0, alpha=0.95, cotan=True).values() * W["a095"].to(dt)).sum(),
                "td": lambda x: (par.to_differential(geo.compute_matrix(x, tf, 19.0, cotan=True), x) * G.to(dt)).sum(),
                "reg_bi": lambda x: (geo.laplacian_cot(x, tf) @ x).square().mean(),
                "reg_lap": lambda x: (x * (geo.laplacian_cot(x, tf) @ x)).mean(),
            }
            for loss, fn in losses.items():
                x = torch.from_numpy(v).to(dt).requires_grad_(True)
                fn(x).backward()
                grads[loss, dt] = x.grad.numpy().astype(np.float64)
        for loss in ("l19", "a095", "td", "reg_bi", "reg_lap"):
            g32, g64 = grads[loss, torch.float32], grads[loss, torch.float64]
            assert np.isfinite(g64).all() and np.isfinite(g32).all()
            out[f"{name}.{loss}.grad"] = g64.astype(np.float32)
            out[f"{name}.{loss}.f32_err"] = np.float64(np.linalg.norm(g32 - g64) / np.linalg.norm(g64))
    path = os.path.join(HERE, "cot_grad.npz")
    np.savez_compressed(path, **out)
    print("cot_grad.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
