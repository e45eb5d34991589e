#!/usr/bin/env python
"""Generate tests/golden/mass.npz by running the UNMODIFIED reference massmatrix_voronoi (scripts/geometry.py:35-89) on the
CPU: in float32 for the values (what the reference computes) and in float64 for the gradients of (m * W).sum() with a seeded
W (a tight reference for the gradients; the float32 gradients are stored too, to measure the reference's own error).

Run where a checkout of the reference is available (make_golden.REF):   python tests/golden/make_golden_mass.py

Meshes:
  ico2     icosphere(2)
  bunny    the bunny of bunny_mesh.npz
  grid     a flat 7 x 6 grid of 0.375 x 0.5 cells cut into 3-4-5 right triangles: every length and squared length is exact in
           float32 and float64, so cos = 0 exactly at the right angles in both runs and the non-obtuse branch applies
  plane    workloads.plane(16): z-noise gives many near-right and obtuse faces
  degen    a face with a zero-length edge (NaN at its vertices), a collinear face with non-zero edges (adds 0 to the values,
           non-finite gradients), a right triangle and an isolated vertex
"""
import importlib.util
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import REF, workloads  # noqa: E402

warnings.filterwarnings("ignore")
torch.set_num_threads(4)


def grid(nx=7, ny=6, hx=0.375, hy=0.5):
    y, x = np.meshgrid(np.arange(ny) * hy, np.arange(nx) * hx, indexing="ij")
    v = np.stack([x.ravel(), y.ravel(), 0 * x.ravel()], 1).astype(np.float32)
    f = []
    for i in range(ny - 1):
        for j in range(nx - 1):
            a, b, c, d = i * nx + j, i * nx + j + 1, (i + 1) * nx + j, (i + 1) * nx + j + 1
            # alternate the diagonal so that right angles sit at every corner position of the faces
            f += [[a, b, d], [a, d, c]] if (i + j) % 2 == 0 else [[a, b, c], [b, d, c]]
    return v, np.array(f, dtype=np.int64)


def degenerate():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0],                  # right triangle 0 1 2
                  [3, 0, 1], [4, 0, 1], [6, 0, 1],                  # collinear 3 4 5 (edges 2, 3, 1)
                  [4, 1, 1],                                        # a proper face on the collinear one's long edge
                  [9, 9, 9]], dtype=np.float32)                     # isolated
    f = np.array([[0, 1, 2], [0, 0, 2], [3, 4, 5], [4, 6, 5]], dtype=np.int64)
    return v, f


def main():
    spec = importlib.util.spec_from_file_location("ref_scripts_geometry", os.path.join(REF, "scripts", "geometry.py"))
    sg = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(sg)
    d = np.load(os.path.join(HERE, "bunny_mesh.npz"))
    meshes = {"ico2": workloads.icosphere(2), "bunny": (d["verts"], d["faces"].astype(np.int64)), "grid": grid(),
              "plane": workloads.plane(16, seed=5), "degen": degenerate()}
    out = {}
    for name, (v, f) in meshes.items():
        v = np.ascontiguousarray(v, dtype=np.float32)
        f = np.ascontiguousarray(f, dtype=np.int64)
        W = np.random.default_rng(7).normal(size=len(v)).astype(np.float32)
        out[f"{name}.verts"], out[f"{name}.faces"], out[f"{name}.W"] = v, f, W
        for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            x = torch.from_numpy(v).to(dt).requires_grad_(True)
            m = sg.massmatrix_voronoi(x, torch.from_numpy(f))
            (m * torch.from_numpy(W).to(dt)).sum().backward()
            out[f"{name}.{tag}.mass"] = m.detach().numpy()
            out[f"{name}.{tag}.grad"] = x.grad.numpy().copy()
    path = os.path.join(HERE, "mass.npz")
    np.savez_compressed(path, **out)
    print("mass.npz", os.path.getsize(path), "bytes;", {k: len(meshes[k][0]) for k in meshes}, "vertices")


if __name__ == "__main__":
    main()
