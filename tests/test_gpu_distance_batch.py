"""GPU: point-to-mesh distances, Hausdorff and chamfer over packed batches (largesteps_b200.distance.MeshDistanceBatch and the
_batch functions, csrc/ls_distance.cu's forest build and batched query) against the single-mesh calls, mesh by mesh: sqrD, I
(less the face offset), C and Hausdorff bitwise, the chamfer values within the bound of summing in another order, and the
chamfer gradients bitwise.  Also: isolation of a bad mesh or row, launch counts that do not grow with B, reproducibility
across runs and streams, and a batched fit of eight spheres to eight targets."""
import math

import numpy as np
import pytest
import torch

from largesteps_b200 import workloads
from largesteps_b200.batch import from_differential_batch, pack_meshes
from largesteps_b200.distance import (MeshDistance, MeshDistanceBatch, chamfer, chamfer_batch, hausdorff, hausdorff_batch,
                                      point_mesh_squared_distance_batch)
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.optimize import AdamUniform
from largesteps_b200.parameterize import to_differential
import largesteps_b200._native as N
from test_gpu_distance import degenerate_mesh, noisy, queries, t

pytestmark = pytest.mark.gpu


def mixed_meshes(bunny_mesh):
    """icosphere(3), the bunny, a noisy plane(64), one face, and a mesh with degenerate and duplicated faces"""
    vb, fb = bunny_mesh
    vp, fp = workloads.plane(64)
    one_v = np.array([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.2, 0.7, 0.1]], np.float32)
    return [workloads.icosphere(3), (vb.astype(np.float32), fb), (noisy(vp, 1e-3, 3), fp),
            (one_v, np.array([[0, 1, 2]], np.int64)), degenerate_mesh()]


def mesh_queries(v, f, seed):
    """queries() (own vertices, near, far and box points) plus points on edges"""
    e = f[:, [0, 1]]
    w = np.random.default_rng(seed).uniform(size=(len(e), 1))
    on_edge = (v[e[:, 0]] * (1 - w) + v[e[:, 1]] * w).astype(np.float32)
    return np.concatenate([queries(v, f, seed, m=120), on_edge[:200], v[e[:50, 0]] * 0.5 + v[e[:50, 1]] * 0.5])


def packed(ms, idx):
    return pack_meshes([t(v) for v, _ in ms], [t(f, idx) for _, f in ms])


@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
def test_squared_distance_is_bitwise_per_mesh(bunny_mesh, idx):
    ms = mixed_meshes(bunny_mesh)
    p = packed(ms, idx)
    Ps = [mesh_queries(v, f, b) for b, (v, f) in enumerate(ms)]
    po = np.concatenate([[0], np.cumsum([len(P) for P in Ps])]).tolist()
    md = MeshDistanceBatch(*p[:4])
    s, I, C = md.squared_distance(t(np.concatenate(Ps)), po)
    md.check()
    s2, I2, C2 = point_mesh_squared_distance_batch(t(np.concatenate(Ps)), torch.tensor(po, device="cuda"), *p[:4])
    assert torch.equal(s, s2) and torch.equal(I, I2) and torch.equal(C, C2)
    for b, ((v, f), P) in enumerate(zip(ms, Ps)):
        rs, ri, rc = MeshDistance(t(v), t(f, idx)).squared_distance(t(P))
        a, e = po[b], po[b + 1]
        assert torch.equal(s[a:e], rs), b
        assert torch.equal(I[a:e] - p.face_offsets_host[b], ri), b
        assert torch.equal(C[a:e], rc), b


def test_hausdorff_is_bitwise_per_mesh(bunny_mesh):
    ms = mixed_meshes(bunny_mesh)
    mA = [(noisy(v, 2e-3, 10 + b), f) for b, (v, f) in enumerate(ms)]
    pA, pB = packed(mA, torch.int64), packed(ms, torch.int32)
    out = hausdorff_batch(*pA[:4], *pB[:4])
    assert out.dtype == torch.float64 and out.shape == (len(ms),)
    want = [hausdorff(t(va), t(fa), t(vb), t(fb)) for (va, fa), (vb, fb) in zip(mA, ms)]
    assert out.tolist() == want
    assert MeshDistanceBatch(*pB[:4]).hausdorff(*pA[:4]).tolist() == want


def test_hausdorff_broadcast_scores_a_trajectory(bunny_mesh):
    vb, fb = bunny_mesh
    vb = vb.astype(np.float32)
    its = [noisy(vb, 1e-3 * (1 + k % 5), 100 + k) for k in range(50)]
    p = pack_meshes([t(v) for v in its], [t(fb)] * 50)
    got = hausdorff_batch(*p[:4], t(vb), t(fb), [0, len(vb)], [0, len(fb)])
    want = [hausdorff(t(v), t(fb), t(vb), t(fb)) for v in its]
    assert got.tolist() == want
    # the other way round: one mesh against 50
    assert hausdorff_batch(t(vb), t(fb), [0, len(vb)], [0, len(fb)], *p[:4]).tolist() == \
        [hausdorff(t(vb), t(fb), t(v), t(fb)) for v in its]


def _chamfer_pairs(bunny_mesh):
    ms = mixed_meshes(bunny_mesh)
    return [(noisy(v, 3e-3, 20 + b), f) for b, (v, f) in enumerate(ms)], ms


@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
def test_chamfer_values_and_gradients_per_mesh(bunny_mesh, idx):
    mA, mB = _chamfer_pairs(bunny_mesh)
    pA, pB = packed(mA, idx), packed(mB, idx)
    VA = pA.verts.clone().requires_grad_(True)
    VB = pB.verts.clone().requires_grad_(True)
    out = chamfer_batch(VA, *pA[1:4], VB, *pB[1:4])
    out.sum().backward()
    for b, ((va, fa), (vb, fb)) in enumerate(zip(mA, mB)):
        a1 = t(va).requires_grad_(True)
        b1 = t(vb).requires_grad_(True)
        ref = chamfer(a1, t(fa, idx), b1, t(fb, idx))
        ref.backward()
        n = len(va) + len(vb)
        assert abs(out[b].item() - ref.item()) <= 2 * n * 2.0 ** -53 * ref.item(), b
        voA, voB = pA.vert_offsets_host, pB.vert_offsets_host
        assert torch.equal(VA.grad[voA[b]:voA[b + 1]], a1.grad), b
        assert torch.equal(VB.grad[voB[b]:voB[b + 1]], b1.grad), b


def test_weighted_chamfer_gradients_per_mesh(bunny_mesh):
    """Any upstream weights, not only .sum(): each mesh's gradients are bitwise those of its own weighted chamfer."""
    mA, mB = _chamfer_pairs(bunny_mesh)
    pA, pB = packed(mA, torch.int64), packed(mB, torch.int64)
    w = torch.from_numpy(np.random.default_rng(5).uniform(0.1, 3.0, len(mA))).cuda()
    VA = pA.verts.clone().requires_grad_(True)
    VB = pB.verts.clone().requires_grad_(True)
    (chamfer_batch(VA, *pA[1:4], VB, *pB[1:4]) * w).sum().backward()
    for b, ((va, fa), (vb, fb)) in enumerate(zip(mA, mB)):
        a1 = t(va).requires_grad_(True)
        b1 = t(vb).requires_grad_(True)
        (chamfer(a1, t(fa), b1, t(fb)) * w[b]).backward()
        voA, voB = pA.vert_offsets_host, pB.vert_offsets_host
        assert torch.equal(VA.grad[voA[b]:voA[b + 1]], a1.grad), b
        assert torch.equal(VB.grad[voB[b]:voB[b + 1]], b1.grad), b


def test_fixed_target_chamfer_sends_gradient_to_va_only(bunny_mesh):
    mA, mB = _chamfer_pairs(bunny_mesh)
    pA, pB = packed(mA, torch.int64), packed(mB, torch.int64)
    VA = pA.verts.clone().requires_grad_(True)
    VB = pB.verts.clone().requires_grad_(True)
    target = MeshDistanceBatch(VB, *pB[1:4])
    out = target.chamfer(VA, *pA[1:4])
    out.sum().backward()
    target.check()
    assert VB.grad is None
    for b, ((va, fa), (vb, fb)) in enumerate(zip(mA, mB)):
        a1 = t(va).requires_grad_(True)
        ref = MeshDistance(t(vb), t(fb)).chamfer(a1, t(fa))
        ref.backward()
        assert abs(out[b].item() - ref.item()) <= 2 * (len(va) + len(vb)) * 2.0 ** -53 * ref.item(), b
        assert torch.equal(VA.grad[pA.vert_offsets_host[b]:pA.vert_offsets_host[b + 1]], a1.grad), b


def test_isolation(bunny_mesh):
    mA, mB = _chamfer_pairs(bunny_mesh)
    pA, pB = packed(mA, torch.int64), packed(mB, torch.int64)
    Ps = [mesh_queries(v, f, b) for b, (v, f) in enumerate(mB)]
    po = np.concatenate([[0], np.cumsum([len(P) for P in Ps])]).tolist()
    P = t(np.concatenate(Ps))
    s0, I0, C0 = MeshDistanceBatch(*pB[:4]).squared_distance(P, po)
    # a NaN corner in mesh 1: mesh 1's rows are NaN and -1, the others unchanged
    Vn = pB.verts.clone()
    Vn[pB.vert_offsets_host[1] + 5, 2] = math.nan
    s, I, C = MeshDistanceBatch(Vn, *pB[1:4]).squared_distance(P, po)
    r1 = slice(po[1], po[2])
    assert torch.isnan(s[r1]).all() and (I[r1] == -1).all() and torch.isnan(C[r1]).all()
    keep = torch.ones(len(P), dtype=torch.bool, device="cuda")
    keep[r1] = False
    assert torch.equal(s[keep], s0[keep]) and torch.equal(I[keep], I0[keep]) and torch.equal(C[keep], C0[keep])
    # a NaN query row: only that row
    Pn = P.clone()
    Pn[po[2] + 3, 0] = math.nan
    s, I, C = MeshDistanceBatch(*pB[:4]).squared_distance(Pn, po)
    row = po[2] + 3
    assert math.isnan(s[row].item()) and I[row].item() == -1
    keep = torch.ones(len(P), dtype=torch.bool, device="cuda")
    keep[row] = False
    assert torch.equal(s[keep], s0[keep]) and torch.equal(I[keep], I0[keep])
    # a face of mesh 2 indexing mesh 0's vertices
    Fbad = pA.faces.clone()
    Fbad[pA.face_offsets_host[2] + 1, 0] = 0
    with pytest.raises(IndexError, match="mesh 2"):
        MeshDistanceBatch(pA.verts, Fbad, *pA[2:4])
    others = [b for b in range(len(mA)) if b != 2]
    good_h = hausdorff_batch(*pA[:4], *pB[:4])
    for bad in (hausdorff_batch(pA.verts, Fbad, *pA[2:4], *pB[:4]), hausdorff_batch(*pB[:4], pA.verts, Fbad, *pA[2:4])):
        assert math.isnan(bad[2].item()) and torch.equal(bad[others], good_h[others])
    target = MeshDistanceBatch(*pB[:4])
    bad = target.hausdorff(pA.verts, Fbad, *pA[2:4])
    assert math.isnan(bad[2].item()) and torch.equal(bad[others], good_h[others])
    with pytest.raises(IndexError):
        target.check()
    good = chamfer_batch(*pA[:4], *pB[:4])
    bad = chamfer_batch(pA.verts, Fbad, *pA[2:4], *pB[:4])
    assert math.isnan(bad[2].item())
    assert torch.equal(bad[others], good[others])
    bad = target.chamfer(pA.verts, Fbad, *pA[2:4])
    assert math.isnan(bad[2].item()) and not torch.isnan(bad[others]).any()
    with pytest.raises(IndexError):
        target.check()
    # the last mesh with faces but no vertices (its vertex range is empty at the end of the batch): NaN in its entry, and
    # nothing reads past the vertices
    vo = pA.vert_offsets_host
    vo_empty = vo[:-2] + (vo[-1], vo[-1])
    last, keep = len(mA) - 1, list(range(len(mA) - 2))
    with pytest.raises(IndexError, match=f"mesh {last}"):
        MeshDistanceBatch(pA.verts, pA.faces, vo_empty, pA.face_offsets_host)
    for bad, ok in ((chamfer_batch(pA.verts, pA.faces, vo_empty, pA.face_offsets_host, *pB[:4]), good),
                    (target.chamfer(pA.verts, pA.faces, vo_empty, pA.face_offsets_host), good),
                    (hausdorff_batch(pA.verts, pA.faces, vo_empty, pA.face_offsets_host, *pB[:4]), good_h)):
        torch.cuda.synchronize()
        assert math.isnan(bad[last].item()) and not math.isnan(bad[last - 1].item())
        assert torch.equal(bad[keep], ok[keep])
    with pytest.raises(IndexError):
        target.check()
    # a mesh without faces
    with pytest.raises(ValueError, match="mesh 1"):
        fo = pA.face_offsets_host
        MeshDistanceBatch(pA.verts, pA.faces, pA.vert_offsets_host, fo[:2] + fo[1:2] + fo[3:])


def _spheres(level, seed):
    v, f = workloads.icosphere(level)
    return pack_meshes([t(noisy(v * (1.0 + 0.02 * (b % 5)), 1e-3, seed + b)) for b in range(64)], [t(f)] * 64)


def test_launch_count_does_not_depend_on_b():
    """The same 64 packed icosphere(4) copies as 1, 8 or 64 meshes (every k-th offset): the totals, and with them the depth of
    the prefix scans inside the ordering and the backward's buckets, are the same, so the counts must be too."""
    pA, pB = _spheres(4, 0), _spheres(4, 100)
    counts = []
    for B in (1, 8, 64):
        k = 64 // B
        vA, fA = pA.vert_offsets_host[::k], pA.face_offsets_host[::k]
        vB, fB = pB.vert_offsets_host[::k], pB.face_offsets_host[::k]
        VA = pA.verts.clone().requires_grad_(True)
        torch.cuda.synchronize()
        n0 = N.launch_count()
        target = MeshDistanceBatch(pB.verts, pB.faces, vB, fB)
        out = target.chamfer(VA, pA.faces, vA, fA)
        out.sum().backward()
        h = target.hausdorff(pA.verts, pA.faces, vA, fA)
        torch.cuda.synchronize()
        counts.append(N.launch_count() - n0)
        assert out.shape == h.shape == (B,)
    assert counts[0] == counts[1] == counts[2], counts


def test_reproducible_across_runs_and_streams(bunny_mesh):
    mA, mB = _chamfer_pairs(bunny_mesh)
    pA, pB = packed(mA, torch.int64), packed(mB, torch.int32)

    def run():
        VA = pA.verts.clone().requires_grad_(True)
        VB = pB.verts.clone().requires_grad_(True)
        out = chamfer_batch(VA, *pA[1:4], VB, *pB[1:4])
        out.sum().backward()
        h = hausdorff_batch(*pA[:4], *pB[:4])
        s, I, C = MeshDistanceBatch(*pB[:4]).squared_distance(pA.verts, pA.vert_offsets)
        return out.detach(), VA.grad, VB.grad, h, s, I, C

    a, b = run(), run()
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        c = run()
    st.synchronize()
    for x, y, z in zip(a, b, c):
        assert torch.equal(x, y) and torch.equal(x, z)


def _rotation(seed):
    q = np.random.default_rng(seed).normal(size=4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def fit_targets(bunny_mesh):
    """eight targets: scaled, rotated and displaced copies of the bunny and of icosphere(5)"""
    vb, fb = bunny_mesh
    vb = vb.astype(np.float64)
    vb = (vb - (vb.max(0) + vb.min(0)) / 2) / np.linalg.norm(vb.max(0) - vb.min(0))
    vi, fi = workloads.icosphere(5)
    out = []
    for k in range(8):
        v, f = (vb * 2.0, fb) if k % 2 == 0 else (vi.astype(np.float64) * np.array([1.0, 0.6, 0.8]), fi.astype(np.int64))
        v = (v * (0.7 + 0.1 * k)) @ _rotation(k).T + np.array([0.3 * k, -0.2 * k, 0.1 * k])
        out.append((v.astype(np.float32), f.astype(np.int64)))
    return out


def fit(bunny_mesh, steps=300, record=None):
    targets = fit_targets(bunny_mesh)
    pT = pack_meshes([t(v) for v, _ in targets], [t(f) for _, f in targets])
    target = MeshDistanceBatch(*pT[:4])
    v0, f0 = workloads.icosphere(4)
    vs = []
    for v, _ in targets:
        c = (v.max(0) + v.min(0)) / 2
        vs.append(t((c + np.linalg.norm(v - c, axis=1).max() * v0).astype(np.float32)))
    fs = [t(f0)] * 8
    p = pack_meshes(vs, fs)
    Ms = [compute_matrix(v, f, 19.0) for v, f in zip(vs, fs)]
    us = [to_differential(M, v).clone().requires_grad_(True) for M, v in zip(Ms, vs)]
    opt = AdamUniform(us, lr=1e-2)
    for it in range(steps + 1):
        x = from_differential_batch(Ms, us, packed=True)
        loss = target.chamfer(x, *p[1:4])
        if record is not None and it % 50 == 0:
            record.append((it, loss.tolist(), hausdorff_batch(x.detach(), *p[1:4], *pT[:4]).tolist()))
        if it == steps:
            break
        opt.zero_grad()
        loss.sum().backward()
        opt.step()
    target.check()
    return x.detach()


def test_fit_eight_spheres_to_eight_targets(bunny_mesh):
    rec = []
    fit(bunny_mesh, 300, record=rec)
    for it, c, h in rec:
        print(f"step {it}: chamfer " + " ".join(f"{x:.3e}" for x in c) + " | hausdorff " + " ".join(f"{x:.3f}" for x in h))
    h0, h1 = rec[0][2], rec[-1][2]
    assert all(b < 0.5 * a for a, b in zip(h0, h1)), (h0, h1)
