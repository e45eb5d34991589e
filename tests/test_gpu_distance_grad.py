"""GPU: the gradients of point-to-mesh squared distances and the chamfer loss (largesteps_b200.distance, ls_distance_grad_f32)
against the float64 model of tests/distance_grad_model.py, fed the device's own (I, C) so that ties (the queries include the
mesh's own vertices) cannot make the comparison flaky.  Also: bitwise reproducibility, the edge cases of the contract, the
fixed-target chamfer computing only the gradients it needs, and an end-to-end fit of a sphere to the bunny."""
import math

import numpy as np
import pytest
import torch

import distance_grad_model as gm
from largesteps_b200 import workloads
from largesteps_b200.distance import MeshDistance, chamfer, hausdorff, point_mesh_squared_distance
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.meshops import average_edge_length
from largesteps_b200.optimize import AdamUniform
from largesteps_b200.parameterize import from_differential, to_differential
from largesteps_b200.remesh import Reparameterizer, remesh_botsch
import largesteps_b200._native as N
from test_gpu_distance import mesh, queries, t

pytestmark = pytest.mark.gpu


def device_grads(P, v, f, G, idx=torch.int64):
    """(sqrD, I, C, grad P, grad V) of (sqrD * G).sum() through point_mesh_squared_distance, as numpy arrays"""
    Pt = t(P).requires_grad_(True)
    Vt = t(v).requires_grad_(True)
    s, I, C = point_mesh_squared_distance(Pt, Vt, t(f, idx))
    (s * t(G)).sum().backward()
    return tuple(x.detach().cpu().numpy() for x in (s, I, C, Pt.grad, Vt.grad))


def assert_matches_model(dev, want, terms):
    """per entry within one float32 rounding of the model's float64 value plus 1e-12 x sum |terms|, and rel-L2 <= 1e-6"""
    dev = dev.astype(np.float64)
    bar = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64) + 1e-12 * terms
    err = np.abs(dev - want)
    assert (err <= bar).all(), float((err / bar).max())
    nrm = np.linalg.norm(want)
    assert np.linalg.norm(dev - want) <= 1e-6 * nrm + 1e-300, (np.linalg.norm(dev - want), nrm)


def check(P, v, f, G, out):
    _, I, C, gP, gV = out
    assert (I >= 0).all()
    wP, wV = gm.grads(P, v, f, I, C, G)
    aP, aV = gm.grad_terms_abs(P, v, f, I, C, G)
    assert_matches_model(gP, wP, aP)
    assert_matches_model(gV, wV, aV)


CASES = ["ico4", "bunny", "plane200", "degen", "shuffled"]


def case(name):
    if name == "shuffled":
        v, f = mesh("plane200")
        return v, f[np.random.default_rng(8).permutation(len(f))]
    return mesh(name)


@pytest.mark.parametrize("idx", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("name", CASES)
def test_gradients_match_the_model(name, idx):
    v, f = case(name)
    P = queries(v, f)
    G = np.random.default_rng(1).normal(size=len(P))
    check(P, v, f, G, device_grads(P, v, f, G, idx))


def test_chamfer_on_the_million_vertex_pair():
    (va, fa), (vb, fb) = workloads.plane(1000), workloads.plane(1000, seed=1)
    VA, VB = t(va).requires_grad_(True), t(vb).requires_grad_(True)
    FA, FB = t(fa), t(fb)
    loss = chamfer(VA, FA, VB, FB)
    loss.backward()
    sa, ia, ca = (x.cpu().numpy() for x in MeshDistance(VB.detach(), FB).squared_distance(VA.detach()))
    sb, ib, cb = (x.cpu().numpy() for x in MeshDistance(VA.detach(), FA).squared_distance(VB.detach()))
    assert loss.dtype == torch.float64 and loss.dim() == 0
    assert abs(loss.item() - (sa.mean() + sb.mean())) <= 1e-12 * loss.item()
    ga, gb = np.full(len(va), 1.0 / len(va)), np.full(len(vb), 1.0 / len(vb))
    pA, vB = gm.grads(va, vb, fb, ia, ca, ga)           # A's vertices as points on B, B's as corners
    pB, vA = gm.grads(vb, va, fa, ib, cb, gb)
    tpA, tvB = gm.grad_terms_abs(va, vb, fb, ia, ca, ga)
    tpB, tvA = gm.grad_terms_abs(vb, va, fa, ib, cb, gb)
    # autograd adds the two float32 terms: one more float32 rounding
    for dev, (p, c), (tp, tc) in ((VA.grad, (pA, vA), (tpA, tvA)), (VB.grad, (pB, vB), (tpB, tvB))):
        dev = dev.cpu().numpy().astype(np.float64)
        want = p + c
        bar = (np.spacing(np.abs(p).astype(np.float32)) + np.spacing(np.abs(c).astype(np.float32))
               + np.spacing(np.abs(want).astype(np.float32))).astype(np.float64) + 1e-12 * (tp + tc)
        assert (np.abs(dev - want) <= bar).all(), float((np.abs(dev - want) / bar).max())
        assert np.linalg.norm(dev - want) <= 1e-6 * np.linalg.norm(want)


def test_bitwise_reproducible_across_runs_index_types_streams_and_builds():
    v, f = mesh("bunny")
    P = queries(v, f, seed=3)
    G = np.random.default_rng(2).normal(size=len(P))
    ref = device_grads(P, v, f, G, torch.int64)
    outs = [device_grads(P, v, f, G, torch.int64), device_grads(P, v, f, G, torch.int32)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        outs.append(device_grads(P, v, f, G, torch.int64))
    s.synchronize()
    for out in outs:
        for x, y in zip(ref, out):
            np.testing.assert_array_equal(x.view(np.uint8), y.view(np.uint8))
    # the fixed-target loss, twice with a rebuilt BVH
    grads = []
    for _ in range(2):
        VA = t(workloads.icosphere(3)[0] * np.float32(0.1)).requires_grad_(True)
        MeshDistance(t(v), t(f)).chamfer(VA, t(workloads.icosphere(3)[1])).backward()
        grads.append(VA.grad.cpu().numpy())
    np.testing.assert_array_equal(grads[0].view(np.uint8), grads[1].view(np.uint8))


def test_edge_cases():
    v, f = mesh("ico4")
    # n = 0: both gradients are zero
    P0 = t(np.zeros((0, 3), np.float32)).requires_grad_(True)
    V0 = t(v).requires_grad_(True)
    s, _, _ = point_mesh_squared_distance(P0, V0, t(f))
    s.sum().backward()
    assert P0.grad.shape == (0, 3) and (V0.grad == 0).all()
    # an unreferenced vertex gets exactly zero; a face that repeats a vertex adds once per corner
    vx = np.concatenate([v, [[5.0, 5.0, 5.0]]]).astype(np.float32)
    fx = np.concatenate([f, [[0, 0, 1]]])
    P = np.concatenate([queries(v, f, seed=4), vx[:2] + np.float32(0.3)]).astype(np.float32)
    G = np.random.default_rng(5).normal(size=len(P))
    out = device_grads(P, vx, fx, G)
    assert out[4][-1].tolist() == [0.0, 0.0, 0.0]
    check(P, vx, fx, G, out)
    # the NaN rule: a NaN point gets NaN in its row of grad P and adds nothing to grad V
    Pn = P.copy()
    Pn[7, 1] = np.nan
    s, I, C, gP, gV = device_grads(Pn, vx, fx, G)
    assert I[7] == -1 and np.isnan(s[7]) and np.isnan(gP[7]).all()
    ok = np.arange(len(P)) != 7
    assert np.isfinite(gP[ok]).all() and np.isfinite(gV).all()
    wP, wV = gm.grads(Pn, vx, fx, I, C, G)
    aP, aV = gm.grad_terms_abs(Pn, vx, fx, I, C, G)
    assert_matches_model(gP[ok], wP[ok], aP[ok])
    assert_matches_model(gV, wV, aV)
    # a non-finite corner: every row is answered with -1, so grad P is NaN and grad V zero
    vn = vx.copy()
    vn[3, 2] = np.nan
    s, I, _, gP, gV = device_grads(P[:10], vn, fx, G[:10])
    assert (I == -1).all() and np.isnan(gP).all() and (gV == 0).all()
    # P and V the same tensor: the mesh's own vertices, both paths summed by autograd
    Vt = t(v).requires_grad_(True)
    s, I, C = point_mesh_squared_distance(Vt, Vt, t(f))
    G2 = np.random.default_rng(6).normal(size=len(v))
    (s * t(G2)).sum().backward()
    wP, wV = gm.grads(v, v, f, I.cpu().numpy(), C.cpu().numpy(), G2)
    np.testing.assert_allclose(Vt.grad.cpu().numpy(), wP + wV, rtol=0, atol=1e-12)
    # an in-place change between forward and backward raises instead of giving a wrong gradient
    for which in (0, 1):
        Pt, Vt = t(P).requires_grad_(True), t(vx).requires_grad_(True)
        s = point_mesh_squared_distance(Pt, Vt, t(fx))[0]
        with torch.no_grad():
            (Pt, Vt)[which].add_(1.0)
        with pytest.raises(RuntimeError, match="inplace"):
            s.sum().backward()
    # outside autograd nothing changes: no graph, the same values
    s1 = point_mesh_squared_distance(t(P), t(vx), t(fx))
    s2 = point_mesh_squared_distance(t(P).requires_grad_(True), t(vx), t(fx))
    assert s1[0].grad_fn is None and s2[0].grad_fn is not None and s2[1].grad_fn is None and s2[2].grad_fn is None
    for x, y in zip(s1, s2):
        assert torch.equal(x, y.detach())


def test_fixed_target_computes_only_the_gradients_it_needs(monkeypatch):
    (va, fa), (vb, fb) = workloads.icosphere(3), workloads.icosphere(4)
    va = (va * np.float32(1.05)).astype(np.float32)
    VB = t(vb).requires_grad_(True)
    target = MeshDistance(VB, t(fb))
    lib = N.lib()
    real = lib.ls_distance_grad_f32
    calls = []

    def spy(*args):
        calls.append((args[10].value is not None, args[11].value is not None))     # grad_points, grad_verts
        return real(*args)

    monkeypatch.setattr(lib, "ls_distance_grad_f32", spy)
    VA = t(va).requires_grad_(True)
    loss = target.chamfer(VA, t(fa))
    loss.backward()
    target.check()
    # first term: A's vertices as points against B (grad P only); second: B's vertices against A (grad V only)
    assert sorted(calls) == [(False, True), (True, False)], calls
    assert VB.grad is None
    s_a, i_a, c_a = (x.cpu().numpy() for x in target.squared_distance(t(va)))
    s_b, i_b, c_b = (x.cpu().numpy() for x in MeshDistance(t(va), t(fa)).squared_distance(t(vb)))
    assert loss.item() == pytest.approx(s_a.mean() + s_b.mean(), rel=1e-12)
    ga, gb = np.full(len(va), 1.0 / len(va)), np.full(len(vb), 1.0 / len(vb))
    want = gm.grads(va, vb, fb, i_a, c_a, ga)[0] + gm.grads(vb, va, fa, i_b, c_b, gb)[1]
    dev = VA.grad.cpu().numpy().astype(np.float64)
    assert np.linalg.norm(dev - want) <= 1e-6 * np.linalg.norm(want)
    # chamfer(VA, FA, VB, FB) gives the same value and the same gradient w.r.t. VA
    VA2 = t(va).requires_grad_(True)
    loss2 = chamfer(VA2, t(fa), t(vb), t(fb))
    loss2.backward()
    assert loss2.item() == loss.item()
    assert torch.equal(VA2.grad, VA.grad)
    # a face index out of range: no read-back in the call, a NaN loss and an IndexError from check()
    fbad = t(fa).clone()
    fbad[3, 1] = len(va) + 7
    assert math.isnan(target.chamfer(t(va), fbad).item())
    with pytest.raises(IndexError):
        target.check()


def _fit(bunny_mesh, steps, remesh_at=200, record=None):
    vb, fb = bunny_mesh
    vb = vb.astype(np.float32)
    target = MeshDistance(t(vb), t(fb))
    v0, f0 = workloads.icosphere(4)
    center = (vb.max(0) + vb.min(0)) / 2
    radius = np.linalg.norm(vb - center, axis=1).max()
    v, f = t((center + radius * v0).astype(np.float32)), t(f0)
    lam, lr = 19.0, 1e-2
    M = compute_matrix(v, f, lam)
    u = to_differential(M, v).clone().requires_grad_(True)
    opt = AdamUniform([u], lr=lr)
    rp = None
    for it in range(steps + 1):
        if it == remesh_at:
            with torch.no_grad():
                v = from_differential(M, u, "Cholesky")
                h = float(average_edge_length(v, f)) * 0.5
                v, f = remesh_botsch(v, f, 5, h, True)
                rp = Reparameterizer(lambda_=lam)
                M, u = rp.update(v, f)
            u = u.clone().requires_grad_(True)
            lr *= 0.8
            opt = AdamUniform([u], lr=lr)
        v = from_differential(M, u, "Cholesky")
        loss = target.chamfer(v, f)
        if record is not None and it % 100 == 0:
            record.append((it, loss.item(), hausdorff(v.detach(), f, t(vb), t(fb)), int(v.shape[0])))
        if it == steps:
            break
        opt.zero_grad()
        loss.backward()
        opt.step()
    target.check()
    return v.detach(), f


# final chamfer of the 400-step fit measured on an H100 80GB HBM3 at 700 W (DESIGN 4.5), times a margin of 1.5
FIT_CHAMFER_BOUND = 1.5 * 1.05e-3


def test_fit_a_sphere_to_the_bunny(bunny_mesh):
    traj = []
    _fit(bunny_mesh, 400, record=traj)
    for it, c, h, n in traj:
        print(f"step {it}: chamfer {c:.4e}  hausdorff {h:.4e}  vertices {n}")
    assert traj[-1][2] < 0.5 * traj[0][2]
    assert traj[-1][1] < FIT_CHAMFER_BOUND
    # the solve, AdamUniform and the backward are deterministic: the first 50 steps twice give the same vertices
    a, _ = _fit(bunny_mesh, 50)
    b, _ = _fit(bunny_mesh, 50)
    assert torch.equal(a, b)
