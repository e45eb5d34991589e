"""GPU: largesteps_b200.remesh.remesh_botsch -- each stage against the numpy model of tests/remesh_model.py fed the device's own
input, the whole call's invariants, reproducibility and projection, a 655K-vertex icosphere, the re-parameterisation of a
remeshed bunny, and the rejected inputs."""
import numpy as np
import pytest
import torch

import oracle
import remesh_model as RM
from largesteps_b200 import workloads
from largesteps_b200.distance import MeshDistance
from largesteps_b200.parameterize import from_differential
from largesteps_b200.remesh import Reparameterizer, _Remesher, remesh_botsch
from gpu_util import DEV, rel_l2
from test_remesh_model import assert_normals_kept, ico, noisy, octahedron, with_small_components

pytestmark = pytest.mark.gpu


def mesh(case, bunny_mesh):
    if case == "octahedron":
        return octahedron()
    if case.startswith("ico_"):
        return ico(1.6 if case == "ico_out" else 0.4)
    if case == "components":
        v, f = workloads.icosphere(2)
        return with_small_components(np.asarray(v, np.float32), np.asarray(f, np.int64))[:2]
    if case == "bunny":
        v, f = bunny_mesh
    else:
        v, f = workloads.icosphere(int(case[-1]))
    v, f, _ = noisy(np.asarray(v, np.float32), np.asarray(f, np.int64), 0.1, seed=len(case))
    return v, f


def mean_edge(v, f):
    return float(np.linalg.norm(v[f[:, 1]] - v[f[:, 0]], axis=1).mean())


def host(r):
    v, f = r.mesh()
    return v.cpu().numpy(), f.cpu().numpy().astype(np.int64)


def assert_ulp(got, want, ulps):
    """Every coordinate within `ulps` float32 ulp of the row's largest coordinate: a coordinate that should be 0 may come out
    as +-1e-16 from the closest-point arithmetic on either side."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    gap = np.abs(got.astype(np.float64) - want.astype(np.float64))
    scale = np.maximum(np.abs(got), np.abs(want)).max(1, keepdims=True)
    assert (gap <= ulps * np.spacing(scale)).all(), float(gap.max())


@pytest.mark.parametrize("scale", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("case", ["octahedron", "ico_out", "ico_in", "components", "ico3", "ico4", "bunny"])
def test_stages_match_the_model(case, scale, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    h = scale * mean_edge(v, f)
    high, low = 1.4 * h, 0.7 * h
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    r = _Remesher(tv, tf)
    r.check()
    r.compact()
    target = MeshDistance(*r.mesh())
    V0, F0 = host(r)
    iters = 2 if len(v) < 1000 else 1
    for _ in range(iters):
        hv, hf = host(r)
        n = r.split(high)
        mv, mf, mn = RM.split(hv, hf, high)
        gv, gf = host(r)
        assert n == mn and np.array_equal(gf, mf) and np.array_equal(gv, mv)
        live = r.V
        while True:
            hv, hf = host(r)
            n = r.collapse_round(low, high, live)
            mv, mf, mn = RM.collapse_round(hv, hf, low, high, live)
            gv, gf = host(r)
            assert n == mn and np.array_equal(gf, mf) and np.array_equal(gv, mv)
            assert_normals_kept(hv, hf, gv, gf)
            live -= n
            if n == 0:
                break
        hv, hf = host(r)
        r.compact()
        mv, mf = RM.compact(hv, hf)
        gv, gf = host(r)
        assert np.array_equal(gf, mf) and np.array_equal(gv, mv)
        while True:
            hv, hf = host(r)
            n = r.flip_round()
            mf, mn = RM.flip_round(hv, hf)
            assert n == mn and np.array_equal(host(r)[1], mf)
            assert_normals_kept(hv, hf, hv, mf)
            if n == 0:
                break
        hv, hf = host(r)
        r.relax(target)
        assert_ulp(host(r)[0], RM.relax(hv, hf, V0, F0), 2)
    RM.assert_invariants(*host(r), RM.euler(v, f))


def edge_share(v, f, h):
    e = np.linalg.norm(v[f] - v[f[:, [1, 2, 0]]], axis=2)
    return float(((e >= 0.7 * h) & (e <= 1.4 * h)).mean())


@pytest.mark.parametrize("project", [True, False])
@pytest.mark.parametrize("case", ["ico3", "components", "bunny"])
def test_end_to_end(case, project, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    h = mean_edge(v, f)
    tv = torch.from_numpy(v).to(DEV)
    outs = [remesh_botsch(tv, torch.from_numpy(f).to(DEV).to(dt), 5, h, project) for dt in (torch.int64, torch.int32, torch.int64)]
    vo, fo = outs[0]
    assert vo.dtype == torch.float32 and fo.dtype == torch.int64 and outs[1][1].dtype == torch.int32
    for w, g in outs:                                                     # own storage, not a view of the work buffers
        assert w.untyped_storage().nbytes() == w.numel() * 4 and g.untyped_storage().nbytes() == g.numel() * g.element_size()
    for w, g in outs[1:]:
        assert torch.equal(w, vo) and torch.equal(g.long(), fo)
    hv, hf = vo.cpu().numpy(), fo.cpu().numpy()
    RM.assert_invariants(hv, hf, RM.euler(v, f))
    assert np.bincount(hf.ravel()).min() >= 3
    if project:
        sq, _, _ = MeshDistance(tv, torch.from_numpy(f).to(DEV)).squared_distance(vo)
        diag = float(np.linalg.norm(v.max(0) - v.min(0)))
        assert float(sq.max()) <= (1e-6 * diag) ** 2
    mv, mf = RM.remesh(v, f, 5, h, project)
    print(f"\n{case} project={project}: {len(hv)} vertices; edges in [0.7 h, 1.4 h]: device {edge_share(hv, hf, h):.3f}, "
          f"model {edge_share(mv, mf, h):.3f}")


def device_invariants(v, f, chi):
    V, F = v.shape[0], f.shape[0]
    f = f.long()
    a, b = f, f[:, [1, 2, 0]]
    fwd = (a * V + b).flatten()
    rev = (b * V + a).flatten()
    s = torch.sort(fwd).values
    assert bool((s[1:] != s[:-1]).all())                                  # no directed edge twice
    assert torch.equal(s, torch.sort(rev).values)                         # every edge has its twin: closed and oriented
    assert V - 3 * F // 2 + F == chi
    assert bool(torch.isfinite(v).all())
    assert bool((torch.bincount(f.flatten(), minlength=V) > 0).all())
    p = v.double()
    n = torch.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]], dim=1)
    assert bool(((n * n).sum(1) > 0).all())


def test_icosphere_level_8():
    v, f = workloads.icosphere(8)
    v, f, mean = noisy(np.asarray(v, np.float32), np.asarray(f, np.int64), 0.1)
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    vo, fo = remesh_botsch(tv, tf, 5, 0.5 * mean, True)
    print(f"\nicosphere 8: {v.shape[0]} -> {vo.shape[0]} vertices")
    assert vo.shape[0] > 2 * v.shape[0]
    device_invariants(vo, fo, 2)


def test_reparameterize_the_remeshed_bunny(bunny_mesh):
    v, f = bunny_mesh
    v = np.asarray(v, np.float32)
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    vo, fo = remesh_botsch(tv, tf, 5, mean_edge(v, f), True)
    rp = Reparameterizer(lambda_=19.0)
    M, u = rp.update(vo, fo)
    hv, hf = vo.cpu().numpy(), fo.cpu().numpy()
    r, c, val, V = oracle.compute_matrix(hv, hf, 19.0)
    ds = oracle.DirectSolver(r, c, val, V)
    assert rel_l2(from_differential(M, u).cpu().numpy(), ds.solve(u.cpu().numpy())) < 1e-5


def test_rejected_inputs():
    v, f = octahedron()
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    with pytest.raises(ValueError, match="closed"):
        remesh_botsch(tv, tf[1:], 1, 0.5)
    with pytest.raises(ValueError, match="more than two faces"):
        remesh_botsch(tv, torch.cat([tf, tf[:1].flip(1)]), 1, 0.5)
    with pytest.raises(ValueError, match="directed edge"):
        g = tf.clone()
        g[0] = g[0].flip(0)
        remesh_botsch(tv, g, 1, 0.5)
    with pytest.raises(ValueError, match="h must be"):
        remesh_botsch(tv, tf, 1, -0.5)
    with pytest.raises(TypeError):
        remesh_botsch(tv.double(), tf, 1, 0.5)
    with pytest.raises(IndexError):
        remesh_botsch(tv[:5], tf, 1, 0.5)
    vo, fo = remesh_botsch(tv, tf.int(), 0, 0.5)                          # zero iterations: the mesh as it came
    assert torch.equal(vo, tv) and torch.equal(fo, tf.int())
