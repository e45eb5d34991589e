"""GPU: the batched solve (BatchSolver / from_differential_batch, csrc/ls_pcg_batch.cu ls_pcg_batch_*) against the fp64 direct-solve
oracle, mesh independence, per-mesh convergence, autograd, launches and rejections."""
import numpy as np
import pytest
import torch

import oracle
from largesteps_b200 import workloads, _native as N
from largesteps_b200.batch import BatchSolver, from_differential_batch
from largesteps_b200 import batch as B
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.optimize import AdamUniform
from largesteps_b200.parameterize import from_differential, to_differential
from largesteps_b200.solvers import PCGSolver
from gpu_util import DEV, to_dev, rel_l2, fan_mesh

pytestmark = pytest.mark.gpu
BAR = 1e-5


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def isolated_vertex_mesh():
    v, f = workloads.icosphere(2)
    return np.concatenate([v, [[2.0, 0.0, 0.0]]]).astype(np.float32), f


def meshes(bunny_mesh):
    """name -> (verts, faces, compute_matrix kwargs): a heterogeneous batch covering every cluster size."""
    bv, bf = bunny_mesh
    return {
        "ico2": (*workloads.icosphere(2), dict(lambda_=10.0)),
        "ico3": (*workloads.icosphere(3), dict(lambda_=10.0)),
        "ico4": (*workloads.icosphere(4), dict(lambda_=10.0)),
        "bunny_cot": (bv.astype(np.float32), bf, dict(lambda_=19.0, cotan=True)),
        "plane_a095": (*workloads.plane(60, seed=1), dict(lambda_=1.0, alpha=0.95)),
        "plane_a0999": (*workloads.plane(60, seed=2), dict(lambda_=1.0, alpha=0.999)),
        "shuffled": (*workloads.shuffle_vertices(*workloads.icosphere(4), seed=3), dict(lambda_=19.0)),
        "fan1000": (*fan_mesh(1000), dict(lambda_=3.0)),
        "isolated": (*isolated_vertex_mesh(), dict(lambda_=10.0)),
        "triangle": (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.array([[0, 1, 2]]), dict(lambda_=2.0)),
        "cs2": (*workloads.plane(80, seed=4), dict(lambda_=19.0)),
        "cs4": (*workloads.plane(120, seed=5), dict(lambda_=19.0)),
        "cs8": (*workloads.plane(160, seed=6), dict(lambda_=19.0)),
        "cs16": (*workloads.plane(220, seed=7), dict(lambda_=19.0)),
    }


@pytest.fixture(scope="module")
def batch_case(bunny_mesh):
    ms = meshes(bunny_mesh)
    names = list(ms)
    Ms, direct, verts = [], [], []
    for n in names:
        v, f, kw = ms[n]
        Ms.append(compute_matrix(*to_dev(v, f), **kw))
        r, c, val, V = oracle.compute_matrix(v, f, **kw)
        direct.append(oracle.DirectSolver(r, c, val, V))
        verts.append(v)
    return names, Ms, direct, verts


def rhs(V, k, seed):
    return np.random.default_rng(seed).normal(size=(V, k)).astype(np.float32)


def test_plan_covers_every_cluster_size(batch_case):
    names, Ms, _, _ = batch_case
    s = BatchSolver(Ms)
    plan, ng = s.plan()
    sizes = {names[i]: p[0] for i, p in enumerate(plan)}
    assert {sizes["ico2"], sizes["cs2"], sizes["cs4"], sizes["cs8"], sizes["cs16"]} == {1, 2, 4, 8, 16}, sizes
    assert plan[names.index("ico2")][1] == 3 and plan[names.index("bunny_cot")][:2] == (1, 2)


@pytest.mark.parametrize("k", [1, 2, 3])
def test_accuracy_against_the_direct_solve(batch_case, k):
    names, Ms, direct, _ = batch_case
    s = BatchSolver(Ms)
    bs = [rhs(M.shape[0], k, 10 + i) for i, M in enumerate(Ms)]
    gs = [rhs(M.shape[0], k, 100 + i) for i, M in enumerate(Ms)]
    xs = s.solve([t(b) for b in bs])
    assert all(st == 1 for st in s.status), s.status
    ys = s.solve([t(g) for g in gs], backward=True)
    for i, n in enumerate(names):
        assert xs[i].shape == (Ms[i].shape[0], k)
        assert rel_l2(xs[i].cpu().numpy(), direct[i].solve(bs[i])) < BAR, (n, k)
        assert rel_l2(ys[i].cpu().numpy(), direct[i].solve(gs[i])) < BAR, (n, k)


def test_forward_backward_through_autograd(batch_case):
    names, Ms, direct, verts = batch_case
    us = [t(rhs(M.shape[0], 3, 20 + i)).requires_grad_(True) for i, M in enumerate(Ms)]
    gs = [rhs(M.shape[0], 3, 200 + i) for i, M in enumerate(Ms)]
    xs = from_differential_batch(Ms, us)
    sum((x * t(g)).sum() for x, g in zip(xs, gs)).backward()
    for i, n in enumerate(names):
        assert rel_l2(xs[i].detach().cpu().numpy(), direct[i].solve(us[i].detach().cpu().numpy())) < BAR, n
        assert rel_l2(us[i].grad.cpu().numpy(), direct[i].solve(gs[i])) < BAR, n
    # the gradients are the backward solve itself, bit for bit
    s = B._cache[(tuple(id(M) for M in Ms), "Cholesky")][0]
    want = s.solve([t(g) for g in gs], backward=True)
    for i in range(len(Ms)):
        assert torch.equal(us[i].grad, want[i])
    # adjoint identity <g, M^-1 u> = <M^-1 g, u> per mesh
    for i in range(len(Ms)):
        lhs = float((t(gs[i]).double() * xs[i].detach().double()).sum())
        rhs_ = float((want[i].double() * us[i].detach().double()).sum())
        assert abs(lhs - rhs_) <= 1e-5 * max(abs(lhs), 1e-30) + 1e-6, (names[i], lhs, rhs_)


def test_meshes_are_independent_and_results_repeat(batch_case):
    names, Ms, _, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 30 + i)) for i, M in enumerate(Ms)]
    full = BatchSolver(Ms)
    x1, it1 = full.solve(bs), full.iterations
    x2, it2 = full.solve(bs), full.iterations
    rev = BatchSolver(Ms[::-1])
    xr, itr = rev.solve(bs[::-1]), rev.iterations
    n = len(Ms)
    for i in range(n):
        alone = BatchSolver([Ms[i]])
        xa = alone.solve([bs[i]])[0]
        assert torch.equal(x1[i], x2[i]) and it1[i] == it2[i], names[i]
        assert torch.equal(x1[i], xa) and it1[i] == alone.iterations[0], names[i]
        assert torch.equal(x1[i], xr[n - 1 - i]) and it1[i] == itr[n - 1 - i], names[i]
    # one-CTA meshes (<= 24 slices) take the single-mesh solver's kernel path: bitwise equal to PCGSolver
    for name in ("ico2", "ico3", "isolated", "triangle"):
        i = names.index(name)
        assert (Ms[i].shape[0] + 31) // 32 <= 24
        ref = PCGSolver(Ms[i], precond="jacobi")
        assert torch.equal(ref.solve(bs[i]), x1[i]) and ref.iterations == it1[i], name


def test_packed_input_and_streams(batch_case):
    _, Ms, _, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 40 + i)) for i, M in enumerate(Ms)]
    s = BatchSolver(Ms)
    x = s.solve(bs)
    xp = s.solve(torch.cat(bs, 0))
    assert all(torch.equal(a, b) for a, b in zip(x, xp))
    assert xp[1].data_ptr() == xp[0].data_ptr() + 4 * 3 * Ms[0].shape[0]   # views of one packed output
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        xs = s.solve(bs)
    st.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(x, xs))


def test_launches_per_solve(batch_case):
    _, Ms, _, _ = batch_case
    s = BatchSolver(Ms)
    bs = [t(rhs(M.shape[0], 3, 50 + i)) for i, M in enumerate(Ms)]
    s.solve(bs)
    n0 = N.launch_count()
    s.solve(bs)
    assert N.launch_count() - n0 == s.plan()[1]
    homo = [Ms[0], compute_matrix(*to_dev(*workloads.icosphere(2)), lambda_=5.0), compute_matrix(*to_dev(*workloads.icosphere(2)), lambda_=7.0)]
    h = BatchSolver(homo)
    assert h.plan()[1] == 1
    n0 = N.launch_count()
    h.solve([t(rhs(M.shape[0], 3, 0)) for M in homo])
    assert N.launch_count() - n0 == 1


def test_maxit_flags_only_the_slow_mesh(batch_case):
    names, Ms, _, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 60 + i)) for i, M in enumerate(Ms)]
    s = BatchSolver(Ms)
    s.solve(bs)
    its = s.iterations
    slow = names.index("plane_a0999")
    others = max(it for i, it in enumerate(its) if i != slow)
    assert its[slow] > others + 1, its
    capped = BatchSolver(Ms, maxit=others + 1)
    capped.solve(bs)
    with pytest.warns(RuntimeWarning, match=f"mesh {slow}"):
        BatchSolver(Ms, maxit=others + 1, check=True).solve(bs)
    st = capped.status
    assert st[slow] == 2 and all(v == 1 for i, v in enumerate(st) if i != slow), st
    with pytest.raises(N.NotConverged, match=f"mesh {slow}"):
        BatchSolver(Ms, maxit=others + 1, strict=True).solve(bs)
    with pytest.raises(N.NotConverged, match=f"mesh {slow}"):
        capped.raise_for_status()


def test_cg_warm_starts_cut_iterations(batch_case):
    _, Ms, _, _ = batch_case
    Ms = Ms[:6]
    us = [t(rhs(M.shape[0], 3, 70 + i)) for i, M in enumerate(Ms)]
    from_differential_batch(Ms, us, "CG")
    s = B._cache[(tuple(id(M) for M in Ms), "CG")][0]
    first = s.iterations
    from_differential_batch(Ms, [u + 1e-4 * u.abs().max() for u in us], "CG")
    second = s.iterations
    assert all(b < a for a, b in zip(first, second)), (first, second)


def test_adam_loop_tracks_the_single_mesh_loop():
    Ms, targets, us_b, us_s = [], [], [], []
    for i in range(8):
        v, f = workloads.icosphere(2 + i % 3)
        v = v + np.random.default_rng(i).normal(0, 0.01, size=v.shape).astype(np.float32)
        tv, tf = to_dev(v, f)
        M = compute_matrix(tv, tf, lambda_=float(5 + 2 * i), cotan=bool(i % 2))
        Ms.append(M)
        targets.append(t(v * 1.1))
        u0 = to_differential(M, tv)
        us_b.append(u0.clone().requires_grad_(True))
        us_s.append(u0.clone().requires_grad_(True))
    ob, os_ = AdamUniform(us_b, lr=0.01), AdamUniform(us_s, lr=0.01)
    for _ in range(50):
        ob.zero_grad()
        os_.zero_grad()
        xs = from_differential_batch(Ms, us_b)
        sum(((x - tg) ** 2).sum() for x, tg in zip(xs, targets)).backward()
        ob.step()
        sum(((from_differential(M, u) - tg) ** 2).sum() for M, u, tg in zip(Ms, us_s, targets)).backward()
        os_.step()
    for i in range(8):
        assert rel_l2(us_b[i].detach().cpu().numpy(), us_s[i].detach().cpu().numpy()) < 1e-5, i


def test_rejections(batch_case):
    _, Ms, _, _ = batch_case
    Ms = Ms[:3]
    s = BatchSolver(Ms)
    good = [t(rhs(M.shape[0], 3, 0)) for M in Ms]
    with pytest.raises(RuntimeError, match="CUDA"):
        s.solve([good[0].cpu(), good[1], good[2]])
    with pytest.raises(TypeError, match="float32"):
        s.solve([good[0].double(), good[1], good[2]])
    with pytest.raises(ValueError, match="rows"):
        s.solve([good[1], good[0], good[2]])
    with pytest.raises(ValueError, match="columns"):
        s.solve([g[:, :0] for g in good])
    with pytest.raises(ValueError, match="columns"):
        s.solve([torch.cat([g, g], 1) for g in good])
    with pytest.raises(ValueError, match="right-hand sides"):
        s.solve(good[:2])
    with pytest.raises(ValueError, match="at least one"):
        BatchSolver([])
    with pytest.raises(ValueError, match="at least one"):
        from_differential_batch([], [])
    with pytest.raises(RuntimeError, match="CUDA"):
        from_differential_batch(Ms, [g.cpu() for g in good])
    big = compute_matrix(*to_dev(*workloads.plane(280, seed=0)), lambda_=19.0)    # 78,400 rows > one cluster of 16
    with pytest.raises(ValueError, match="mesh 1.*from_differential"):
        BatchSolver([Ms[0], big])
    with pytest.raises(RuntimeError, match="SELL-32"):   # one row of 3001 entries: no SELL-32 copy (as for the single-mesh solver's fused kernel)
        BatchSolver([compute_matrix(*to_dev(*fan_mesh(3000)), lambda_=3.0)])
