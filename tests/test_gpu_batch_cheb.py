"""GPU: the batched solve with the Chebyshev preconditioner (BatchSolver / from_differential_batch with precond='chebyshev' or
a per-mesh list) against the fp64 direct-solve oracle, its outer-iteration count against the Jacobi batch, mesh independence,
the bitwise anchor to the single-mesh PCGSolver(M, precond='chebyshev'), warm starts, maxit, autograd, launches and streams.

The batch is test_gpu_batch.py's 14 meshes with one change: a Chebyshev mesh keeps 24 more bytes per row in shared memory, so
one cluster of 16 holds 48,128 rows (pattern copy) and plane(220) (48,400 rows) no longer fits; plane(200) (40,000 rows) takes
its place as the second 16-CTA mesh, and test_the_cluster_limit checks that plane(220) is rejected as Chebyshev and accepted
as Jacobi.  Under Chebyshev the meshes take cluster sizes 1 (ico*, fan1000, isolated, triangle), 2 (bunny_cot and the
alpha planes), 4 (cs2), 8 (cs4) and 16 (cs8, cs16)."""
import numpy as np
import pytest
import torch

import oracle
from largesteps_b200 import workloads, _native as N
from largesteps_b200.batch import BatchSolver, from_differential_batch
from largesteps_b200 import batch as B
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.solvers import PCGSolver
from gpu_util import DEV, to_dev, rel_l2, fan_mesh

pytestmark = pytest.mark.gpu
BAR = 1e-5


def bar(name):
    """1e-5 rel-L2 against the direct solve, except on the alpha = 0.999 plane: both preconditioners stop at the same residual
    (rtol 1e-7), which on a matrix this stiff bounds the error only to about 1e-5.  The Jacobi batch stays below 1e-5 there
    (test_gpu_batch.py), the Chebyshev batch lands at 1.0e-5 to 1.15e-5 (H100, the seeds of these tests): its last outer
    iteration is worth about three Jacobi iterations and stops at a different point below rtol.  2e-5 there."""
    return 2e-5 if name == "plane_a0999" else BAR


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def isolated_vertex_mesh():
    v, f = workloads.icosphere(2)
    return np.concatenate([v, [[2.0, 0.0, 0.0]]]).astype(np.float32), f


def meshes(bunny_mesh):
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
        "cs16": (*workloads.plane(200, seed=7), dict(lambda_=19.0)),
    }


@pytest.fixture(scope="module")
def batch_case(bunny_mesh):
    ms = meshes(bunny_mesh)
    names = list(ms)
    Ms, direct = [], []
    for n in names:
        v, f, kw = ms[n]
        Ms.append(compute_matrix(*to_dev(v, f), **kw))
        r, c, val, V = oracle.compute_matrix(v, f, **kw)
        direct.append(oracle.DirectSolver(r, c, val, V))
    return names, Ms, direct


def rhs(V, k, seed):
    return np.random.default_rng(seed).normal(size=(V, k)).astype(np.float32)


def mixed(n):
    """Chebyshev on the even meshes, Jacobi on the odd ones"""
    return ["chebyshev" if i % 2 == 0 else "jacobi" for i in range(n)]


def test_plan_covers_every_cluster_size(batch_case):
    names, Ms, _ = batch_case
    s = BatchSolver(Ms, precond="chebyshev")
    plan, ng = s.plan()
    sizes = {names[i]: p[0] for i, p in enumerate(plan)}
    assert {p[0] for p in plan} == {1, 2, 4, 8, 16}, sizes
    assert all(p[1] == 2 for p in plan), plan                     # never RES 3
    assert sizes["bunny_cot"] == 2 and sizes["plane_a0999"] == 2 and sizes["cs16"] == 16, sizes
    assert ng == len({p[2] for p in plan})
    m = BatchSolver(Ms, precond=mixed(len(Ms)))
    mplan, mng = m.plan()
    for i, p in enumerate(mplan):
        if i % 2 == 0:
            assert p[:2] == plan[i][:2], names[i]
    assert mng > ng


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("mode", ["chebyshev", "mixed"])
def test_accuracy_against_the_direct_solve(batch_case, k, mode):
    names, Ms, direct = batch_case
    s = BatchSolver(Ms, precond="chebyshev" if mode == "chebyshev" else mixed(len(Ms)))
    bs = [rhs(M.shape[0], k, 10 + i) for i, M in enumerate(Ms)]
    gs = [rhs(M.shape[0], k, 100 + i) for i, M in enumerate(Ms)]
    xs = s.solve([t(b) for b in bs])
    assert all(st == 1 for st in s.status), s.status
    ys = s.solve([t(g) for g in gs], backward=True)
    assert all(st == 1 for st in s.status), s.status
    for i, n in enumerate(names):
        assert xs[i].shape == (Ms[i].shape[0], k)
        assert rel_l2(xs[i].cpu().numpy(), direct[i].solve(bs[i])) < bar(n), (n, k)
        assert rel_l2(ys[i].cpu().numpy(), direct[i].solve(gs[i])) < bar(n), (n, k)


def test_outer_iterations_against_the_jacobi_batch(batch_case):
    """the single-mesh solver's bound (test_gpu_pcg.py): itc <= (itj + 2) // 3 + 2 for every mesh on more than one CTA"""
    names, Ms, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 80 + i)) for i, M in enumerate(Ms)]
    jac = BatchSolver(Ms)
    jac.solve(bs)
    che = BatchSolver(Ms, precond="chebyshev")
    che.solve(bs)
    plan, _ = che.plan()
    itj, itc = jac.iterations, che.iterations
    checked = 0
    for i, n in enumerate(names):
        print(f"{n:>12}: cluster {plan[i][0]:2d}  Jacobi {itj[i]:4d}  Chebyshev {itc[i]:4d}")
        if plan[i][0] > 1:
            assert itc[i] <= (itj[i] + 2) // 3 + 2, (n, itj[i], itc[i])
            checked += 1
    assert checked >= 7


def test_meshes_are_independent_and_results_repeat(batch_case):
    names, Ms, _ = batch_case
    n = len(Ms)
    bs = [t(rhs(M.shape[0], 3, 30 + i)) for i, M in enumerate(Ms)]
    full = BatchSolver(Ms, precond="chebyshev")
    x1, it1 = full.solve(bs), full.iterations
    x2, it2 = full.solve(bs), full.iterations
    rev = BatchSolver(Ms[::-1], precond="chebyshev")
    xr, itr = rev.solve(bs[::-1]), rev.iterations
    mix = BatchSolver(Ms, precond=mixed(n))
    xm, itm = mix.solve(bs), mix.iterations
    mix2 = BatchSolver(Ms, precond=["jacobi" if p == "chebyshev" else "chebyshev" for p in mixed(n)])
    xm2, itm2 = mix2.solve(bs), mix2.iterations
    jac = BatchSolver(Ms)
    xj, itj = jac.solve(bs), jac.iterations
    for i in range(n):
        alone = BatchSolver([Ms[i]], precond="chebyshev")
        xa = alone.solve([bs[i]])[0]
        assert torch.equal(x1[i], x2[i]) and it1[i] == it2[i], names[i]
        assert torch.equal(x1[i], xa) and it1[i] == alone.iterations[0], names[i]
        assert torch.equal(x1[i], xr[n - 1 - i]) and it1[i] == itr[n - 1 - i], names[i]
        # in a batch mixed with Jacobi meshes: Chebyshev meshes as in the all-Chebyshev batch, Jacobi meshes as in the Jacobi batch
        xc, ic = (xm[i], itm[i]) if i % 2 == 0 else (xm2[i], itm2[i])
        xo, io = (xm2[i], itm2[i]) if i % 2 == 0 else (xm[i], itm[i])
        assert torch.equal(x1[i], xc) and it1[i] == ic, names[i]
        assert torch.equal(xj[i], xo) and itj[i] == io, names[i]


def test_bitwise_equal_to_the_single_mesh_solver(batch_case):
    """meshes of <= 24 slices: the single-mesh PCGSolver(M, precond='chebyshev') runs them on a cluster of one CTA at RES 2 with
    the same coefficients -- the batch gives the same bits and iteration counts"""
    names, Ms, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 90 + i)) for i, M in enumerate(Ms)]
    full = BatchSolver(Ms, precond="chebyshev")
    xs, its = full.solve(bs), full.iterations
    checked = 0
    for name in ("ico2", "ico3", "isolated", "triangle"):
        i = names.index(name)
        assert (Ms[i].shape[0] + 31) // 32 <= 24
        ref = PCGSolver(Ms[i], precond="chebyshev")
        d = ref.describe()
        assert d["precond"] == "chebyshev" and d["cluster"] == 1 and d["residency"] == 2, (name, d)
        for k in (3, 1):
            x = ref.solve(bs[i][:, :k].contiguous())
            y = full.solve([b[:, :k].contiguous() for b in bs])[i] if k != 3 else xs[i]
            it = full.iterations[i] if k != 3 else its[i]
            assert torch.equal(x, y) and ref.iterations == it, (name, k, ref.iterations, it)
        checked += 1
    assert checked == 4


def test_packed_input_and_streams(batch_case):
    _, Ms, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 40 + i)) for i, M in enumerate(Ms)]
    s = BatchSolver(Ms, precond="chebyshev")
    x = s.solve(bs)
    xp = s.solve(torch.cat(bs, 0))
    assert all(torch.equal(a, b) for a, b in zip(x, xp))
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        xs = s.solve(bs)
    st.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(x, xs))


@pytest.mark.parametrize("mode", ["chebyshev", "mixed"])
def test_launches_per_solve(batch_case, mode):
    _, Ms, _ = batch_case
    s = BatchSolver(Ms, precond="chebyshev" if mode == "chebyshev" else mixed(len(Ms)))
    bs = [t(rhs(M.shape[0], 3, 50 + i)) for i, M in enumerate(Ms)]
    s.solve(bs)
    n0 = N.launch_count()
    s.solve(bs)
    assert N.launch_count() - n0 == s.plan()[1]
    homo = [Ms[0], compute_matrix(*to_dev(*workloads.icosphere(2)), lambda_=5.0), compute_matrix(*to_dev(*workloads.icosphere(3)), lambda_=7.0)]
    h = BatchSolver(homo, precond="chebyshev")
    assert h.plan()[1] == 1
    n0 = N.launch_count()
    h.solve([t(rhs(M.shape[0], 3, 0)) for M in homo])
    assert N.launch_count() - n0 == 1


def test_maxit_flags_only_the_slow_mesh(batch_case):
    names, Ms, _ = batch_case
    bs = [t(rhs(M.shape[0], 3, 60 + i)) for i, M in enumerate(Ms)]
    s = BatchSolver(Ms, precond="chebyshev")
    s.solve(bs)
    its = s.iterations
    slow = names.index("plane_a0999")
    others = max(it for i, it in enumerate(its) if i != slow)
    assert its[slow] > others + 1, its
    capped = BatchSolver(Ms, maxit=others + 1, precond="chebyshev")
    capped.solve(bs)
    st = capped.status
    assert st[slow] == 2 and all(v == 1 for i, v in enumerate(st) if i != slow), st
    with pytest.warns(RuntimeWarning, match=f"mesh {slow}"):
        BatchSolver(Ms, maxit=others + 1, check=True, precond="chebyshev").solve(bs)
    with pytest.raises(N.NotConverged, match=f"mesh {slow}"):
        BatchSolver(Ms, maxit=others + 1, strict=True, precond="chebyshev").solve(bs)
    with pytest.raises(N.NotConverged, match=f"mesh {slow}"):
        capped.raise_for_status()


def test_forward_backward_through_autograd(batch_case):
    names, Ms, direct = batch_case
    us = [t(rhs(M.shape[0], 3, 20 + i)).requires_grad_(True) for i, M in enumerate(Ms)]
    gs = [rhs(M.shape[0], 3, 200 + i) for i, M in enumerate(Ms)]
    xs = from_differential_batch(Ms, us, precond="chebyshev")
    sum((x * t(g)).sum() for x, g in zip(xs, gs)).backward()
    for i, n in enumerate(names):
        assert rel_l2(xs[i].detach().cpu().numpy(), direct[i].solve(us[i].detach().cpu().numpy())) < bar(n), n
        assert rel_l2(us[i].grad.cpu().numpy(), direct[i].solve(gs[i])) < bar(n), n
    ids = tuple(id(M) for M in Ms)
    s = B._cache[(ids, "Cholesky", ("chebyshev",) * len(Ms))][0]
    assert s.precond == ["chebyshev"] * len(Ms)
    want = s.solve([t(g) for g in gs], backward=True)
    for i in range(len(Ms)):
        assert torch.equal(us[i].grad, want[i])
    for i in range(len(Ms)):
        lhs = float((t(gs[i]).double() * xs[i].detach().double()).sum())
        rhs_ = float((want[i].double() * us[i].detach().double()).sum())
        assert abs(lhs - rhs_) <= 1e-5 * max(abs(lhs), 1e-30) + 1e-6, (names[i], lhs, rhs_)
    # the preconditioner is part of the cache key: the Jacobi solver of the same matrices is another object
    from_differential_batch(Ms, [u.detach() for u in us])
    assert B._cache[(ids, "Cholesky")][0] is not s
    from_differential_batch(Ms, [u.detach() for u in us], precond=mixed(len(Ms)))
    assert B._cache[(ids, "Cholesky", tuple(mixed(len(Ms))))][0].precond == mixed(len(Ms))


def test_cg_warm_starts_cut_iterations(batch_case):
    _, Ms, _ = batch_case
    Ms = Ms[:6]
    for precond in ("chebyshev", mixed(len(Ms))):
        us = [t(rhs(M.shape[0], 3, 70 + i)).requires_grad_(True) for i, M in enumerate(Ms)]
        gs = [t(rhs(M.shape[0], 3, 170 + i)) for i, M in enumerate(Ms)]
        sum((x * g).sum() for x, g in zip(from_differential_batch(Ms, us, "CG", precond=precond), gs)).backward()
        key = (tuple(id(M) for M in Ms), "CG", tuple(B.preconditioners(precond, len(Ms))))
        s = B._cache[key][0]
        assert s.guess_fwd is not None and s.guess_bwd is not None and s.guess_fwd is not s.guess_bwd
        bwd_first = s.iterations
        fwd = from_differential_batch(Ms, [u.detach() + 1e-4 * u.detach().abs().max() for u in us], "CG", precond=precond)
        fwd_second = s.iterations
        # the forward warm start is the forward solution, the backward one the backward solution
        gb = s.guess_bwd.clone()
        assert torch.equal(torch.cat(fwd, 0), s.guess_fwd)
        ys = s.solve([g + 1e-4 * g.abs().max() for g in gs], backward=True)
        assert all(b < a for a, b in zip(bwd_first, s.iterations)), (bwd_first, s.iterations)
        assert not torch.equal(gb, s.guess_bwd) and torch.equal(torch.cat(ys, 0), s.guess_bwd)
        cold = BatchSolver(Ms, precond=precond)
        cold.solve([u.detach() + 1e-4 * u.detach().abs().max() for u in us])
        assert all(b < a for a, b in zip(cold.iterations, fwd_second)), (cold.iterations, fwd_second)


def test_the_cluster_limit(batch_case):
    _, Ms, _ = batch_case
    big = compute_matrix(*to_dev(*workloads.plane(220, seed=0)), lambda_=19.0)    # 48,400 rows > 48,128 with Chebyshev
    with pytest.raises(ValueError, match="mesh 1.*Chebyshev.*from_differential"):
        BatchSolver([Ms[0], big], precond="chebyshev")
    s = BatchSolver([Ms[0], big], precond=["chebyshev", "jacobi"])
    plan, ng = s.plan()
    assert plan[1][:2] == (16, 2) and plan[0][:2] == (1, 2) and ng == 2
    b = [t(rhs(M.shape[0], 3, 7 + i)) for i, M in enumerate([Ms[0], big])]
    s.solve(b)
    assert s.status == [1, 1]
    with pytest.raises(ValueError, match="Unknown preconditioner"):
        BatchSolver(Ms[:2], precond="auto")
    with pytest.raises(ValueError, match="preconditioners for 2 meshes"):
        BatchSolver(Ms[:2], precond=["chebyshev"])
