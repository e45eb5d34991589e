"""GPU parity: from_differential / the solver plug-ins (csrc/ls_pcg.cu through the C ABI) vs the fp64 direct-solve
oracle on identical seeded inputs.  Bar (north_star): vertex positions within 1e-5 rel-L2, forward and backward."""
import gc
import warnings

import numpy as np
import pytest
import torch

import oracle
from largesteps_b200 import workloads, _native as N
from largesteps_b200.geometry import compute_matrix
from largesteps_b200 import parameterize
from largesteps_b200.parameterize import to_differential, from_differential
from largesteps_b200.solvers import (PCGSolver, CholeskySolver, ConjugateGradientSolver, plan, solve)
from gpu_util import DEV, to_dev, rel_l2, rhs, config1, config2, coo_np

pytestmark = pytest.mark.gpu
BAR = 1e-5


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def direct_for(v, f, kw):
    r, c, val, V = oracle.compute_matrix(v, f, **kw)
    return (r, c, val, V), oracle.DirectSolver(r, c, val, V)


@pytest.mark.parametrize("cfg", ["config1", "config2"])
def test_baseline_configs_forward_backward(cfg, bunny_mesh):
    """BASELINE configs 1 (icosphere 2562 V, uniform, lambda=10) and 2 (bunny x2 subdiv 52786 V, cot, lambda=19)."""
    v, f, kw = config1() if cfg == "config1" else config2(bunny_mesh)
    (r, c, val, V), ds = direct_for(v, f, kw)
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    for method in ("Cholesky", "CG", "PCG"):
        u = t(b).requires_grad_(True)
        x = from_differential(M, u, method)
        assert rel_l2(x.detach().cpu().numpy(), ds.solve(b)) < BAR, method
        # backward with O(1) gradients and with tiny gradients (the reference's absolute tolerance fails the latter)
        for scale in (1.0, 1e-4):
            u.grad = None
            gg = (scale * g).astype(np.float32)
            x = from_differential(M, u, method)
            (x * t(gg)).sum().backward()
            assert rel_l2(u.grad.cpu().numpy(), ds.solve(gg)) < BAR, (method, scale)


def test_against_reference_outputs(golden_assembly, golden_solve):
    """Same inputs as the unmodified reference ran on (tests/golden/solve.npz)."""
    g, s = golden_assembly, golden_solve
    for mesh, kw in (("ico2", dict(lambda_=10.0)), ("bunny", dict(lambda_=19.0, cotan=True))):
        M = compute_matrix(*to_dev(g[f"{mesh}.verts"], g[f"{mesh}.faces"]), **kw)
        u = t(s[f"{mesh}.b"]).requires_grad_(True)
        vout = from_differential(M, u, "Cholesky")
        (vout * t(s[f"{mesh}.g"])).sum().backward()
        assert rel_l2(vout.detach().cpu().numpy(), s[f"{mesh}.fd_v"]) < BAR       # reference CG forward result
        r, c, val, V = oracle.compute_matrix(g[f"{mesh}.verts"], g[f"{mesh}.faces"], **kw)
        ds = oracle.DirectSolver(r, c, val, V)
        assert rel_l2(u.grad.cpu().numpy(), ds.solve(s[f"{mesh}.g"])) < BAR
        # and we are *closer* to the exact gradient than the reference's absolute-tolerance CG was
        assert rel_l2(u.grad.cpu().numpy(), ds.solve(s[f"{mesh}.g"])) < rel_l2(s[f"{mesh}.fd_grad"], ds.solve(s[f"{mesh}.g"]))


@pytest.mark.parametrize("alpha", [0.5, 0.95, 0.99])
def test_plane_alpha(alpha):
    v, f = workloads.plane(300, seed=0)
    kw = dict(lambda_=1.0, alpha=alpha)
    (r, c, val, V), ds = direct_for(v, f, kw)
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    s = PCGSolver(M)
    assert rel_l2(s.solve(t(b)).cpu().numpy(), ds.solve(b)) < BAR
    assert 0 < s.iterations < 2000 and max(s.relres[:3]) <= 5e-5
    assert rel_l2(s.solve(t(g), backward=True).cpu().numpy(), ds.solve(g)) < BAR


@pytest.mark.parametrize("n", [200, 500])
def test_ill_conditioned_alpha_0999(n):
    """alpha = 0.999 (figures/influence/generate_data.py:28), kappa ~ 1.2e4: the stress case.  The north-star bar (1e-5)
    holds here too: the solve restarts from the fp64-accumulated true residual when the recursive one has drifted."""
    v, f = workloads.plane(n, seed=0)
    kw = dict(lambda_=1.0, alpha=0.999)
    (r, c, val, V), ds = direct_for(v, f, kw)
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    s = PCGSolver(M)
    err = rel_l2(s.solve(t(b)).cpu().numpy(), ds.solve(b))
    print(f"alpha=0.999 n={n}: fwd err {err:.2e}, iterations {s.iterations}, restarts {s.restarts}")
    assert err < BAR, err
    assert s.iterations < 5000 and s.restarts <= 1
    errb = rel_l2(s.solve(t(g), backward=True).cpu().numpy(), ds.solve(g))
    print(f"alpha=0.999 n={n}: bwd err {errb:.2e}, iterations {s.iterations}, restarts {s.restarts}")
    assert errb < BAR, errb
    # the default plug-in (what from_differential uses) takes the same path
    u = t(b).requires_grad_(True)
    x = from_differential(M, u)
    (x * t(g)).sum().backward()
    assert rel_l2(x.detach().cpu().numpy(), ds.solve(b)) < BAR and rel_l2(u.grad.cpu().numpy(), ds.solve(g)) < BAR
    # without the guard the recurrence-carried s = A p may drift past the bar over ~600 iterations: documented, not asserted
    s0 = PCGSolver(M, refine=0)
    e0 = rel_l2(s0.solve(t(b)).cpu().numpy(), ds.solve(b))
    print(f"alpha=0.999 n={n}: refine=0 err {e0:.2e}, iterations {s0.iterations}")
    assert e0 < 1e-4


@pytest.mark.parametrize("k", [1, 2, 4, 6])
def test_column_counts(k):
    v, f = workloads.icosphere(3)
    kw = dict(lambda_=10.0)
    (r, c, val, V), ds = direct_for(v, f, kw)
    b = np.random.default_rng(k).normal(size=(V, k)).astype(np.float32)
    M = compute_matrix(*to_dev(v, f), **kw)
    x = PCGSolver(M).solve(t(b))
    assert x.shape == (V, k)
    assert rel_l2(x.cpu().numpy(), ds.solve(b)) < BAR


@pytest.mark.parametrize("res", ["2", "1", "0"])
def test_two_and_four_columns_on_the_cooperative_grid(res, monkeypatch):
    """k = 4 runs the 4-column instantiations of the fused kernel, k = 2 the 3-column ones with a runtime column count; here on
    the cooperative grid at every residency level (test_column_counts covers the one-CTA path)."""
    monkeypatch.setenv("LS_PCG_RES", res)
    v, f = workloads.plane(120, seed=3)
    kw = dict(lambda_=1.0, alpha=0.9)
    (r, c, val, V), ds = direct_for(v, f, kw)
    M = compute_matrix(*to_dev(v, f), **kw)
    s = PCGSolver(M)
    d = s.describe()
    assert d["algo"] == "fused" and d["cluster"] == 0 and d["residency"] == int(res)
    for k in (4, 2):
        b = np.random.default_rng(k).normal(size=(V, k)).astype(np.float32)
        x = s.solve(t(b))
        assert x.shape == (V, k) and s.status == 1
        assert rel_l2(x.cpu().numpy(), ds.solve(b)) < BAR


def test_columns_freeze_independently_and_zero_rhs():
    v, f = workloads.icosphere(3)
    (r, c, val, V), ds = direct_for(v, f, dict(lambda_=10.0))
    M = compute_matrix(*to_dev(v, f), 10.0)
    s = PCGSolver(M)
    z = s.solve(torch.zeros(V, 3, device=DEV))
    assert float(z.abs().max()) == 0.0 and s.iterations == 0
    b = np.random.default_rng(0).normal(size=(V, 3)).astype(np.float32)
    b[:, 1] = 0.0                      # one zero column
    b[:, 2] *= 1e-6                    # one tiny column: relative tolerance must still hold
    x = s.solve(t(b)).cpu().numpy()
    xd = ds.solve(b)
    assert np.abs(x[:, 1]).max() == 0.0
    assert rel_l2(x[:, 0], xd[:, 0]) < BAR and rel_l2(x[:, 2], xd[:, 2]) < BAR


def test_warm_start_like_reference_cg():
    v, f = workloads.plane(200, seed=0)
    kw = dict(lambda_=1.0, alpha=0.95)
    (r, c, val, V), ds = direct_for(v, f, kw)
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    s = ConjugateGradientSolver(M)
    x1 = s.solve(t(b))
    it_cold = s.iterations
    b2 = (b + 1e-3 * np.random.default_rng(7).normal(size=b.shape)).astype(np.float32)   # an optimiser-sized change
    x2 = s.solve(t(b2))
    it_warm = s.iterations
    assert it_warm < it_cold
    assert rel_l2(x2.cpu().numpy(), ds.solve(b2)) < BAR
    # backward guess is kept separately (solvers.py:107-110)
    xb = s.solve(t(g), backward=True)
    assert rel_l2(xb.cpu().numpy(), ds.solve(g)) < BAR
    assert s.guess_fwd is x2 and s.guess_bwd is xb
    # solving the same system again from its own solution needs only a few clean-up iterations
    # (the true fp32 residual of the previous answer sits slightly above the recursive one)
    s.solve(t(b2))
    assert s.iterations <= it_cold // 3
    # a warm start that is worse than x = 0 (RHS scale changed by 1e4) falls back to a cold start
    tiny = (1e-4 * g).astype(np.float32)
    xt = s.solve(t(tiny), backward=True)
    assert rel_l2(xt.cpu().numpy(), ds.solve(tiny)) < BAR


def test_morton_reorder_is_transparent(bunny_mesh):
    """The solver's private copy of M is re-ordered along a Morton curve (csrc/ls_order.cu); b and x stay in the
    caller's numbering, and the answer is the same as without re-ordering."""
    from largesteps_b200.geometry import morton_order, order_of
    v, f = bunny_mesh
    v, f = workloads.subdivide(v, f)
    v, f = workloads.shuffle_vertices(v.astype(np.float32), f, seed=11)      # worst-case native numbering
    kw = dict(lambda_=19.0, cotan=True)
    (r, c, val, V), ds = direct_for(v, f, kw)
    tv, tf = to_dev(v, f)
    M = compute_matrix(tv, tf, **kw)
    perm = order_of(M)
    assert perm is not None and perm.dtype == torch.int32
    assert sorted(perm.cpu().tolist()) == list(range(V))                      # a permutation
    assert torch.equal(perm, morton_order(tv))                                # deterministic
    # locality: consecutive new rows are close in space (median hop << random-order hop)
    pv = tv[perm.long()]
    hop = (pv[1:] - pv[:-1]).norm(dim=1).median().item()
    hop_native = (tv[1:] - tv[:-1]).norm(dim=1).median().item()
    assert hop < 0.2 * hop_native
    _, b, g = rhs(r, c, val, V, v)
    x_re = PCGSolver(M, reorder=True).solve(t(b))
    x_no = PCGSolver(M, reorder=False).solve(t(b))
    xd = ds.solve(b)
    assert rel_l2(x_re.cpu().numpy(), xd) < BAR and rel_l2(x_no.cpu().numpy(), xd) < BAR
    assert rel_l2(x_re.cpu().numpy(), x_no.cpu().numpy()) < 2e-6
    # warm start and backward go through the same permutation
    s = ConjugateGradientSolver(M)
    s.solve(t(b))
    assert rel_l2(s.solve(t(b)).cpu().numpy(), xd) < BAR
    assert rel_l2(s.solve(t(g), backward=True).cpu().numpy(), ds.solve(g)) < BAR
    # a bogus permutation is rejected
    import ctypes
    from largesteps_b200.geometry import csr_of
    rowptr, col, vals = csr_of(M)
    bad = perm.clone()
    bad[0] = bad[1]
    nbytes = ctypes.c_size_t(0)
    N.lib().ls_pcg_workspace_bytes(V, vals.shape[0], 4, ctypes.byref(nbytes))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=DEV)
    h = ctypes.c_void_p(0)
    rc = N.lib().ls_pcg_create(ctypes.byref(h), V, vals.shape[0], N.ptr(rowptr), N.ptr(col), N.ptr(vals), N.ptr(bad),
                               1, 4, N.ptr(ws), nbytes.value, N.stream_ptr(torch.device(DEV)))
    assert rc == N.LS_ERR_BAD_ARG and "permutation" in N.last_error()


MODES = [
    {},                                                         # default: fused kernel on the cooperative grid (one CTA for tiny meshes), pattern copy if uniform
    {"LS_PCG_CLUSTER": "16"},                                   # one thread-block cluster of 16 CTAs (DSMEM all-reduce, barrier.cluster)
    {"LS_PCG_CLUSTER": "16", "LS_PCG_RES": "2"},                # ... publishing through global memory (the cluster-resident rows switched off)
    {"LS_PCG_CLRES": "384"},                                    # cluster-resident mode (opt-in): <= 12 K vertices in one cluster, rows gathered through DSMEM
    {"LS_PCG_CLRES": "384", "LS_PCG_SMALLCTA": "0"},            # ... 768-thread CTAs
    {"LS_PCG_CLRES": "384", "LS_PCG_PATTERN": "0"},             # ... general matrix copy
    {"LS_PCG_CLUSTER": "0"},                                    # fused, cooperative grid, everything in shared memory (256-thread CTAs)
    {"LS_PCG_CLUSTER": "0", "LS_PCG_SMALLCTA": "0"},            # ... 768-thread CTAs
    {"LS_PCG_CLUSTER": "0", "LS_PCG_RES": "1"},                 # ... x / p in global memory
    {"LS_PCG_CLUSTER": "0", "LS_PCG_RES": "0"},                 # ... every vector in global memory
    {"LS_PCG_CLUSTER": "0", "LS_PCG_FASTRED": "0"},             # fenced partial-array all-reduce only
    {"LS_PCG_CLUSTER": "0", "LS_PCG_FASTRED": "11"},            # fast all-reduce for 11 reductions, then the fenced one takes over mid-solve
    {"LS_PCG_CLUSTER": "4"},                                    # one cluster of 4 / 8 CTAs (meshes that do not fit fall back to the grid)
    {"LS_PCG_CLUSTER": "8"},
    {"LS_PCG_PATTERN": "0"},                                    # general matrix copy even for uniform Laplacians
    {"LS_PCG_REFINE": "0"},                                     # no true-residual check
    {"LS_PCG_MODE": "graph"},                                   # CUDA graph of 3 kernels per iteration, SELL SpMM engine (TMA-staged)
    {"LS_PCG_MODE": "graph", "LS_SELL_TMA": "0"},               # ... register-prefetch SELL kernel
    {"LS_PCG_MODE": "graph", "LS_SPMM_ENGINE": "csr"},          # ... with the TMA-staged CSR SpMM engine
    {"LS_FORCE_REORDER": "1"},                                  # Morton re-ordered private copy
]


def mode_cases(bunny_mesh):
    return [config2(bunny_mesh), (*workloads.plane(260, seed=1), dict(lambda_=1.0, alpha=0.95)),
            (*workloads.icosphere(5), dict(lambda_=10.0)), (*workloads.icosphere(3), dict(lambda_=10.0)),
            (*workloads.plane(50, seed=2), dict(lambda_=19.0, cotan=True))]


def mode_id(env):
    return ",".join(f"{k[3:]}={v}" for k, v in env.items()) or "default"


@pytest.mark.parametrize("env", MODES, ids=mode_id)
def test_every_solver_mode_meets_the_bar(env, bunny_mesh, monkeypatch):
    """All execution modes of the solve (selected at handle creation) give the direct-solve answer."""
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count     # the cooperative grid is one CTA per SM
    for v, f, kw in mode_cases(bunny_mesh):
        (r, c, val, V), ds = direct_for(v, f, kw)
        _, b, g = rhs(r, c, val, V, v)
        M = compute_matrix(*to_dev(v, f), **kw)
        s = PCGSolver(M)
        d = s.describe()
        uniform = not kw.get("cotan")
        if env.get("LS_PCG_MODE") == "graph":
            assert d["algo"] == "graph" and d["persistent"] == 0
            assert d["sell_engine"] == (0 if env.get("LS_SPMM_ENGINE") == "csr" else 1)
        else:
            assert d["algo"] == "fused"
            assert d["sell_engine"] == (2 if uniform and env.get("LS_PCG_PATTERN") != "0" else 1)
            tiny = V <= 24 * 32                      # <= 24 slices (one per warp): one CTA holds everything, gathered vector included
            if env.get("LS_PCG_CLUSTER") == "0":
                assert d["cluster"] == 0 and d["grid"] == min(sms, (V + 31) // 32)
                assert d["residency"] == int(env.get("LS_PCG_RES", "2"))
                if not tiny:
                    per_cta = -(-((V + 31) // 32) // d["grid"])          # slices per CTA: the 256-thread CTA takes up to 16
                    small = env.get("LS_PCG_SMALLCTA") != "0" and d["residency"] == 2 and per_cta <= 16
                    assert d["threads"] == (256 if small else 768)
            elif "LS_PCG_CLUSTER" in env:
                assert d["cluster"] in (0, int(env["LS_PCG_CLUSTER"]))
                if V < 20000:
                    assert d["cluster"] == int(env["LS_PCG_CLUSTER"])
            elif tiny:
                assert d["cluster"] == 1 and d["grid"] == 1 and d["residency"] == int(env.get("LS_PCG_RES", "3"))
            elif V <= 32 * int(env.get("LS_PCG_CLRES", "0")):
                # a few thousand vertices: one cluster of 16 CTAs, the published rows gathered through distributed shared memory
                assert d["cluster"] == 16 and d["grid"] == 16 and d["residency"] == 4
                assert d["threads"] == (256 if (V + 31) // 32 <= 16 * 8 and env.get("LS_PCG_SMALLCTA") != "0" else 768)
            else:
                assert d["cluster"] == 0 and d["grid"] == min(sms, (V + 31) // 32) and d["residency"] == 2
        if "LS_FORCE_REORDER" in env and V >= 8192:      # (smaller meshes carry no Morton order: everything is cache resident)
            assert d["reordered"] == 1
        assert rel_l2(s.solve(t(b)).cpu().numpy(), ds.solve(b)) < BAR, (env, kw)
        assert 0 < s.iterations < 1000 and max(s.relres[:3]) <= 5e-5     # relres is the TRUE residual once the guard has run
        assert rel_l2(s.solve(t(g), backward=True).cpu().numpy(), ds.solve(g)) < BAR, (env, kw)
        # warm start through the same path (the reference CG plug-in's behaviour, solvers.py:102-110)
        w = PCGSolver(M, warm_start=True)
        x1 = w.solve(t(b))
        it_cold = w.iterations
        b2 = (b + 1e-3 * np.random.default_rng(7).normal(size=b.shape)).astype(np.float32)
        assert rel_l2(w.solve(t(b2)).cpu().numpy(), ds.solve(b2)) < BAR, (env, kw)
        assert w.iterations < it_cold


@pytest.fixture(scope="module")
def mode_matrices(bunny_mesh):
    return [compute_matrix(*to_dev(v, f), **kw) for v, f, kw in mode_cases(bunny_mesh)]


@pytest.mark.parametrize("env", MODES, ids=mode_id)
def test_describe_matches_the_host_plan(env, mode_matrices, monkeypatch):
    """The launch plan the handle reports is the one the host-only planner (solvers.plan, tested on the CPU) computes."""
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    props = torch.cuda.get_device_properties(DEV)
    for M in mode_matrices:
        for precond in ("jacobi", "chebyshev", "auto"):
            s = PCGSolver(M, precond=precond)
            d = s.describe()
            args = ((M.shape[0] + 31) // 32, s.pattern_copy()["on"], props.multi_processor_count, props.shared_memory_per_block_optin)
            p = plan(*args, precond=precond)
            if p.get("cluster", 0) > 1 and d.get("cluster") == 0:
                # a cluster the device cannot schedule falls back to the cooperative grid (test_every_solver_mode_meets_the_bar
                # allows it for meshes of 20 000 vertices and more)
                assert M.shape[0] >= 20000
                with monkeypatch.context() as m:
                    m.setenv("LS_PCG_CLUSTER", "0")
                    p = plan(*args, precond=precond)
            assert {k: d.get(k) for k in p} == p, (M.shape[0], precond, d, p)


@pytest.mark.parametrize("env", [{}, {"LS_PCG_CLUSTER": "0", "LS_PCG_RES": "1"}, {"LS_PCG_CLUSTER": "0", "LS_PCG_RES": "0"},
                                 {"LS_PCG_CLUSTER": "8"}], ids=["default", "res1", "res0", "cluster8"])
def test_chebyshev_preconditioner(env, bunny_mesh, monkeypatch):
    """precond = 2: a degree-3 Chebyshev polynomial in D^-1 M on top of Jacobi (SURVEY 8 f3).  Same answers; at alpha = 0.999
    (kappa ~ 1.2e4) at most a third of the Jacobi iterations, i.e. a third of the all-reduces."""
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)
    cases = [(*workloads.plane(200, seed=0), dict(lambda_=1.0, alpha=0.999)), config2(bunny_mesh),
             (*workloads.icosphere(3), dict(lambda_=10.0))]
    for v, f, kw in cases:
        (r, c, val, V), ds = direct_for(v, f, kw)
        _, b, g = rhs(r, c, val, V, v)
        M = compute_matrix(*to_dev(v, f), **kw)
        sj = PCGSolver(M)
        xj = sj.solve(t(b))
        itj = sj.iterations
        sc = PCGSolver(M, precond="chebyshev")
        assert sc.describe()["algo"] == "fused"
        xc = sc.solve(t(b))
        itc = sc.iterations
        print(f"V={V} {kw}: Jacobi {itj} iterations, Chebyshev {itc}")
        assert rel_l2(xc.cpu().numpy(), ds.solve(b)) < BAR and rel_l2(xj.cpu().numpy(), ds.solve(b)) < BAR
        assert rel_l2(sc.solve(t(g), backward=True).cpu().numpy(), ds.solve(g)) < BAR
        assert itc <= (itj + 2) // 3 + 2, (itj, itc)
        assert torch.equal(sc.solve(t(b)), xc)          # deterministic
        w = PCGSolver(M, precond="chebyshev", warm_start=True)
        w.solve(t(b))
        b2 = (b + 1e-3 * np.random.default_rng(7).normal(size=b.shape)).astype(np.float32)
        assert rel_l2(w.solve(t(b2)).cpu().numpy(), ds.solve(b2)) < BAR and w.iterations <= itc
    with pytest.raises(ValueError, match="Unknown preconditioner"):
        PCGSolver(M, precond="ic0")


def test_auto_preconditioner_choice(bunny_mesh):
    """from_differential's plug-ins use precond='auto': Chebyshev where it is measured faster (cooperative grid with every solver
    vector in shared memory), Jacobi for one-CTA meshes and for meshes too large for that residency level."""
    for (v, f, kw), want in ((config2(bunny_mesh), "chebyshev"), ((*workloads.icosphere(3), dict(lambda_=10.0)), "jacobi"),
                             ((*workloads.plane(800, seed=0), dict(lambda_=1.0, alpha=0.95)), "jacobi")):
        M = compute_matrix(*to_dev(v, f), **kw)
        assert CholeskySolver(M).describe()["precond"] == want
        assert PCGSolver(M).describe()["precond"] == "jacobi"


def test_two_live_solvers_of_different_size():
    """Handles of different sizes share kernel functions: the opt-in shared-memory attribute of a function must never
    be lowered by a later, smaller handle (ADVICE r1).  Interleave solves of a big and a small mesh."""
    big_v, big_f = workloads.plane(700, seed=0)
    small_v, small_f = workloads.plane(330, seed=0)
    kw = dict(lambda_=1.0, alpha=0.95)
    Mb = compute_matrix(*to_dev(big_v, big_f), **kw)
    sb = PCGSolver(Mb)
    Ms = compute_matrix(*to_dev(small_v, small_f), **kw)
    ss = PCGSolver(Ms)
    db, dsm = sb.describe(), ss.describe()
    assert db["algo"] == "fused" and dsm["algo"] == "fused"
    (rs, cs, vals, Vs), ds_small = direct_for(small_v, small_f, kw)
    bs = np.random.default_rng(0).normal(size=(Vs, 3)).astype(np.float32)
    tvb = to_dev(big_v, big_f)[0]
    for _ in range(2):
        xb = sb.solve(to_differential(Mb, tvb))
        xs = ss.solve(t(bs))
        assert rel_l2(xb.cpu().numpy(), big_v) < BAR
        assert rel_l2(xs.cpu().numpy(), ds_small.solve(bs)) < BAR
    assert sb.describe() == db and ss.describe() == dsm      # neither fell back to another path


def test_deterministic_bitwise():
    v, f = workloads.plane(150, seed=0)
    M = compute_matrix(*to_dev(v, f), 1.0, alpha=0.95)
    b = torch.randn(M.shape[0], 3, device=DEV)
    s = PCGSolver(M)
    x1 = s.solve(b).clone()
    it1 = s.iterations
    x2 = s.solve(b)
    assert s.iterations == it1 and torch.equal(x1, x2)


def test_failure_modes():
    v, f = workloads.icosphere(2)
    M = compute_matrix(*to_dev(v, f), 10.0)
    V = M.shape[0]
    s = PCGSolver(M)
    bad = torch.randn(V, 3, device=DEV)
    bad[5, 1] = float("nan")
    with pytest.raises(N.Breakdown):
        s.solve(bad)
    # after a failure the handle is still usable
    ok = torch.randn(V, 3, device=DEV)
    assert torch.isfinite(s.solve(ok)).all()
    # iteration cap: warn by default, raise under strict
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        PCGSolver(M, maxit=3).solve(ok)
        assert any("maxit" in str(x.message) for x in w)
    with pytest.raises(N.NotConverged):
        PCGSolver(M, maxit=3, strict=True).solve(ok)
    # non-SPD: non-positive diagonal is rejected at create; indefinite with positive diagonal breaks down in CG
    idx, val = coo_np(M)
    neg = torch.sparse_coo_tensor(torch.from_numpy(idx).to(DEV), torch.from_numpy(-val).to(DEV), (V, V)).coalesce()
    with pytest.raises(N.Breakdown):
        PCGSolver(neg)
    ind = torch.sparse_coo_tensor(torch.tensor([[0, 0, 1, 1], [0, 1, 0, 1]], device=DEV),
                                  torch.tensor([1., 5., 5., 1.], device=DEV), (2, 2)).coalesce()
    with pytest.raises(N.Breakdown):
        PCGSolver(ind).solve(torch.tensor([[1., 0.], [0., 1.]], device=DEV))
    # argument errors keep the reference's exception types
    with pytest.raises(ValueError, match="expected shape"):
        s.solve(torch.zeros(V, device=DEV))
    with pytest.raises(TypeError):
        s.solve(torch.zeros(V, 3, device=DEV, dtype=torch.float64))
    with pytest.raises(ValueError):
        s.solve(torch.zeros(V + 1, 3, device=DEV))


def test_asynchronous_solve_and_lazy_status():
    """CholeskySolver (what from_differential uses by default) launches one kernel and returns without a host round
    trip, like cholespy; status and iteration count are fetched on demand."""
    v, f = workloads.icosphere(3)
    (r, c, val, V), ds = direct_for(v, f, dict(lambda_=10.0))
    M = compute_matrix(*to_dev(v, f), 10.0)
    s = CholeskySolver(M)
    assert s.check is False
    b = np.random.default_rng(0).normal(size=(V, 3)).astype(np.float32)
    x = s.solve(t(b))
    assert s.status in (0, 1) and 0 < s.iterations < 500
    s.raise_for_status()
    assert rel_l2(x.cpu().numpy(), ds.solve(b)) < BAR
    bad = t(b).clone()
    bad[3, 0] = float("nan")
    s.solve(bad)                    # no exception here (the reference has no failure path either) ...
    assert s.status == 3
    with pytest.raises(N.Breakdown):
        s.raise_for_status()        # ... the failure is reported on demand
    capped = PCGSolver(M, maxit=2, check=False)
    capped.solve(t(b))
    with pytest.raises(N.NotConverged):
        capped.raise_for_status()


def test_solver_cache_semantics():
    v, f = workloads.icosphere(2)
    M = compute_matrix(*to_dev(v, f), 10.0)
    u = torch.randn(M.shape[0], 3, device=DEV)
    gc.collect()
    n0 = len(parameterize._cache)
    from_differential(M, u)
    from_differential(M, u)
    from_differential(M, u, "CG")
    assert len(parameterize._cache) == n0 + 2
    key1, key2 = (id(M), "Cholesky"), (id(M), "CG")
    s1 = parameterize._cache[key1][0]
    assert isinstance(s1, CholeskySolver) and isinstance(parameterize._cache[key2][0], ConjugateGradientSolver)
    del M, s1
    gc.collect()
    # dropped when the matrix died (parameterize.py:7-17)
    assert key1 not in parameterize._cache and key2 not in parameterize._cache


def test_non_default_stream_and_noncontiguous_input():
    v, f = workloads.icosphere(3)
    (r, c, val, V), ds = direct_for(v, f, dict(lambda_=10.0))
    M = compute_matrix(*to_dev(v, f), 10.0)
    b = np.random.default_rng(0).normal(size=(V, 3)).astype(np.float32)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        bt = t(np.concatenate([b, b], 1))[:, :3]        # non-contiguous view
        x = from_differential(M, bt, "PCG")
    st.synchronize()
    assert rel_l2(x.cpu().numpy(), ds.solve(b)) < BAR


def test_full_size_roundtrip_adjoint_linearity():
    """BASELINE config 3 (plane 1000^2, V = 1e6, uniform, alpha = 0.95) through size-independent properties."""
    v, f = workloads.plane(1000, seed=0)
    tv, tf = to_dev(v, f)
    M = compute_matrix(tv, tf, 1.0, alpha=0.95)
    V = M.shape[0]
    s = PCGSolver(M)
    # round trip: from_differential(M, to_differential(M, v)) == v
    v2 = s.solve(to_differential(M, tv))
    assert rel_l2(v2.cpu().numpy(), v) < BAR
    assert s.iterations < 400 and max(s.relres[:3]) <= 5e-5
    # true residual of a random solve, measured with torch's own sparse matmul in fp64-ish
    b = torch.randn(V, 3, device=DEV)
    x = s.solve(b)
    res = (M @ x - b).norm(dim=0) / b.norm(dim=0)
    assert float(res.max()) < 5e-6
    # adjoint identity <g, M^-1 u> = <M^-1 g, u>  (M symmetric: backward solve == forward solve)
    g = torch.randn(V, 3, device=DEV)
    y = s.solve(g, backward=True)
    lhs = (g.double() * x.double()).sum().item()
    rhs_ = (y.double() * b.double()).sum().item()
    assert abs(lhs - rhs_) <= 1e-5 * max(abs(lhs), abs(rhs_), float(g.norm() * x.norm()))
    # linearity
    x2 = s.solve(2.0 * b + g)
    assert rel_l2(x2.cpu().numpy(), (2.0 * x + y).cpu().numpy()) < BAR


@pytest.fixture(scope="module")
def direct_1m():
    """fp64 SuperLU factorisation of BASELINE config 3's matrix (V = 1e6): ~25-60 s on one host core, done once."""
    v, f = workloads.plane(1000, seed=0)
    kw = dict(lambda_=1.0, alpha=0.95)
    (r, c, val, V), ds = direct_for(v, f, kw)
    return v, f, kw, (r, c, val, V), ds


def test_full_size_forward_backward_vs_direct(direct_1m):
    """BASELINE config 3 at full size against the oracle itself: forward and backward (O(1) and 1e-4 gradients)."""
    v, f, kw, (r, c, val, V), ds = direct_1m
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    u = t(b).requires_grad_(True)
    x = from_differential(M, u)
    e_fwd = rel_l2(x.detach().cpu().numpy(), ds.solve(b))
    errs = [e_fwd]
    for scale in (1.0, 1e-4):
        u.grad = None
        gg = (scale * g).astype(np.float32)
        x = from_differential(M, u)
        (x * t(gg)).sum().backward()
        errs.append(rel_l2(u.grad.cpu().numpy(), ds.solve(gg)))
    print("1M fwd / bwd / bwd 1e-4 rel-L2 vs fp64 direct:", ["%.2e" % e for e in errs])
    assert max(errs) < BAR, errs
    # the warm-started plug-in at full size
    w = ConjugateGradientSolver(M)
    w.solve(t(b))
    b2 = (b + 1e-3 * np.random.default_rng(7).normal(size=b.shape)).astype(np.float32)
    assert rel_l2(w.solve(t(b2)).cpu().numpy(), ds.solve(b2)) < BAR


def test_config4_quarter_million_uniform_vs_direct():
    """BASELINE config 4's mesh (plane 500^2, uniform, alpha = 0.95) against the fp64 direct solve, forward and backward."""
    v, f = workloads.plane(500, seed=5)
    kw = dict(lambda_=1.0, alpha=0.95)
    (r, c, val, V), ds = direct_for(v, f, kw)
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    u = t(b).requires_grad_(True)
    x = from_differential(M, u)
    (x * t(g)).sum().backward()
    assert rel_l2(x.detach().cpu().numpy(), ds.solve(b)) < BAR
    assert rel_l2(u.grad.cpu().numpy(), ds.solve(g)) < BAR


def test_four_million_vertices_roundtrip():
    """Largest size exercised: plane 2000^2 (V = 4e6, nnz = 27,984,002).  The CTAs' rows no longer fit in shared memory, so
    the fused kernel keeps every vector in global memory (RES = 0); round trip + true residual."""
    v, f = workloads.plane(2000, seed=0)
    tv, tf = to_dev(v, f)
    M = compute_matrix(tv, tf, 1.0, alpha=0.95)
    assert M._nnz() == 7 * 2000 * 2000 - 8 * 2000 + 2
    s = PCGSolver(M)
    assert s.describe()["residency"] == 0
    x = s.solve(to_differential(M, tv))
    assert rel_l2(x.cpu().numpy(), v) < BAR
    b = torch.randn(M.shape[0], 3, device=DEV)
    y = s.solve(b)
    res = (M @ y - b).norm(dim=0) / b.norm(dim=0)
    assert float(res.max()) < 5e-6


def test_config4_batch_of_meshes_one_rank():
    """BASELINE config 4 (8 independent 250K-vertex meshes) on however many GPUs there are: mesh i -> rank i mod N
    (distributed.assign); with one rank the same code walks all eight.  Round-trip property per mesh."""
    from largesteps_b200 import distributed as D
    mine = D.assign(8, D.rank(), D.world())
    assert len(mine) == 8 // D.world()
    for i in mine:
        v, f = workloads.plane(500, seed=i)
        tv, tf = to_dev(v, f)
        M = compute_matrix(tv, tf, 1.0, alpha=0.95)
        assert M._nnz() == 1746002
        x = from_differential(M, to_differential(M, tv))
        assert rel_l2(x.cpu().numpy(), v) < BAR
        del M


def test_quarter_million_cotangent_vs_direct():
    """250K vertices, cotangent Laplacian, lambda = 19 against the fp64 direct solve (the largest size the CPU
    factorisation finishes in seconds)."""
    v, f = workloads.plane(500, seed=3)
    kw = dict(lambda_=19.0, cotan=True)
    (r, c, val, V), ds = direct_for(v, f, kw)
    _, b, g = rhs(r, c, val, V, v)
    M = compute_matrix(*to_dev(v, f), **kw)
    u = t(b).requires_grad_(True)
    x = from_differential(M, u)
    (x * t(g)).sum().backward()
    assert rel_l2(x.detach().cpu().numpy(), ds.solve(b)) < BAR
    assert rel_l2(u.grad.cpu().numpy(), ds.solve(g)) < BAR


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_independent_meshes():
    """Config 4 in miniature: one mesh per GPU, solved independently (no collective on the solve path)."""
    outs = []
    for d in range(2):
        dev = f"cuda:{d}"
        v, f = workloads.plane(120, seed=d)
        tv = torch.from_numpy(v).to(dev)
        tf = torch.from_numpy(f).to(dev)
        M = compute_matrix(tv, tf, 1.0, alpha=0.95)
        outs.append((from_differential(M, to_differential(M, tv)), v))
    for x, v in outs:
        assert rel_l2(x.cpu().numpy(), v) < BAR
