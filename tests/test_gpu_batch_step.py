"""GPU: the batched optimisation step -- the multi-tensor AdamUniform (ls_adam_uniform_step_multi) against per-parameter
ls_adam_uniform_step calls, per-mesh vertex normals on packed meshes (compute_vertex_normals_batch) against
compute_vertex_normals on each mesh, and a whole batched loop against the per-mesh loop."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from largesteps_b200 import meshops, workloads, _native as N
from largesteps_b200.batch import from_differential_batch, pack_meshes
from largesteps_b200.geometry import compute_matrix
from largesteps_b200.optimize import AdamUniform
from largesteps_b200.parameterize import from_differential, to_differential
from gpu_util import DEV, to_dev, rel_l2, fan_mesh

pytestmark = pytest.mark.gpu


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


# ---- AdamUniform ----------------------------------------------------------------------------------------------------------
class RefAdam:
    """The per-parameter path: one ls_adam_uniform_step call per parameter on cloned state."""

    def __init__(self, params, lr, betas):
        self.p = [p.detach().clone() for p in params]
        self.g1 = [torch.zeros_like(p) for p in self.p]
        self.g2 = [torch.zeros_like(p) for p in self.p]
        self.lr, self.betas, self.steps = lr, betas, [0] * len(self.p)
        self.scratch = torch.zeros(4, dtype=torch.int32, device=DEV)

    def step(self, grads):
        b1, b2 = self.betas
        for i, (p, g) in enumerate(zip(self.p, grads)):
            self.steps[i] += 1
            s = self.steps[i]
            g = g.contiguous()
            N.check(N.lib().ls_adam_uniform_step(N.ptr(p), N.ptr(g), N.ptr(self.g1[i]), N.ptr(self.g2[i]), p.numel(),
                                                  float(self.lr), float(b1), float(b2), float(1 - b1), float(1 - b2),
                                                  float(1 - b1 ** s), float(1 - b2 ** s), N.ptr(self.scratch),
                                                  N.stream_ptr(DEV)), "ls_adam_uniform_step")


SIZES = [(0,), (1,), (17,), (5000, 3), (100003, 3)]


def make_params(n, seed, sizes=SIZES):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return [torch.randn(sizes[i % len(sizes)], generator=g).to(DEV).requires_grad_(True) for i in range(n)]


def grads_for(params, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    return [torch.randn(p.shape, generator=g).to(DEV) for p in params]


def same(a, b):
    return torch.equal(a, b)


def test_adam_multi_is_bitwise_the_per_parameter_step():
    params = make_params(70, 0)
    late = make_params(1, 99, [(5000, 3)])[0]
    g1, g2 = params[:40], params[40:]
    opt = AdamUniform([dict(params=g1), dict(params=g2, lr=0.03, betas=(0.8, 0.99))], lr=0.1)
    ref1, ref2 = RefAdam(g1, 0.1, (0.9, 0.999)), RefAdam(g2, 0.03, (0.8, 0.99))
    ref3 = None
    for it in range(5):
        if it == 2:      # a parameter added after two steps: its step count runs behind the others
            opt.add_param_group(dict(params=[late], lr=0.2, betas=(0.7, 0.9)))
            ref3 = RefAdam([late], 0.2, (0.7, 0.9))
        ps = params + ([late] if ref3 else [])
        gs = grads_for(ps, 10 + it)
        gs[3] = torch.randn(3, 5000, device=DEV).t()        # a non-contiguous gradient of a (5000, 3) parameter
        for p, g in zip(ps, gs):
            p.grad = g
        opt.step()
        ref1.step(gs[:40])
        ref2.step(gs[40:70])
        if ref3:
            ref3.step(gs[70:])
        for ref, group in ((ref1, g1), (ref2, g2), (ref3, [late] if ref3 else [])):
            for i, p in enumerate(group):
                st = opt.state[p]
                assert same(p.detach(), ref.p[i]) and same(st["g1"], ref.g1[i]) and same(st["g2"], ref.g2[i]), (it, i)
                assert st["step"] == ref.steps[i]


def test_a_nan_poisons_only_its_own_parameter():
    a, b = make_params(8, 1), make_params(8, 1)
    oa, ob = AdamUniform(a, lr=0.05), AdamUniform(b, lr=0.05)
    for it in range(3):
        gs = grads_for(a, 20 + it)
        for p, g in zip(a, gs):
            p.grad = g.clone()
        if it == 1:
            gs[4] = gs[4].clone()
            gs[4].view(-1)[7] = float("nan")
        for p, g in zip(b, gs):
            p.grad = g
        oa.step()
        ob.step()
    assert torch.isnan(b[4]).all()
    for i in range(8):
        if i != 4:
            assert same(a[i].detach(), b[i].detach()), i


@pytest.mark.parametrize("n", [1, 8, 64])
def test_launches_per_step_do_not_depend_on_the_parameter_count(n):
    ps = make_params(n, 2, [(300, 3), (17,)])
    opt = AdamUniform(ps, lr=0.1)
    for p, g in zip(ps, grads_for(ps, 3)):
        p.grad = g
    opt.step()
    n0 = N.launch_count()
    opt.step()
    assert N.launch_count() - n0 == 2


def test_more_tensors_than_one_table():
    ps = make_params(600, 4, [(1,), (3,), (17, 3)])
    opt = AdamUniform(ps, lr=0.1)
    ref = RefAdam(ps, 0.1, (0.9, 0.999))
    for it in range(3):
        gs = grads_for(ps, 30 + it)
        for p, g in zip(ps, gs):
            p.grad = g
        n0 = N.launch_count()
        opt.step()
        assert N.launch_count() - n0 == 2 * 3          # 600 tensors: three tables of at most 256
        ref.step(gs)
    assert all(same(p.detach(), r) for p, r in zip(ps, ref.p))


@pytest.mark.parametrize("bad", ["no_grad", "cpu", "float64"])
def test_an_invalid_parameter_changes_nothing(bad):
    ps = make_params(5, 5)
    opt = AdamUniform(ps, lr=0.1)
    for p, g in zip(ps, grads_for(ps, 6)):
        p.grad = g
    opt.step()
    extra = {"no_grad": torch.zeros(4, device=DEV, requires_grad=True),
             "cpu": torch.zeros(4, requires_grad=True),
             "float64": torch.zeros(4, device=DEV, dtype=torch.float64, requires_grad=True)}[bad]
    if bad != "no_grad":
        extra.grad = torch.ones_like(extra)
    opt.add_param_group(dict(params=[extra]))
    for p, g in zip(ps, grads_for(ps, 7)):
        p.grad = g
    before = [(p.detach().clone(), opt.state[p]["g1"].clone(), opt.state[p]["g2"].clone(), opt.state[p]["step"]) for p in ps]
    with pytest.raises(TypeError if bad == "float64" else RuntimeError):
        opt.step()
    torch.cuda.synchronize()
    for p, (x, m1, m2, s) in zip(ps, before):
        st = opt.state[p]
        assert same(p.detach(), x) and same(st["g1"], m1) and same(st["g2"], m2) and st["step"] == s
    assert len(opt.state[extra]) == 0


def test_a_state_dict_of_the_per_parameter_optimiser_continues_bitwise():
    ps = make_params(6, 8)
    ref = RefAdam(ps, 0.1, (0.9, 0.999))
    for it in range(2):
        ref.step(grads_for(ps, 40 + it))
    # the layout the per-parameter optimiser saved: step, g1, g2 and its 16-byte scratch per parameter
    sd = {"state": {i: {"step": ref.steps[i], "g1": ref.g1[i].clone(), "g2": ref.g2[i].clone(),
                        "scratch": torch.zeros(4, dtype=torch.int32, device=DEV)} for i in range(len(ps))},
          "param_groups": [dict(lr=0.1, betas=(0.9, 0.999), params=list(range(len(ps))))]}
    fresh = [r.clone().requires_grad_(True) for r in ref.p]
    opt = AdamUniform(fresh, lr=0.1)
    opt.load_state_dict(sd)
    for it in range(3):
        gs = grads_for(ps, 50 + it)
        for p, g in zip(fresh, gs):
            p.grad = g
        opt.step()
        ref.step(gs)
    for i, p in enumerate(fresh):
        assert same(p.detach(), ref.p[i]) and same(opt.state[p]["g1"], ref.g1[i]) and opt.state[p]["step"] == 5


# ---- vertex normals on packed meshes -------------------------------------------------------------------------------------------
def mesh_set(bunny_mesh):
    bv, bf = bunny_mesh
    mass = np.load(os.path.join(GOLDEN, "mass.npz"))
    pv, pf = workloads.plane(60, seed=3)
    pv = pv + np.random.default_rng(3).normal(0, 0.002, size=pv.shape).astype(np.float32)
    iv, if_ = workloads.icosphere(2)
    big = workloads.plane(300, seed=9)          # more faces than 528 blocks of 256: the block cap of the reduction
    return {
        "ico1": workloads.icosphere(1), "ico2": workloads.icosphere(2), "ico3": workloads.icosphere(3),
        "ico4": workloads.icosphere(4), "bunny": (bv.astype(np.float32), bf), "plane60": (pv, pf),
        "fan1000": fan_mesh(1000), "isolated": (np.concatenate([iv, [[2.0, 0.0, 0.0]]]).astype(np.float32), if_),
        "degen": (mass["degen.verts"], mass["degen.faces"]), "grid": (mass["grid.verts"], mass["grid.faces"]),
        "mass_plane": (mass["plane.verts"], mass["plane.faces"]), "plane300": big,
    }


def nan_equal(a, b):
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(a[~na], b[~nb])


def single(v, f, gout):
    x = v.clone().requires_grad_(True)
    fn = meshops.compute_face_normals(x, f).detach().requires_grad_(True)
    n = meshops.compute_vertex_normals(x, f, fn)
    n.backward(gout)
    return n.detach(), x.grad, fn.grad, fn.detach()


@pytest.fixture(scope="module", params=[torch.int32, torch.int64], ids=["int32", "int64"])
def normals_case(request, bunny_mesh):
    ms = mesh_set(bunny_mesh)
    names = list(ms)
    data, want = [], []
    for i, nm in enumerate(names):
        v, f = to_dev(*ms[nm], idx_dtype=request.param)
        gout = t(np.random.default_rng(100 + i).normal(size=(v.shape[0], 3)).astype(np.float32))
        data.append((v, f, gout))
        want.append(single(v, f, gout))
    return names, data, want


def run_batch(data, idx):
    p = pack_meshes([data[i][0] for i in idx], [data[i][1] for i in idx])
    x = p.verts.clone().requires_grad_(True)
    fn = meshops.compute_face_normals(x, p.faces).detach().requires_grad_(True)
    n = meshops.compute_vertex_normals_batch(x, p.faces, fn, p.vert_offsets, p.face_offsets)
    n.backward(torch.cat([data[i][2] for i in idx]))
    vo, fo = p.vert_offsets_host, p.face_offsets_host
    return [(n[vo[k]:vo[k + 1]].detach(), x.grad[vo[k]:vo[k + 1]], fn.grad[:, fo[k]:fo[k + 1]], fn[:, fo[k]:fo[k + 1]].detach())
            for k in range(len(idx))]


@pytest.mark.parametrize("order", ["all", "reversed", "dropped", "single"])
def test_vertex_normals_batch_is_bitwise_the_per_mesh_op(normals_case, order):
    names, data, want = normals_case
    n = len(names)
    idx = {"all": list(range(n)), "reversed": list(range(n))[::-1], "dropped": [i for i in range(n) if i != 4],
           "single": [names.index("bunny")]}[order]
    got = run_batch(data, idx)
    for k, i in enumerate(idx):
        for what, a, b in zip(("normals", "grad verts", "grad face normals", "face normals"), got[k], want[i]):
            assert nan_equal(a, b), (names[i], what)
    assert torch.isnan(want[names.index("degen")][0]).any()      # the degenerate mesh does exercise the NaN paths


def test_face_normals_and_gathers_on_the_packed_mesh(normals_case):
    """The per-face and per-vertex ops need no batch variant: on a packed mesh they give every mesh its own result."""
    names, data, _ = normals_case
    p = pack_meshes([d[0] for d in data], [d[1] for d in data])
    x = p.verts.clone().requires_grad_(True)
    fn = meshops.compute_face_normals(x, p.faces)
    gf = torch.randn_like(fn)
    fn.backward(gf)
    idx = torch.cat([torch.arange(v.shape[0] - 1, -1, -1, device=DEV) + p.vert_offsets_host[k] for k, (v, _, _) in enumerate(data)])
    y = p.verts.clone().requires_grad_(True)
    rows = meshops.gather_rows(y, idx)
    gr = torch.randn_like(rows)
    rows.backward(gr)
    vo, fo = p.vert_offsets_host, p.face_offsets_host
    for k, (v, f, _) in enumerate(data):
        xs = v.clone().requires_grad_(True)
        fs = meshops.compute_face_normals(xs, f)
        fs.backward(gf[:, fo[k]:fo[k + 1]])
        assert nan_equal(fn[:, fo[k]:fo[k + 1]].detach(), fs.detach()) and nan_equal(x.grad[vo[k]:vo[k + 1]], xs.grad), names[k]
        ys = v.clone().requires_grad_(True)
        rs = meshops.gather_rows(ys, idx[vo[k]:vo[k + 1]] - vo[k])
        rs.backward(gr[vo[k]:vo[k + 1]])
        assert torch.equal(rows[vo[k]:vo[k + 1]].detach(), rs.detach()) and torch.equal(y.grad[vo[k]:vo[k + 1]], ys.grad)


def test_vertex_normals_batch_launches(normals_case):
    _, data, _ = normals_case
    counts = []
    for idx in ([0, 1], list(range(len(data)))):
        p = pack_meshes([data[i][0] for i in idx], [data[i][1] for i in idx])
        x = p.verts.clone().requires_grad_(True)
        fn = meshops.compute_face_normals(x, p.faces).detach().requires_grad_(True)
        for rep in range(2):            # the first call builds the incidence list and checks the faces' mesh ranges
            n0 = N.launch_count()
            meshops.compute_vertex_normals_batch(x, p.faces, fn, p.vert_offsets, p.face_offsets).sum().backward()
            counts.append(N.launch_count() - n0)
    assert counts[1] == counts[3] == 4, counts     # two kernels per direction, whatever B is


def test_vertex_normals_batch_rejections():
    (v1, f1), (v2, f2) = to_dev(*workloads.icosphere(1)), to_dev(*workloads.icosphere(2))
    p = pack_meshes([v1, v2], [f1, f2])
    fn = meshops.compute_face_normals(p.verts, p.faces)
    meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, p.vert_offsets, p.face_offsets)
    bad = p.faces.clone()
    bad[p.face_offsets_host[1] + 5, 0] = 3           # a face of mesh 1 pointing into mesh 0
    with pytest.raises(IndexError, match="mesh 1"):
        meshops.compute_vertex_normals_batch(p.verts, bad, fn, p.vert_offsets, p.face_offsets)
    bad0 = p.faces.clone()
    bad0[0, 1] = p.vert_offsets_host[1]              # a face of mesh 0 pointing into mesh 1
    with pytest.raises(IndexError, match="mesh 0"):
        meshops.compute_vertex_normals_batch(p.verts, bad0, fn, p.vert_offsets, p.face_offsets)
    V, F = p.verts.shape[0], p.faces.shape[0]
    with pytest.raises(ValueError, match="non-decreasing"):
        meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, [0, 50, 20, V], [0, 10, 20, F])
    with pytest.raises(ValueError, match="end at"):
        meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, [0, 42, V - 1], list(p.face_offsets_host))
    with pytest.raises(ValueError, match="end at"):
        meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, list(p.vert_offsets_host), [0, 80, F + 1])
    with pytest.raises(RuntimeError, match="CUDA"):
        meshops.compute_vertex_normals_batch(p.verts.cpu(), p.faces, fn, p.vert_offsets, p.face_offsets)
    with pytest.raises(RuntimeError, match="CUDA"):
        meshops.compute_vertex_normals_batch(p.verts, p.faces, fn.cpu(), p.vert_offsets, p.face_offsets)
    # offsets as Python ints give the same result as the device tensors
    a = meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, p.vert_offsets, p.face_offsets)
    b = meshops.compute_vertex_normals_batch(p.verts, p.faces, fn, list(p.vert_offsets_host), list(p.face_offsets_host))
    assert torch.equal(a, b)


# ---- the whole step -------------------------------------------------------------------------------------------------------
def loop_meshes(n, levels):
    out = []
    for i in range(n):
        v, f = workloads.icosphere(levels[i % len(levels)])
        v = v + np.random.default_rng(i).normal(0, 0.01, size=v.shape).astype(np.float32)
        tv, tf = to_dev(v, f)
        M = compute_matrix(tv, tf, lambda_=float(5 + 2 * i), cotan=bool(i % 2))
        out.append((tv, tf, M))
    return out


def test_batched_loop_is_bitwise_the_per_mesh_loop():
    ms = loop_meshes(8, [2, 3, 2, 2, 3, 2, 2, 4])       # mesh 7 (icosphere 4, 81 slices) solves on a larger cluster
    targets = [t(v.cpu().numpy() * 1.1) for v, _, _ in ms]
    ntargets = [torch.nn.functional.normalize(tg, dim=1) for tg in targets]
    us_b = [to_differential(M, v).clone().requires_grad_(True) for v, _, M in ms]
    us_s = [u.detach().clone().requires_grad_(True) for u in us_b]
    Ms = [M for _, _, M in ms]
    p = pack_meshes([v for v, _, _ in ms], [f for _, f, _ in ms])
    tg_p, nt_p = torch.cat(targets), torch.cat(ntargets)
    ob, os_ = AdamUniform(us_b, lr=0.01), AdamUniform(us_s, lr=0.01)
    for _ in range(50):
        ob.zero_grad()
        x = from_differential_batch(Ms, us_b, packed=True)
        fn = meshops.compute_face_normals(x, p.faces)
        n = meshops.compute_vertex_normals_batch(x, p.faces, fn, p.vert_offsets, p.face_offsets)
        (((x - tg_p) ** 2).sum() + ((n - nt_p) ** 2).sum()).backward()
        ob.step()
        os_.zero_grad()
        loss = 0
        for (_, f, M), u, tg, nt in zip(ms, us_s, targets, ntargets):
            xs = from_differential(M, u)
            ns = meshops.compute_vertex_normals(xs, f, meshops.compute_face_normals(xs, f))
            loss = loss + ((xs - tg) ** 2).sum() + ((ns - nt) ** 2).sum()
        loss.backward()
        os_.step()
    for i, (v, _, M) in enumerate(ms):
        if (v.shape[0] + 31) // 32 <= 24:
            assert torch.equal(us_b[i].detach(), us_s[i].detach()), i
        else:
            assert rel_l2(us_b[i].detach().cpu().numpy(), us_s[i].detach().cpu().numpy()) < 1e-5, i


def batched_step(Ms, us, p, opt):
    opt.zero_grad()
    x = from_differential_batch(Ms, us, packed=True)
    fn = meshops.compute_face_normals(x, p.faces)
    n = meshops.compute_vertex_normals_batch(x, p.faces, fn, p.vert_offsets, p.face_offsets)
    ((x ** 2).sum() + n.sum()).backward()
    opt.step()


def test_launches_per_batched_step_do_not_depend_on_the_batch_size():
    counts = []
    for B in (8, 32):
        ms = loop_meshes(B, [2])
        Ms = [M for _, _, M in ms]
        us = [to_differential(M, v).clone().requires_grad_(True) for v, _, M in ms]
        p = pack_meshes([v for v, _, _ in ms], [f for _, f, _ in ms])
        opt = AdamUniform(us, lr=0.01)
        batched_step(Ms, us, p, opt)
        n0 = N.launch_count()
        batched_step(Ms, us, p, opt)
        counts.append(N.launch_count() - n0)
    assert counts[0] == counts[1], counts


def test_packed_solution_and_packed_right_hand_sides():
    ms = loop_meshes(4, [2, 3])
    Ms = [M for _, _, M in ms]
    us = [to_differential(M, v).clone().requires_grad_(True) for v, _, M in ms]
    xs = from_differential_batch(Ms, us)
    xp = from_differential_batch(Ms, us, packed=True)
    assert xp.shape == (sum(u.shape[0] for u in us), 3)
    assert torch.equal(xp, torch.cat(xs))
    up = torch.cat([u.detach() for u in us]).requires_grad_(True)
    xq = from_differential_batch(Ms, up, packed=True)
    assert torch.equal(xq, xp)
    g = torch.randn_like(xp)
    (xp * g).sum().backward()
    (xq * g).sum().backward()
    assert torch.equal(up.grad, torch.cat([u.grad for u in us]))
    assert all(torch.equal(a, b) for a, b in zip(from_differential_batch(Ms, up.detach()), xs))
    with pytest.raises(ValueError, match="rows"):
        from_differential_batch(Ms, up[:-1])
