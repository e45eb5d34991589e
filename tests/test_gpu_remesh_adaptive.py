"""GPU: remesh_botsch with a per-vertex target edge length and feature vertices -- each stage against the numpy model fed the
device's own input, attributes included; the whole call's invariants, reproducibility, the scalar call's bits for a constant
target, pinned features and the graded field's edge lengths; a graded level-8 icosphere; and the _v entry points with null
attributes against the scalar entry points."""
import ctypes

import numpy as np
import pytest
import torch

import largesteps_b200._native as N
import remesh_adaptive_model as AM
import remesh_model as RM
from largesteps_b200 import workloads
from largesteps_b200.distance import MeshDistance
from largesteps_b200.remesh import _Remesher, remesh_botsch
from gpu_util import DEV
from test_gpu_remesh_botsch import assert_ulp, device_invariants, mean_edge, mesh
from test_remesh_adaptive_model import features, graded_target
from test_remesh_model import assert_normals_kept, noisy

pytestmark = pytest.mark.gpu


def host(r):
    v, f = r.mesh()
    return (v.cpu().numpy(), f.cpu().numpy().astype(np.int64), r.high[:r.V].cpu().numpy(), r.low[:r.V].cpu().numpy(),
            r.feat[:r.V].cpu().numpy().astype(bool))


def assert_same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and np.array_equal(g, w)


@pytest.mark.parametrize("scale", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("case", ["octahedron", "ico_out", "ico_in", "components", "ico3", "ico4", "bunny"])
def test_stages_match_the_model(case, scale, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    t = graded_target(v, scale * mean_edge(v, f))
    feat = features(v, f)
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    r = _Remesher(tv, tf, torch.from_numpy(t).to(DEV), torch.from_numpy(feat).to(DEV))
    r.check()
    hv, hf, hh, hl, hm = host(r)
    r.compact()
    mv, mf, (mh, ml, mm) = AM.compact(hv, hf, hh, hl, hm)
    assert_same(host(r), (mv, mf, mh, ml, mm))
    target = MeshDistance(*r.mesh())
    V0, F0 = host(r)[:2]
    iters = 2 if len(v) < 1000 else 1
    for _ in range(iters):
        hv, hf, hh, hl, hm = host(r)
        n = r.split(0.0)
        mv, mf, mn, (mh, ml, mm) = AM.split(hv, hf, hh, hl, hm)
        assert n == mn
        assert_same(host(r), (mv, mf, mh, ml, mm))
        live = r.V
        while True:
            hv, hf, hh, hl, hm = host(r)
            n = r.collapse_round(0.0, 0.0, live)
            mv, mf, mn = AM.collapse_round(hv, hf, live, hh, hl, hm)
            assert n == mn
            got = host(r)
            assert_same(got, (mv, mf, hh, hl, hm))                     # the survivor keeps its own bounds
            assert_normals_kept(hv, hf, got[0], got[1])
            live -= n
            if n == 0:
                break
        hv, hf, hh, hl, hm = host(r)
        r.compact()
        mv, mf, (mh, ml, mm) = AM.compact(hv, hf, hh, hl, hm)
        assert_same(host(r), (mv, mf, mh, ml, mm))
        while True:
            hv, hf, hh, hl, hm = host(r)
            n = r.flip_round()
            mf, mn = AM.flip_round(hv, hf, hm)
            assert n == mn
            assert_same(host(r), (hv, mf, hh, hl, hm))
            if n == 0:
                break
        hv, hf, hh, hl, hm = host(r)
        r.relax(target)
        got = host(r)
        assert_ulp(got[0], AM.relax(hv, hf, V0, F0, hm), 2)
        assert np.array_equal(got[0][hm], hv[hm])                       # feature rows bit for bit
        assert_same(got[1:], (hf, hh, hl, hm))
    RM.assert_invariants(*host(r)[:2], RM.euler(v, f))


def graded_share(vo, fo, v, h0):
    """The share of edges within [0.7, 1.4] x the graded field of graded_target(v, h0) at their midpoint."""
    x = np.asarray(v, np.float64)[:, 0]
    lo, hi = x.min(), x.max()
    a, b = vo[fo].astype(np.float64), vo[fo[:, [1, 2, 0]]].astype(np.float64)
    length = np.linalg.norm(a - b, axis=2)
    t = h0 * (0.5 + 1.5 * (0.5 * (a[..., 0] + b[..., 0]) - lo) / (hi - lo))
    return float(((length >= 0.7 * t) & (length <= 1.4 * t)).mean())


@pytest.mark.parametrize("project", [True, False])
@pytest.mark.parametrize("case", ["ico3", "components", "bunny"])
def test_end_to_end(case, project, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    h0 = mean_edge(v, f)
    t = graded_target(v, h0)
    feat = features(v, f)
    tv, tt = torch.from_numpy(v).to(DEV), torch.from_numpy(t).to(DEV)
    idx = np.random.default_rng(5).permutation(np.r_[np.flatnonzero(feat), np.flatnonzero(feat)[:3]])   # any order, repeats
    spellings = [(torch.int64, tt, torch.from_numpy(idx).to(DEV)),
                 (torch.int32, tt, torch.from_numpy(feat).to(DEV)),
                 (torch.int64, tt, torch.from_numpy(idx).to(DEV).int())]
    outs = [remesh_botsch(tv, torch.from_numpy(f).to(DEV).to(dt), 5, h, project, feature=ft, return_feature=True)
            for dt, h, ft in spellings]
    vo, fo, fto = outs[0]
    assert vo.dtype == torch.float32 and fo.dtype == torch.int64 and outs[1][1].dtype == torch.int32 and fto.dtype == torch.int64
    for w, g, k in outs[1:]:
        assert torch.equal(w, vo) and torch.equal(g.long(), fo) and torch.equal(k, fto)
    hv, hf, hk = vo.cpu().numpy(), fo.cpu().numpy(), fto.cpu().numpy()
    RM.assert_invariants(hv, hf, RM.euler(v, f))
    assert np.bincount(hf.ravel()).min() >= 3
    assert (np.diff(hk) > 0).all() and len(hk) == int(feat.sum())        # ascending; every referenced feature survives
    assert np.array_equal(hv[hk], v[feat])                              # where it was, bit for bit
    if project:
        sq, _, _ = MeshDistance(tv, torch.from_numpy(f).to(DEV)).squared_distance(vo)
        diag = float(np.linalg.norm(v.max(0) - v.min(0)))
        assert float(sq.max()) <= (1e-6 * diag) ** 2
    # a constant float64 target is the scalar call, bit for bit
    tf = torch.from_numpy(f).to(DEV)
    sv, sf = remesh_botsch(tv, tf, 5, h0, project)
    cv, cf, ck = remesh_botsch(tv, tf, 5, torch.full((len(v),), h0, dtype=torch.float64, device=DEV), project, return_feature=True)
    assert torch.equal(cv, sv) and torch.equal(cf, sf) and ck.numel() == 0
    # the graded call follows the field better than the uniform call at the field's mean, with the same features
    uv, uf = remesh_botsch(tv, tf, 5, float(t.mean()), project, feature=torch.from_numpy(feat).to(DEV))
    graded, uniform = graded_share(hv, hf, v, h0), graded_share(uv.cpu().numpy(), uf.cpu().numpy(), v, h0)
    print(f"\n{case} project={project}: {len(hv)} vertices, {len(hk)} features; edges within [0.7, 1.4] x the graded field: "
          f"graded {graded:.3f}, uniform at its mean {uniform:.3f}")
    assert graded > uniform


def test_float32_targets_are_widened_before_the_bounds():
    v, f = mesh("ico3", None)
    t = graded_target(v, mean_edge(v, f)).astype(np.float32)
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    a = remesh_botsch(tv, tf, 2, torch.from_numpy(t).to(DEV), True)
    b = remesh_botsch(tv, tf, 2, torch.from_numpy(t.astype(np.float64)).to(DEV), True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_icosphere_level_8_graded_with_features():
    v, f = workloads.icosphere(8)
    v, f, mean = noisy(np.asarray(v, np.float32), np.asarray(f, np.int64), 0.1)
    t = graded_target(v, 0.5 * mean)
    feat = np.zeros(len(v), bool)
    feat[np.random.default_rng(8).choice(len(v), len(v) // 100, replace=False)] = True
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    vo, fo, fto = remesh_botsch(tv, tf, 5, torch.from_numpy(t).to(DEV), True, feature=torch.from_numpy(feat).to(DEV),
                                return_feature=True)
    print(f"\nicosphere 8, graded: {v.shape[0]} -> {vo.shape[0]} vertices, {fto.numel()} features")
    device_invariants(vo, fo, 2)
    assert fto.numel() == int(feat.sum())
    assert torch.equal(vo[fto], tv[torch.from_numpy(np.flatnonzero(feat)).to(DEV)])


# ---- the _v entry points with null attributes are the scalar entry points ----------------------------------------------------
def old_split(r, high):
    r.ensure(r.V + 3 * r.F // 2, 4 * r.F)
    n = ctypes.c_int64(0)
    N.check(N.lib().ls_remesh_split(*r.args(), r.V, r.F, r.verts.shape[0], r.faces.shape[0], high, N.ptr(r.ws), r.ws.numel(),
                                    ctypes.byref(n), N.stream_ptr(r.dev)), "ls_remesh_split")
    r.V += n.value
    r.F += 2 * n.value
    return n.value


def old_collapse_round(r, low, high, live):
    n = ctypes.c_int64(0)
    N.check(N.lib().ls_remesh_collapse_round(*r.args(), r.V, r.F, live, low, high, N.ptr(r.ws), r.ws.numel(), ctypes.byref(n),
                                             N.stream_ptr(r.dev)), "ls_remesh_collapse_round")
    return n.value


def old_compact(r):
    nv, nf = ctypes.c_int64(0), ctypes.c_int64(0)
    N.check(N.lib().ls_remesh_compact(*r.args(), r.V, r.F, N.ptr(r.ws), r.ws.numel(), ctypes.byref(nv), ctypes.byref(nf),
                                      N.stream_ptr(r.dev)), "ls_remesh_compact")
    r.V, r.F = nv.value, nf.value


def old_flip_round(r):
    n = ctypes.c_int64(0)
    N.check(N.lib().ls_remesh_flip_round(*r.args(), r.V, r.F, N.ptr(r.ws), r.ws.numel(), ctypes.byref(n), N.stream_ptr(r.dev)),
            "ls_remesh_flip_round")
    return n.value


def old_relax(r, target):
    N.check(N.lib().ls_remesh_relax(*r.args(), r.V, r.F, N.ptr(target._bvh), target.F, N.ptr(r.ws), r.ws.numel(),
                                    N.stream_ptr(r.dev)), "ls_remesh_relax")


@pytest.mark.parametrize("case", ["components", "bunny"])
def test_v_entry_points_with_null_attributes_equal_the_scalar_ones(case, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    h = 0.5 * mean_edge(v, f)
    high, low = 1.4 * h, 0.7 * h
    tv, tf = torch.from_numpy(v).to(DEV), torch.from_numpy(f).to(DEV)
    new, old = _Remesher(tv, tf), _Remesher(tv, tf)
    assert new.high is None                                             # the methods pass null attributes

    def same():
        return new.V == old.V and new.F == old.F and all(torch.equal(a, b) for a, b in zip(new.mesh(), old.mesh()))

    new.compact()
    old_compact(old)
    assert same()
    target = MeshDistance(*new.mesh())
    for _ in range(2):
        assert new.split(high) == old_split(old, high) and same()
        live = new.V
        while True:
            n = new.collapse_round(low, high, live)
            assert n == old_collapse_round(old, low, high, live) and same()
            live -= n
            if n == 0:
                break
        new.compact()
        old_compact(old)
        assert same()
        while True:
            n = new.flip_round()
            assert n == old_flip_round(old) and same()
            if n == 0:
                break
        new.relax(target)
        old_relax(old, target)
        assert same()
