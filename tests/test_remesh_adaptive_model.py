"""CPU: the adaptive remesher's numpy model (per-vertex target lengths and feature vertices, tests/remesh_adaptive_model.py) and
remesh_botsch's new arguments.  A constant target with no feature is the scalar model bit for bit; a feature vertex is never
in a split, a collapse or a flip and never moves; a graded target keeps the invariants.  The _v entry points reject a partial
attribute set and NULL counts."""
import ctypes

import numpy as np
import pytest
import torch

import largesteps_b200._native as N
import remesh_adaptive_model as AM
import remesh_model as RM
from largesteps_b200.remesh import remesh_botsch
from test_gpu_remesh_botsch import mean_edge, mesh

CASES = ["octahedron", "ico_out", "ico_in", "components", "ico3", "ico4", "bunny"]


def graded_target(v, h0):
    """t_i = h0 (0.5 + 1.5 s_i), s_i the vertex's normalised x coordinate: a 4x ratio across the mesh."""
    x = np.asarray(v, np.float64)[:, 0]
    s = (x - x.min()) / (x.max() - x.min())
    return h0 * (0.5 + 1.5 * s)


def features(v, f, seed=0, share=0.02):
    """A seeded `share` of the vertices, plus the band |y - median y| < 0.4 x the mean edge: a ring of adjacent vertices, a
    pinned crease."""
    v = np.asarray(v, np.float64)
    rng = np.random.default_rng(seed)
    mask = np.zeros(len(v), bool)
    mask[rng.choice(len(v), max(1, int(round(share * len(v)))), replace=False)] = True
    y = v[:, 1] - np.median(v[:, 1])
    mask |= np.abs(y) < 0.4 * mean_edge(np.asarray(v, np.float32), f)
    return mask


def iters_for(v):
    return 2 if len(v) < 1000 else 1


@pytest.mark.parametrize("case", CASES)
def test_constant_target_is_the_scalar_model(case, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    h = mean_edge(v, f)
    it = iters_for(v)
    sv, sf = RM.remesh(v, f, it, h, True)
    for feature in (None, np.zeros(len(v), bool)):
        av, af, afeat = AM.remesh(v, f, it, np.full(len(v), h), True, feature=feature)
        assert np.array_equal(av, sv) and np.array_equal(af, sf) and not afeat.any()


def edges_of(f):
    f = np.asarray(f, np.int64)
    f = f[f[:, 0] >= 0]
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    return {(min(a, b), max(a, b)) for a, b in e.tolist()}


def faces_at(f, mask):
    f = np.asarray(f, np.int64)
    f = f[f[:, 0] >= 0]
    return sorted(tuple(np.roll(t, -int(np.argmin(t))).tolist()) for t in f[mask[f].any(1)])


def adaptive_stages(v, f, t, feat, iters, check):
    """The stages of AM.remesh(v, f, iters, t, feature=feat), with check(stage, before, after) after each one; `before` and
    `after` are (v, f, feature mask)."""
    v, f, (vh, vl, ft) = AM.compact(v, f, 1.4 * t, 0.7 * t, feat)
    V0, F0 = v.copy(), f.copy()
    for _ in range(iters):
        v1, f1, _n, (vh, vl, ft1) = AM.split(v, f, vh, vl, ft)
        check("split", (v, f, ft), (v1, f1, ft1))
        v, f, ft = v1, f1, ft1
        live = len(v)
        while True:
            v1, f1, n = AM.collapse_round(v, f, live, vh, vl, ft)
            check("collapse", (v, f, ft), (v1, f1, ft))
            v, f, live = v1, f1, live - n
            if n == 0:
                break
        v1, f1, (vh, vl, ft1) = AM.compact(v, f, vh, vl, ft)
        check("compact", (v, f, ft), (v1, f1, ft1))
        v, f, ft = v1, f1, ft1
        while True:
            f1, n = AM.flip_round(v, f, ft)
            check("flip", (v, f, ft), (v, f1, ft))
            f = f1
            if n == 0:
                break
        v1 = AM.relax(v, f, V0, F0, ft)
        check("relax", (v, f, ft), (v1, f, ft))
        v = v1
    return v, f, ft


def check_features_untouched(stage, before, after):
    (v0, f0, m0), (v1, f1, m1) = before, after
    k0 = np.flatnonzero(m0)
    if stage == "compact":                                              # the features move with their vertices
        assert np.array_equal(v1[m1], v0[m0])
        return
    assert np.array_equal(m1[:len(m0)], m0) and not m1[len(m0):].any()   # a new midpoint is never a feature
    assert np.array_equal(v1[k0], v0[k0])                               # not moved: no collapse survivor, no relax
    live = np.zeros(len(v1), bool)
    live[f1[f1[:, 0] >= 0].ravel()] = True
    assert live[k0].all()                                               # not collapsed away
    if stage == "split":                                                # every edge at a feature is still an edge
        e0, e1 = edges_of(f0), edges_of(f1)
        assert all(e in e1 for e in e0 if m0[e[0]] or m0[e[1]])
    if stage == "flip":                                                 # a flip rewrites the faces of all four vertices
        assert faces_at(f1, m1) == faces_at(f0, m0)


@pytest.mark.parametrize("scale", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("case", ["octahedron", "ico_in", "components", "ico3"])
def test_features_are_never_split_collapsed_flipped_or_moved(case, scale, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    t = graded_target(v, scale * mean_edge(v, f))
    feat = features(v, f)
    stages = []

    def check(stage, before, after):
        stages.append(stage)
        check_features_untouched(stage, before, after)

    vo, fo, fto = adaptive_stages(v, f, t, feat, 2, check)
    assert {"split", "collapse", "compact", "flip", "relax"} <= set(stages)
    mv, mf, mfeat = AM.remesh(v, f, 2, t, True, feature=feat)           # the stages are the whole call
    assert np.array_equal(vo, mv) and np.array_equal(fo, mf) and np.array_equal(fto, mfeat)
    used = np.zeros(len(v), bool)
    used[f.ravel()] = True
    assert np.array_equal(vo[fto], v[feat & used])                      # every feature survives, in order, where it was


@pytest.mark.parametrize("scale", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("case", ["ico_out", "components", "ico3", "bunny"])
def test_graded_target_keeps_the_invariants(case, scale, bunny_mesh):
    v, f = mesh(case, bunny_mesh)
    t = graded_target(v, scale * mean_edge(v, f))
    for feat in (None, features(v, f, seed=1)):
        vo, fo, fto = AM.remesh(v, f, iters_for(v), t, True, feature=feat)
        RM.assert_invariants(vo, fo, RM.euler(v, f))
        if feat is not None:
            assert np.array_equal(vo[fto], v[feat])


def test_split_and_compact_carry_the_attributes():
    v, f = mesh("octahedron", None)
    vh, vl = np.arange(1.0, 7.0) * 0.3, np.arange(1.0, 7.0) * 0.15
    feat = np.zeros(6, bool)
    feat[5] = True
    v2, f2, n, (h2, l2, ft2) = AM.split(v, f, vh, vl, feat)
    t = RM.Topo(f, 6)
    long = [(a, b) for a, b in t.ev.tolist() if 5 not in (a, b) and np.sum((v[a] - v[b]) ** 2) > ((vh[a] + vh[b]) / 2) ** 2]
    assert n == len(long) > 0 and len(h2) == 6 + n
    assert np.array_equal(h2[6:], [(vh[a] + vh[b]) / 2 for a, b in long]) and np.array_equal(l2[6:], [(vl[a] + vl[b]) / 2 for a, b in long])
    assert np.array_equal(ft2, np.r_[feat, np.zeros(n, bool)])
    g = f.copy()
    g[:, :] = np.where(g == 1, 0, g)                                    # vertex 1 unreferenced, faces with 0 twice are fine here
    cv, cf, (ch, cl, cft) = AM.compact(v, g, vh, vl, feat)
    keep = np.array([0, 2, 3, 4, 5])
    assert np.array_equal(ch, vh[keep]) and np.array_equal(cl, vl[keep]) and np.array_equal(cft, feat[keep])


# ---- remesh_botsch's new arguments and the _v entry points, without a GPU ---------------------------------------------------
def cpu_mesh():
    return torch.zeros(4, 3), torch.tensor([[0, 1, 2], [0, 2, 3], [0, 3, 1], [1, 3, 2]])


@pytest.mark.parametrize("h", [torch.ones(3), torch.ones(4, 1), torch.tensor([1.0, 1.0, float("nan"), 1.0]),
                               torch.tensor([1.0, float("inf"), 1.0, 1.0]), torch.tensor([1.0, 0.0, 1.0, 1.0]),
                               torch.tensor([1.0, 1.0, 1.0, -2.0]), torch.ones(4, dtype=torch.int64),
                               torch.ones(4, dtype=torch.float16)])
def test_bad_per_vertex_h_is_a_value_error(h):
    v, f = cpu_mesh()
    with pytest.raises(ValueError, match="h must be"):
        remesh_botsch(v, f, 1, h)


def test_bad_features():
    v, f = cpu_mesh()
    with pytest.raises(IndexError, match="feature index"):
        remesh_botsch(v, f, 1, 0.5, feature=torch.tensor([0, 4]))
    with pytest.raises(IndexError, match="feature index"):
        remesh_botsch(v, f, 1, 0.5, feature=torch.tensor([-1]))
    with pytest.raises(TypeError, match="feature must be"):
        remesh_botsch(v, f, 1, 0.5, feature=torch.tensor([0.0, 1.0]))
    with pytest.raises(TypeError, match="feature must be"):
        remesh_botsch(v, f, 1, 0.5, feature=[0, 1])
    with pytest.raises(ValueError, match="mask must have shape"):
        remesh_botsch(v, f, 1, 0.5, feature=torch.zeros(5, dtype=torch.bool))
    with pytest.raises(ValueError, match="1-D"):
        remesh_botsch(v, f, 1, 0.5, feature=torch.zeros(2, 2, dtype=torch.int64))


def test_cpu_targets_and_features_are_refused():
    v, f = cpu_mesh()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        remesh_botsch(v, f, 1, torch.full((4,), 0.5))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        remesh_botsch(v, f, 1, 0.5, feature=torch.tensor([0, 1, 1]))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        remesh_botsch(v, f, 1, torch.full((4,), 0.5, dtype=torch.float64), feature=torch.ones(4, dtype=torch.bool))


def aligned_ws(size):
    buf = ctypes.create_string_buffer(size + 256)
    return buf, ctypes.c_void_p((ctypes.addressof(buf) + 255) // 256 * 256)


def test_v_entry_points_need_all_attributes_or_none():
    lib = N.lib()
    n, nv, nf = ctypes.c_int64(-1), ctypes.c_int64(-1), ctypes.c_int64(-1)
    buf, ws = aligned_ws(1 << 16)
    fake = ctypes.c_void_p(256)
    bvh = ctypes.c_void_p(512)
    partial = [(fake, None, None), (None, fake, None), (None, None, fake), (fake, fake, None), (fake, None, fake), (None, fake, fake)]
    for a in partial:
        assert lib.ls_remesh_split_v(fake, fake, 5, 0, 5, 0, 1.0, *a, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
        assert lib.ls_remesh_collapse_round_v(fake, fake, 5, 0, 5, 0.5, 1.0, *a, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
        assert lib.ls_remesh_flip_round_v(fake, fake, 5, 0, *a, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
        assert lib.ls_remesh_compact_v(fake, fake, 5, 0, *a, ws, 1 << 15, ctypes.byref(nv), ctypes.byref(nf), None) == N.LS_ERR_BAD_ARG
        assert lib.ls_remesh_relax_v(fake, fake, 5, 0, bvh, 4, *a, ws, 1 << 15, None) == N.LS_ERR_BAD_ARG
    # with every attribute set the scalar bounds are not read; with none, they are checked as by the scalar entry points
    full, none = (fake, fake, fake), (None, None, None)
    assert lib.ls_remesh_split_v(fake, fake, 5, 0, 5, 0, 0.0, *full, ws, 1 << 15, ctypes.byref(n), None) == N.LS_OK and n.value == 0
    assert lib.ls_remesh_split_v(fake, fake, 5, 0, 5, 0, 0.0, *none, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    n.value = -1
    assert lib.ls_remesh_collapse_round_v(fake, fake, 5, 0, 5, 0.0, 0.0, *full, ws, 1 << 15, ctypes.byref(n), None) == N.LS_OK
    assert n.value == 0
    assert lib.ls_remesh_collapse_round_v(fake, fake, 5, 0, 5, 1.0, 0.5, *none, ws, 1 << 15, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    n.value = -1
    assert lib.ls_remesh_flip_round_v(fake, fake, 5, 0, *full, ws, 1 << 15, ctypes.byref(n), None) == N.LS_OK and n.value == 0
    assert lib.ls_remesh_compact_v(fake, fake, 5, 0, *full, ws, 1 << 15, ctypes.byref(nv), ctypes.byref(nf), None) == N.LS_OK
    assert nv.value == 0 and nf.value == 0


def test_v_entry_points_reject_null_counts_and_small_workspaces():
    lib = N.lib()
    n = ctypes.c_int64(0)
    buf, ws = aligned_ws(4096)
    fake = ctypes.c_void_p(256)
    full = (fake, fake, fake)
    assert lib.ls_remesh_split_v(fake, fake, 4, 4, 10, 16, 1.0, *full, ws, 1 << 20, None, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_split_v(fake, fake, 4, 4, 9, 16, 1.0, *full, ws, 1 << 20, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_collapse_round_v(fake, fake, 4, 4, 4, 0.5, 1.0, *full, ws, 1 << 20, None, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_collapse_round_v(None, fake, 4, 4, 4, 0.5, 1.0, *full, ws, 1 << 20, ctypes.byref(n), None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_flip_round_v(fake, fake, 4, 4, *full, ws, 1 << 20, None, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_flip_round_v(fake, fake, 4, 4, *full, ws, 16, ctypes.byref(n), None) == N.LS_ERR_WORKSPACE
    assert lib.ls_remesh_compact_v(fake, fake, 4, 4, *full, ws, 1 << 20, None, None, None) == N.LS_ERR_BAD_ARG
    assert lib.ls_remesh_compact_v(fake, fake, 4, 4, *full, ws, 16, ctypes.byref(n), ctypes.byref(n), None) == N.LS_ERR_WORKSPACE
    assert lib.ls_remesh_relax_v(fake, fake, 4, 4, None, 4, *full, ws, 1 << 20, None) == N.LS_ERR_BAD_ARG
