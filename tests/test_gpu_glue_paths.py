"""GPU: the loop glue of csrc/ls_glue.cu one gradient path at a time, against the float64 model of tests/glue_model.py.

gather_rows is checked bitwise: its forward is x[idx], its backward a strict left-to-right float32 sum of the incoming rows
in ascending position order.  The normals are checked per path, each by its own rel-L2, so a path that is small in the
loop's total gradient cannot hide under the others:
  face normals: forward (per face, against a rounding bound) and the backward of sum(W3 fn);
  vertex normals: (a) the forward, (b) the gradient reaching the face normals, (c) the gradient reaching the positions
  through the corner angles, with the face normals a constant.
The bars follow tests/test_gpu_meshops.py: rel-L2 below max(5e-6, 20 x the error of the same model run in float32)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from largesteps_b200 import meshops, workloads
from largesteps_b200.batch import pack_meshes
from gpu_util import DEV, fan_mesh, rel_l2
import glue_model as M

pytestmark = pytest.mark.gpu

EPS = float(np.finfo(np.float32).eps) / 2          # unit roundoff u of float32
IDX = pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["int32", "int64"])


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def gamma(k):
    return k * EPS / (1 - k * EPS)


def bar(w32, w64):
    return max(5e-6, 20 * rel_l2(w32, w64))


# ---- gather_rows --------------------------------------------------------------------------------------------------------
def sequential_rows_sum(g, idx, V):
    """out[v] = (((+0 + g[p0]) + g[p1]) + ...) over the positions p0 < p1 < ... with idx[p] = v, in float32."""
    k = g.shape[1]
    out = np.zeros((V, k), np.float32)
    order = np.argsort(idx, kind="stable")                 # ascending position within each row
    rows = idx[order]
    counts = np.bincount(idx, minlength=V)
    start = np.concatenate([[0], np.cumsum(counts)[:-1]])
    rank = np.arange(len(idx)) - start[rows]
    long_rows = np.nonzero(counts > 64)[0]
    for v in long_rows:                                    # np.cumsum adds strictly left to right
        out[v] = np.cumsum(g[order[start[v]:start[v] + counts[v]]], axis=0, dtype=np.float32)[-1]
    short = ~np.isin(rows, long_rows)
    for r in range(int(rank[short].max()) + 1 if short.any() else 0):
        sel = short & (rank == r)
        out[rows[sel]] = out[rows[sel]] + g[order[sel]]
    return out


def gather_pattern(name, rng):
    if name == "random":
        V = 1000
        return V, rng.integers(0, V, 5000)
    if name == "hub":               # one row 2e5 times: a long bucket through the shell sort
        V = 1000
        idx = np.concatenate([np.full(200000, 17), rng.integers(0, V, 3000)])
        return V, rng.permutation(idx)
    if name == "one_row":
        return 50, np.full(10000, 3)
    if name == "unhit":             # odd rows are never hit: their gradient is exactly zero
        V = 1000
        return V, 2 * rng.integers(0, V // 2, 4000)
    if name == "empty":
        return 10, np.zeros(0, np.int64)
    if name == "large":
        V = 1000000
        return V, rng.integers(0, V, 1200000)
    raise KeyError(name)


@pytest.mark.parametrize("k", [1, 2, 3, 4, 7])
@pytest.mark.parametrize("pattern", ["random", "hub", "one_row", "unhit", "empty", "large"])
@IDX
def test_gather_rows(pattern, k, idx_dtype):
    rng = np.random.default_rng(k)
    V, idx = gather_pattern(pattern, rng)
    x_np = rng.normal(size=(V, k)).astype(np.float32)
    # magnitudes over six decades, so that another summation order gives other bits
    g_np = (rng.normal(size=(len(idx), k)) * 10.0 ** rng.uniform(-3, 3, size=(len(idx), k))).astype(np.float32)
    x = t(x_np).requires_grad_(True)
    ti = t(idx).to(idx_dtype)
    y = meshops.gather_rows(x, ti)
    assert y.shape == (len(idx), k)
    assert torch.equal(y.detach().cpu(), torch.from_numpy(x_np[idx]))
    y.backward(t(g_np))
    got = x.grad.cpu().numpy()
    want = sequential_rows_sum(g_np, idx, V)
    np.testing.assert_array_equal(got, want)               # values: the sign of a zero may differ
    hit = np.bincount(idx, minlength=V) > 0
    assert (got[~hit] == 0).all()
    if pattern == "unhit":
        assert (~hit).sum() >= V // 2


# ---- the meshes -------------------------------------------------------------------------------------------------------------
MESHES = ["triangle", "two_triangles", "tetrahedron", "icosahedron", "isolated", "ico2", "bunny", "fan3000", "plane1000"]
_cache = {}


def mesh(name):
    if name not in _cache:
        small = M.small_meshes()
        if name in small:
            v, f = small[name]
        elif name == "ico2":
            g = np.load(os.path.join(GOLDEN, "glue.npz"))
            v, f = g["ico2.v_unique"], g["ico2.f_unique"]
        elif name == "bunny":
            d = np.load(os.path.join(GOLDEN, "bunny_mesh.npz"))
            v, f = d["verts"].astype(np.float32), d["faces"].astype(np.int64)
        elif name == "fan3000":
            v, f = fan_mesh(3000)
        else:                       # V = 1e6, F ~ 2e6: the reductions run on the full grid of 528 CTAs
            v, f = workloads.plane(1000)
        _cache[name] = (np.ascontiguousarray(v, np.float32), np.ascontiguousarray(f, np.int64))
    return _cache[name]


def model(name):
    """The model's face normals, the three paths of the vertex normals (float64 and float32), and the sizes of the paths
    within the total gradient of the loop's combined loss sum(W1 v_opt) + sum(W2 n_opt) + sum(W3 fn)."""
    key = ("model", name)
    if key in _cache:
        return _cache[key]
    v, f = mesh(name)
    V, F = len(v), len(f)
    rng = np.random.default_rng(5)
    W3 = rng.normal(size=(3, F)).astype(np.float32)
    gout = rng.normal(size=(V, 3)).astype(np.float32)
    fn64, gfw64 = M.face_normal_vjp(v, f, W3)
    _, gfw32 = M.face_normal_vjp(v, f, W3, dtype=torch.float32)
    fn = fn64.astype(np.float32)
    m64 = M.vertex_normal_paths(v, f, fn, gout)
    m32 = M.vertex_normal_paths(v, f, fn, gout, dtype=torch.float32)
    # path sizes in the combined loss (dup = identity, W1 = W2 = gout: every term has unit-scale weights)
    _, total, _, _ = M.loop_loss(v, f, np.arange(V), gout, gout, W3)
    full = M.vertex_normal_paths(v, f, fn64, gout)
    _, via_fn = M.face_normal_vjp(v, f, W3.astype(np.float64) + full["g_fn"])
    _, via_nfn = M.face_normal_vjp(v, f, full["g_fn"])
    nt = np.linalg.norm(total)
    sizes = dict(angle=np.linalg.norm(full["g_angle"]) / nt, face_normals_of_n=np.linalg.norm(via_nfn) / nt,
                 all_face_normals=np.linalg.norm(via_fn) / nt, gather=np.linalg.norm(gout) / nt)
    _cache[key] = out = dict(W3=W3, gout=gout, fn64=fn64, fn=fn, gfw64=gfw64, gfw32=gfw32, m64=m64, m32=m32, sizes=sizes)
    return out


@pytest.mark.parametrize("name", MESHES)
@IDX
def test_face_normals(name, idx_dtype):
    v, f = mesh(name)
    m = model(name)
    x = t(v).requires_grad_(True)
    fn = meshops.compute_face_normals(x, t(f).to(idx_dtype))
    # |n - n64|_inf <= gamma_12 (1 + |e1| |e2| / |e1 x e2|): e1, e2 and the cross product's components carry gamma_5 of
    # |e1| |e2|, normalising by |c| doubles that relative to |c| and adds the rounding of the norm and the division
    v64, fl = v.astype(np.float64), f
    e1, e2 = v64[fl[:, 1]] - v64[fl[:, 0]], v64[fl[:, 2]] - v64[fl[:, 0]]
    cond = np.linalg.norm(e1, axis=1) * np.linalg.norm(e2, axis=1) / np.linalg.norm(np.cross(e1, e2), axis=1)
    err = np.abs(fn.detach().cpu().numpy().astype(np.float64) - m["fn64"]).max(0)
    assert (err <= gamma(12) * (1 + cond)).all(), (err / (1 + cond)).max()
    fn.backward(t(m["W3"]))
    e = rel_l2(x.grad.cpu().numpy(), m["gfw64"])
    b = bar(m["gfw32"], m["gfw64"])
    print(f"{name}: face normals forward max err / bound {(err / (gamma(12) * (1 + cond))).max():.2f}, "
          f"backward rel-L2 {e:.2e} (bound {b:.2e})")
    assert e < b, (e, b)


def vertex_paths(x_np, f, fn_np, gout_np):
    """compute_vertex_normals' three paths, each from its own call: the forward, the gradient reaching the face normals
    (positions without grad), and the gradient reaching the positions (face normals a constant)."""
    fn_leaf = t(fn_np).requires_grad_(True)
    n = meshops.compute_vertex_normals(t(x_np), f, fn_leaf)
    n.backward(t(gout_np))
    x = t(x_np).requires_grad_(True)
    meshops.compute_vertex_normals(x, f, t(fn_np)).backward(t(gout_np))
    return dict(n=n.detach().cpu().numpy(), g_fn=fn_leaf.grad.cpu().numpy(), g_angle=x.grad.cpu().numpy())


def check_paths(name, got, m64, m32, gout):
    nan = np.isnan(m64["n"]).any(1)
    np.testing.assert_array_equal(np.isnan(got["n"]).any(1), nan)
    assert nan.any() == (name == "isolated")
    report = []
    for path in ("n", "g_fn", "g_angle"):
        a, w64, w32 = got[path], m64[path], m32[path]
        if path == "n":
            a, w64, w32 = a[~nan], w64[~nan], w32[~nan]
        assert np.isfinite(a).all(), path
        if name == "triangle" and path == "g_angle":
            # every vertex normal is the face normal whatever the angles: the path is zero up to rounding
            assert np.abs(w64).max() < 1e-12
            e = np.linalg.norm(a) / np.linalg.norm(gout)
            report.append(f"{path} |g|/|gout| {e:.1e} (bound {64 * 2 * EPS:.1e})")
            assert e < 64 * 2 * EPS, e
            continue
        e, b = rel_l2(a, w64), bar(w32, w64)
        report.append(f"{path} {e:.2e} (bound {b:.2e})")
        assert e < b, (name, path, e, b)
    return report


@pytest.mark.parametrize("name", MESHES)
@IDX
def test_vertex_normals_paths(name, idx_dtype):
    v, f = mesh(name)
    m = model(name)
    got = vertex_paths(v, t(f).to(idx_dtype), m["fn"], m["gout"])
    report = check_paths(name, got, m["m64"], m["m32"], m["gout"])
    s = m["sizes"]
    print(f"{name}: " + ", ".join(report) + f"; share of the combined loss's gradient: angle path {s['angle']:.1e}, "
          f"face normals via n {s['face_normals_of_n']:.1e}, all face normals {s['all_face_normals']:.1e}, "
          f"gather {s['gather']:.1e}; norms {m['m64']['norms']}, T {m['m64']['T']}")


@IDX
def test_full_grid_reductions_are_reproducible(idx_dtype):
    """plane1000 runs k_edge_norms_batch and bwd1 on all 528 CTAs: repeated calls, and a call on another stream, give the same
    bits (the ticket of the last-CTA reduction is reset by every call)."""
    v, f = mesh("plane1000")
    m = model("plane1000")
    tf = t(f).to(idx_dtype)
    runs = [vertex_paths(v, tf, m["fn"], m["gout"]) for _ in range(3)]
    s = torch.cuda.Stream(device=DEV)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        runs.append(vertex_paths(v, tf, m["fn"], m["gout"]))
    torch.cuda.current_stream().wait_stream(s)
    for r in runs[1:]:
        for path in ("n", "g_fn", "g_angle"):
            np.testing.assert_array_equal(r[path], runs[0][path])


# ---- packed meshes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["forward", "reversed"])
@IDX
def test_vertex_normals_batch_paths(order, idx_dtype):
    """Each mesh of a packed batch against the model on that mesh alone.  The tiny meshes' global norms are orders of
    magnitude below bunny's, so taking another mesh's norms or T is far outside the bound."""
    names = ["triangle", "empty", "tetrahedron", "bunny"]
    if order == "reversed":
        names = names[::-1]
    empty = (np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64))
    ms = [empty if nm == "empty" else mesh(nm) for nm in names]
    p = pack_meshes([t(v) for v, _ in ms], [t(f).to(idx_dtype) for _, f in ms])
    rng = np.random.default_rng(9)
    models, fns, gouts = [], [], []
    for v, f in ms:
        fn = M.face_normal_vjp(v, f, np.zeros((3, len(f))))[0].astype(np.float32) if len(f) else np.zeros((3, 0), np.float32)
        gout = rng.normal(size=(len(v), 3)).astype(np.float32)
        fns.append(fn)
        gouts.append(gout)
        models.append((M.vertex_normal_paths(v, f, fn, gout), M.vertex_normal_paths(v, f, fn, gout, dtype=torch.float32))
                      if len(f) else None)
    fn_all, gout_all = np.concatenate(fns, 1), np.concatenate(gouts, 0)
    vo, fo = p.vert_offsets_host, p.face_offsets_host
    fn_leaf = t(fn_all).requires_grad_(True)
    n = meshops.compute_vertex_normals_batch(p.verts, p.faces, fn_leaf, p.vert_offsets, p.face_offsets)
    n.backward(t(gout_all))
    x = p.verts.clone().requires_grad_(True)
    meshops.compute_vertex_normals_batch(x, p.faces, t(fn_all), p.vert_offsets, p.face_offsets).backward(t(gout_all))
    n, g_fn, g_angle = n.detach().cpu().numpy(), fn_leaf.grad.cpu().numpy(), x.grad.cpu().numpy()
    for i, nm in enumerate(names):
        if nm == "empty":
            continue
        got = dict(n=n[vo[i]:vo[i + 1]], g_fn=g_fn[:, fo[i]:fo[i + 1]], g_angle=g_angle[vo[i]:vo[i + 1]])
        print(f"batch {nm}: " + ", ".join(check_paths(nm, got, *models[i], gouts[i])))
