"""GPU: the matrix-free cotangent product laplacian_cot_product(v, f, x) = laplacian_cot(v, f) @ x (ls_cot_laplacian_product_f32
/ _bwd_f32) and its gradients w.r.t. the positions and x.  Small meshes against the reference's float64 gradients
(tests/golden/cot_grad.npz), large ones against the float64 numpy model (tests/cot_grad_model.py) and the matrix path."""
import os

import numpy as np
import pytest
import torch

import cot_grad_model as model
from conftest import GOLDEN
from gpu_util import DEV, config2, rel_l2
from largesteps_b200 import _native as N, batch, meshops, workloads
from largesteps_b200.geometry import laplacian_cot
from largesteps_b200.meshops import laplacian_cot_product
from test_cot_product_host import forward_bound, model_product

pytestmark = pytest.mark.gpu

MESHES = ["ico2", "bunny", "grid", "plane", "degen"]
IDX = [torch.int64, torch.int32]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "cot_grad.npz"))


@pytest.fixture(scope="module")
def big(bunny_mesh):
    v2, f2, _ = config2(bunny_mesh)
    vp, fp = workloads.plane(300)
    return {"bunny_x2": (v2, f2), "plane300": (vp.astype(np.float32), fp)}


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def reg(v, f, loss):
    y = laplacian_cot_product(v, f, v)
    return y.square().mean() if loss == "reg_bi" else (v * y).mean()


def grad_of(fn, v):
    x = v.clone().requires_grad_(True)
    loss = fn(x)
    loss.backward()
    return loss.detach(), x.grad


@pytest.mark.parametrize("idx_dtype", IDX)
@pytest.mark.parametrize("loss", ["reg_bi", "reg_lap"])
@pytest.mark.parametrize("mesh", MESHES)
def test_regulariser_gradient_matches_reference(golden, mesh, loss, idx_dtype):
    v, f = model.golden_mesh(golden, mesh)
    _, grad = grad_of(lambda x: reg(x, t(f).to(idx_dtype), loss), t(v))
    grad = grad.cpu().numpy()
    assert np.isfinite(grad).all()
    err, ref_err = rel_l2(grad, golden[f"{mesh}.{loss}.grad"]), float(golden[f"{mesh}.{loss}.f32_err"])
    print(f"{mesh} {loss}: rel-L2 vs the reference's float64 run {err:.2e} (its float32 run: {ref_err:.2e})")
    assert err < max(5e-6, 20 * ref_err), (err, ref_err)


@pytest.mark.parametrize("k", [1, 3, 4])
@pytest.mark.parametrize("mesh", MESHES + ["bunny_x2", "plane300"])
def test_forward_matches_float64_model(golden, big, mesh, k):
    v, f = big[mesh] if mesh in big else model.golden_mesh(golden, mesh)
    x = np.random.default_rng(k).normal(size=(len(v), k)).astype(np.float32)
    y = laplacian_cot_product(t(v), t(f), t(x)).cpu().numpy()
    err, bound = np.abs(y - model_product(v, f, x)).max(), forward_bound(v, f, x)
    assert err <= bound, (err, bound)


@pytest.mark.parametrize("name", ["bunny_x2", "plane300"])
def test_each_gradient_alone(big, name):
    v, f = big[name]
    rng = np.random.default_rng(7)
    x = rng.normal(size=(len(v), 3)).astype(np.float32)
    gy = rng.normal(size=(len(v), 3)).astype(np.float32)
    tv, tf, tx, tgy = t(v), t(f), t(x), t(gy)
    laplacian_cot_product(tv, tf, tx)                      # caches the incidence list
    rows, cols, _ = model.laplacian(v, f)
    want_v = model.cot_vjp(v, f, rows, cols, model.spmm_grad_values(rows, cols, gy, x), 1.0)
    want_x = laplacian_cot_product(tv, tf, tgy)
    for need_v, need_x, launches in ((True, False, 2), (False, True, 1), (True, True, 3)):
        a = tv.clone().requires_grad_(need_v)
        b = tx.clone().requires_grad_(need_x)
        y = laplacian_cot_product(a, tf, b)
        torch.cuda.synchronize()
        n0 = N.launch_count()
        y.backward(tgy)
        torch.cuda.synchronize()
        assert N.launch_count() - n0 == launches
        assert (a.grad is not None) == need_v and (b.grad is not None) == need_x
        if need_v:
            err = rel_l2(a.grad.cpu().numpy(), want_v)
            print(f"{name}: gradient w.r.t. verts, rel-L2 vs the float64 model {err:.2e}")
            assert torch.isfinite(a.grad).all() and err < 2e-5, err
        if need_x:
            assert torch.equal(b.grad.view(torch.int32), want_x.view(torch.int32))


@pytest.mark.parametrize("loss", ["reg_bi", "reg_lap"])
@pytest.mark.parametrize("name", ["bunny_x2", "plane300"])
def test_agrees_with_the_matrix_path(big, name, loss):
    """The loss agrees with laplacian_regularizer(laplacian_cot(v, f), v) to 2e-5.  The gradients are both held against the
    float64 model: the matrix path's weight gradient Gbar_ii + Gbar_jj - Gbar_ij - Gbar_ji, Gbar_ij = gy_i . v_j, cancels in
    float32 (for reg_lap it is |v_i - v_j|^2 / n formed as |v_i|^2 + |v_j|^2 - 2 v_i . v_j: about 1e-2 rel-L2 on plane(300)),
    whereas the matrix-free path forms the differences first.  So the bar is the model's, and the new path must be no
    further from it than the matrix path."""
    v, f = big[name]
    tv, tf = t(v), t(f)
    l0, g0 = grad_of(lambda x: meshops.laplacian_regularizer(laplacian_cot(x, tf), x, bilaplacian=loss == "reg_bi"), tv)
    l1, g1 = grad_of(lambda x: reg(x, tf, loss), tv)
    want = model.loss_grad(v, f, loss)
    el = abs(float(l1) - float(l0)) / abs(float(l0))
    e0, e1 = rel_l2(g0.cpu().numpy(), want), rel_l2(g1.cpu().numpy(), want)
    print(f"{name} {loss}: loss rel {el:.2e} vs the matrix path; gradient rel-L2 vs the float64 model: matrix-free {e1:.2e}, "
          f"matrix path {e0:.2e}")
    assert el < 2e-5, el
    assert e1 < 2e-5 and e1 <= e0, (e1, e0)


def run(v, f, x, gy):
    """(y, grad verts, grad x) of one call and its backward."""
    a, b = v.clone().requires_grad_(True), x.clone().requires_grad_(True)
    y = laplacian_cot_product(a, f, b)
    y.backward(gy)
    return y.detach(), a.grad, b.grad


def bits(*ts):
    return [u.contiguous().view(torch.int32) for u in ts]


@pytest.mark.parametrize("idx_dtype", IDX)
def test_packed_meshes_are_bitwise_per_mesh(golden, bunny_mesh, idx_dtype):
    vb, fb, _ = config2(bunny_mesh)
    meshes = [model.golden_mesh(golden, m) for m in ("ico2", "degen", "grid")] + [(vb, fb)]
    rng = np.random.default_rng(11)
    vs = [t(np.asarray(v, np.float32)) for v, _ in meshes]
    fs = [t(f).to(idx_dtype) for _, f in meshes]
    xs = [t(rng.normal(size=(len(v), 3)).astype(np.float32)) for v, _ in meshes]
    gys = [t(rng.normal(size=(len(v), 3)).astype(np.float32)) for v, _ in meshes]
    p = batch.pack_meshes(vs, fs)
    got = run(p.verts, p.faces, torch.cat(xs), torch.cat(gys))
    vo = p.vert_offsets_host
    for i in range(len(meshes)):
        want = run(vs[i], fs[i], xs[i], gys[i])
        for g, w in zip(bits(*got), bits(*want)):
            assert torch.equal(g[vo[i]:vo[i + 1]], w)


def test_bitwise_reproducible_stream_and_index_type_independent(big):
    v, f = big["bunny_x2"]
    rng = np.random.default_rng(5)
    tv, tx, tgy = t(v), t(rng.normal(size=(len(v), 4)).astype(np.float32)), t(rng.normal(size=(len(v), 4)).astype(np.float32))
    f64, f32 = t(f), t(f).to(torch.int32)
    a, b = run(tv, f64, tx, tgy), run(tv, f64, tx, tgy)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c = run(tv, f64, tx, tgy)
    torch.cuda.current_stream().wait_stream(s)
    d = run(tv, f32, tx, tgy)
    torch.cuda.synchronize()
    for other in (b, c, d):
        for g, w in zip(bits(*a), bits(*other)):
            assert torch.equal(g, w)


def test_graph_only_where_asked_for(golden):
    v, f = model.golden_mesh(golden, "ico2")
    tv, tf = t(v), t(f)
    assert laplacian_cot_product(tv, tf, tv).grad_fn is None
    x = tv.clone().requires_grad_(True)
    with torch.no_grad():
        assert laplacian_cot_product(x, tf, x).grad_fn is None
    assert laplacian_cot_product(x, tf, tv).grad_fn is not None
    assert laplacian_cot_product(tv, tf, x).grad_fn is not None


def test_bad_input_raises(golden):
    v, f = model.golden_mesh(golden, "ico2")
    tv, tf = t(v), t(f)
    V = len(v)
    with pytest.raises(RuntimeError):
        laplacian_cot_product(tv.cpu(), tf.cpu(), tv.cpu())
    with pytest.raises(RuntimeError):
        laplacian_cot_product(tv, tf, tv.cpu())
    with pytest.raises(RuntimeError):
        laplacian_cot_product(tv, tf.cpu(), tv)
    with pytest.raises(ValueError):
        laplacian_cot_product(tv, tf, tv[:, 0])
    with pytest.raises(ValueError):
        laplacian_cot_product(tv, tf, tv[:-1])
    with pytest.raises(ValueError):
        laplacian_cot_product(tv, tf, tv[:, :0])
    with pytest.raises(TypeError):
        laplacian_cot_product(tv, tf, tv.double())
    with pytest.raises(TypeError):
        laplacian_cot_product(tv.double(), tf, tv)
    with pytest.raises(TypeError):
        laplacian_cot_product(tv, tf.to(torch.int16), tv)
    with pytest.raises(ValueError):
        laplacian_cot_product(tv[:, :2], tf, tv)
    bad = tf.clone()
    bad[0, 2] = V
    with pytest.raises(IndexError):
        laplacian_cot_product(tv, bad, tv)
    bad[0, 2] = -1
    with pytest.raises(IndexError):
        laplacian_cot_product(tv, bad.to(torch.int32), tv)
