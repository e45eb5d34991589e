"""GPU: gradients of the cotangent matrices w.r.t. the vertex positions (ls_laplacian_cot_bwd_f32) and of L @ v w.r.t. L's
values (ls_spmm_csr_grad_val_f32), through compute_matrix / laplacian_cot, to_differential, laplacian_regularizer and
torch's own sparse product.  Small meshes against the reference's float64 gradients (tests/golden/cot_grad.npz), large ones
against the float64 numpy model (tests/cot_grad_model.py)."""
import os

import numpy as np
import pytest
import torch

import cot_grad_model as model
from conftest import GOLDEN
from gpu_util import DEV, config2, rel_l2
from largesteps_b200 import geometry, meshops, remesh, workloads
from largesteps_b200.geometry import compute_matrix, laplacian_cot, laplacian_uniform
from largesteps_b200.parameterize import from_differential, spmm, spmm_grad_values, to_differential

pytestmark = pytest.mark.gpu

IDX = [torch.int64, torch.int32]
MESHES = ["ico2", "bunny", "grid", "plane", "degen"]
LOSSES = ["l19", "a095", "td", "reg_bi", "reg_lap"]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "cot_grad.npz"))


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def mesh_of(g, mesh):
    v, f = model.golden_mesh(g, mesh)
    return t(v), t(f)


def loss_fn(g, mesh, loss):
    if loss in ("l19", "a095", "td"):
        w = t(model.golden_weights(g, mesh, loss))
    if loss == "l19":
        return lambda x, f: (compute_matrix(x, f, 19.0, cotan=True).values() * w).sum()
    if loss == "a095":
        return lambda x, f: (compute_matrix(x, f, 1.0, alpha=0.95, cotan=True).values() * w).sum()
    if loss == "td":
        return lambda x, f: (to_differential(compute_matrix(x, f, 19.0, cotan=True), x) * w).sum()
    bi = loss == "reg_bi"
    return lambda x, f: meshops.laplacian_regularizer(laplacian_cot(x, f), x, bilaplacian=bi)


def grad_of(fn, v, f):
    x = v.clone().requires_grad_(True)
    fn(x, f).backward()
    return x.grad


@pytest.mark.parametrize("idx_dtype", IDX)
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("mesh", MESHES)
def test_gradient_matches_reference(golden, mesh, loss, idx_dtype):
    g = golden
    v, f = mesh_of(g, mesh)
    grad = grad_of(loss_fn(g, mesh, loss), v, f.to(idx_dtype)).cpu().numpy()
    assert np.isfinite(grad).all()              # as the reference's: the area clamp keeps degenerate faces finite
    err, ref_err = rel_l2(grad, g[f"{mesh}.{loss}.grad"]), float(g[f"{mesh}.{loss}.f32_err"])
    print(f"{mesh} {loss}: rel-L2 vs the reference's float64 run {err:.2e} (its float32 run: {ref_err:.2e})")
    assert err < max(5e-6, 20 * ref_err), (err, ref_err)


@pytest.mark.parametrize("mesh", MESHES)
def test_values_match_reference(golden, mesh):
    """The reference's pattern; values against the float64 model (pinned to the reference's float32 values on ico2 and the
    bunny in tests/test_cot_grad_model.py)."""
    v, f = mesh_of(golden, mesh)
    M = compute_matrix(v.requires_grad_(True), f, 19.0, cotan=True)
    assert M.requires_grad
    np.testing.assert_array_equal(M.indices().cpu().numpy(), golden[f"{mesh}.idx"])
    _, _, ref = model.matrix(*model.golden_mesh(golden, mesh), 1.0, 19.0)
    assert np.abs(M.values().detach().cpu().numpy() - ref).max() <= 2e-6 * np.abs(ref).max()


def big_meshes(bunny_mesh):
    v2, f2, _ = config2(bunny_mesh)
    vp, fp = workloads.plane(300)
    return {"bunny_x2": (v2, f2), "plane300": (vp.astype(np.float32), fp)}


@pytest.mark.parametrize("name", ["bunny_x2", "plane300"])
def test_large_meshes_match_model(bunny_mesh, name):
    v, f = big_meshes(bunny_mesh)[name]
    rng = np.random.default_rng(3)
    M = compute_matrix(t(v), t(f), 19.0, cotan=True)
    W = rng.normal(size=M._nnz()).astype(np.float32)
    G = rng.normal(size=v.shape).astype(np.float32)
    idx = M.indices().cpu().numpy()
    for loss, fn, Wl in (("l19", lambda x, ff: (compute_matrix(x, ff, 19.0, cotan=True).values() * t(W)).sum(), W),
                         ("td", lambda x, ff: (to_differential(compute_matrix(x, ff, 19.0, cotan=True), x) * t(G)).sum(), None)):
        grad = grad_of(fn, t(v), t(f)).cpu().numpy()
        want = model.loss_grad(v, f, loss, W=Wl, G=G)
        if loss == "l19":
            rows, cols, _ = model.laplacian(v, f)
            np.testing.assert_array_equal(idx, np.stack([rows, cols]))
        err = rel_l2(grad, want)
        print(f"{name} {loss}: rel-L2 vs the float64 model {err:.2e}")
        assert np.isfinite(grad).all() and err < 2e-5, err


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5])
def test_values_gradient_kernel_within_gamma_bound(bunny_mesh, k):
    """ls_spmm_csr_grad_val_f32 against an fp64 sum_k gy x per entry: |err| <= gamma_k sum_k |gy x| (k products summed)."""
    v, f, _ = config2(bunny_mesh)
    M = compute_matrix(t(v), t(f), 19.0, cotan=True)
    rng = np.random.default_rng(k)
    x = rng.normal(size=(len(v), k)).astype(np.float32)
    gy = rng.normal(size=(len(v), k)).astype(np.float32)
    got = spmm_grad_values(M, t(gy), t(x)).cpu().numpy().astype(np.float64)
    r, c = M.indices().cpu().numpy()
    prod = gy.astype(np.float64)[r] * x.astype(np.float64)[c]
    gamma = k * 2.0 ** -24 / (1 - k * 2.0 ** -24)
    assert (np.abs(got - prod.sum(1)) <= gamma * np.abs(prod).sum(1) + 1e-30).all()
    if k == 1:      # 1-D vectors take the same path
        got1 = spmm_grad_values(M, t(gy[:, 0]), t(x[:, 0]))
        assert torch.equal(got1, t(got.astype(np.float32)))


def test_gradients_are_bitwise_reproducible_and_stream_independent(bunny_mesh):
    v, f, _ = config2(bunny_mesh)
    tv, tf = t(v), t(f)
    G = t(np.random.default_rng(5).normal(size=v.shape).astype(np.float32))

    def run():
        return grad_of(lambda x, ff: (to_differential(compute_matrix(x, ff, 19.0, cotan=True), x) * G).sum()
                       + meshops.laplacian_regularizer(laplacian_cot(x, ff), x), tv, tf)

    a, b = run(), run()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        c = run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(a.view(torch.int32), c.view(torch.int32))


@pytest.mark.parametrize("kw", [dict(lambda_=19.0), dict(lambda_=1.0, alpha=0.95)])
def test_values_bitwise_with_and_without_requires_grad(golden, kw):
    v, f = mesh_of(golden, "bunny")
    M0 = compute_matrix(v, f, cotan=True, **kw)
    M1 = compute_matrix(v.clone().requires_grad_(True), f, cotan=True, **kw)
    assert not M0.requires_grad and M1.requires_grad
    assert torch.equal(M0.indices(), M1.indices())
    assert torch.equal(M0.values().view(torch.int32), M1.values().detach().view(torch.int32))
    L0, L1 = laplacian_cot(v, f), laplacian_cot(v.clone().requires_grad_(True), f)
    assert torch.equal(L0.values().view(torch.int32), L1.values().detach().view(torch.int32))


def test_no_graph_where_none_is_asked_for(golden):
    v, f = mesh_of(golden, "ico2")
    x = v.clone().requires_grad_(True)
    assert not compute_matrix(v, f, 19.0, cotan=True).requires_grad
    with torch.no_grad():
        M = compute_matrix(x, f, 19.0, cotan=True)
        assert not M.requires_grad and not laplacian_cot(x, f).requires_grad
        assert not to_differential(M, x).requires_grad
    assert not compute_matrix(x, f, 19.0).requires_grad            # uniform: values do not depend on positions
    assert not laplacian_uniform(x, f).requires_grad
    assert geometry.values_with_graph(compute_matrix(x, f, 19.0)) is None
    rp = remesh.Reparameterizer(lambda_=19.0, cotan=True, method="CG")
    M, u = rp.update(x, f)
    assert not M.requires_grad and u.requires_grad                  # u = M v keeps its graph to v only
    u.sum().backward()
    assert torch.equal(x.grad, spmm(M, torch.ones_like(v)))         # M^T 1 = M 1: the SpMM, as before


def test_from_differential_gradient_goes_to_u_only(golden):
    v, f = mesh_of(golden, "bunny")
    G = t(model.golden_weights(golden, "bunny", "td"))
    M0 = compute_matrix(v, f, 19.0, cotan=True)
    x = v.clone().requires_grad_(True)
    M1 = compute_matrix(x, f, 19.0, cotan=True)
    grads = []
    for M in (M0, M1):
        u = to_differential(M0, v).clone().requires_grad_(True)
        (from_differential(M, u, "Cholesky") * G).sum().backward()
        grads.append(u.grad)
    assert torch.equal(grads[0], grads[1])
    assert x.grad is None


@pytest.mark.parametrize("idx_dtype", IDX)
def test_torch_sparse_product_gives_the_same_gradient(golden, idx_dtype):
    v, f = mesh_of(golden, "bunny")
    f = f.to(idx_dtype)
    G = t(model.golden_weights(golden, "bunny", "td"))
    grads = []
    for prod in (to_differential, lambda M, x: M @ x, torch.sparse.mm):
        x = v.clone().requires_grad_(True)
        (prod(compute_matrix(x, f, 19.0, cotan=True), x.detach()) * G).sum().backward()
        grads.append(x.grad)
    assert rel_l2(grads[1].cpu(), grads[0].cpu()) < 1e-6 and rel_l2(grads[2].cpu(), grads[0].cpu()) < 1e-6


def test_foreign_matrix_gets_a_sparse_values_gradient(golden):
    """A torch sparse matrix whose values require grad (not built by compute_matrix) gets the sampled product as its
    gradient on its coalesced pattern, as torch's own L @ v gives it."""
    v, f = mesh_of(golden, "ico2")
    M = compute_matrix(v, f, 19.0, cotan=True)
    vals = M.values().clone().requires_grad_(True)
    G = t(model.golden_weights(golden, "ico2", "td"))
    grads = []
    for prod in (to_differential, lambda A, x: A @ x):
        A = torch.sparse_coo_tensor(M.indices(), vals, M.shape).coalesce()
        (prod(A, v) * G).sum().backward()
        grads.append(vals.grad.clone())
        vals.grad = None
    assert rel_l2(grads[0].cpu(), grads[1].cpu()) < 1e-6


def test_bad_input_raises_as_the_forward_does(golden):
    v, f = mesh_of(golden, "ico2")
    x = v.clone().requires_grad_(True)
    with pytest.raises(RuntimeError):
        compute_matrix(x.cpu(), f.cpu(), 19.0, cotan=True)
    with pytest.raises(RuntimeError):
        compute_matrix(x, f.cpu(), 19.0, cotan=True)
    with pytest.raises(TypeError):
        compute_matrix(x, f.to(torch.int16), 19.0, cotan=True)
    with pytest.raises(ValueError):
        compute_matrix(x[:, :2], f, 19.0, cotan=True)
    with pytest.raises(IndexError):
        compute_matrix(x, torch.tensor([[0, 1, len(v)]], device=DEV), 19.0, cotan=True)
    M = compute_matrix(x, f, 19.0, cotan=True)
    with pytest.raises(TypeError):
        to_differential(M, x.double())
    with pytest.raises(RuntimeError):
        spmm_grad_values(M, v.cpu(), v)
    # float64 positions are assembled in float32, as without a graph, and get a float64 gradient
    x64 = v.double().requires_grad_(True)
    compute_matrix(x64, f, 19.0, cotan=True).values().sum().backward()
    assert x64.grad.dtype == torch.float64 and torch.isfinite(x64.grad).all()
