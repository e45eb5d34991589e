"""GPU parity: massmatrix_voronoi (csrc/ls_glue.cu through largesteps_b200.meshops) against values AND gradients of the
unmodified reference (scripts/geometry.py:35-89) run on the CPU by tests/golden/make_golden_mass.py.  Values vs the
reference's own float32 run; gradients of (m * W).sum() vs its float64 run."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from largesteps_b200 import meshops
from gpu_util import DEV, fan_mesh, rel_l2

pytestmark = pytest.mark.gpu

IDX = [torch.int64, torch.int32]


@pytest.fixture(scope="module")
def mass():
    return np.load(os.path.join(GOLDEN, "mass.npz"))


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def run(g, mesh, idx_dtype):
    x = t(g[f"{mesh}.verts"]).requires_grad_(True)
    m = meshops.massmatrix_voronoi(x, t(g[f"{mesh}.faces"]).to(idx_dtype))
    (m * t(g[f"{mesh}.W"])).sum().backward()
    return m.detach(), x.grad


@pytest.mark.parametrize("mesh", ["ico2", "bunny", "grid", "plane", "degen"])
@pytest.mark.parametrize("idx_dtype", IDX)
def test_massmatrix_voronoi_matches_reference(mass, mesh, idx_dtype):
    g = mass
    m, grad = run(g, mesh, idx_dtype)
    assert m.shape == (len(g[f"{mesh}.verts"]),) and m.dtype == torch.float32
    m, grad = m.cpu().numpy(), grad.cpu().numpy()
    ref = g[f"{mesh}.f32.mass"]
    np.testing.assert_array_equal(np.isnan(m), np.isnan(ref))
    fin = ~np.isnan(ref)
    np.testing.assert_allclose(m[fin], ref[fin], rtol=0, atol=2e-6 * np.abs(ref[fin]).max())
    g64, g32 = g[f"{mesh}.f64.grad"], g[f"{mesh}.f32.grad"]
    bad = ~np.isfinite(g64).all(axis=1)
    np.testing.assert_array_equal(~np.isfinite(grad).all(axis=1), bad)
    err = rel_l2(grad[~bad], g64[~bad])
    ref_err = rel_l2(g32[~bad], g64[~bad])               # what the reference's own float32 run achieves
    print(f"{mesh}: gradient rel-L2 vs the reference's float64 run {err:.2e} (the reference's float32 run: {ref_err:.2e})")
    if mesh != "degen":
        assert not bad.any()
        assert err < max(5e-6, 20 * ref_err), (err, ref_err)


@pytest.mark.parametrize("idx_dtype", IDX)
def test_massmatrix_voronoi_is_bit_reproducible(mass, idx_dtype):
    for mesh in ("bunny", "degen"):
        m_a, g_a = run(mass, mesh, idx_dtype)
        m_b, g_b = run(mass, mesh, idx_dtype)
        assert torch.equal(m_a.view(torch.int32), m_b.view(torch.int32))     # bit patterns, NaN included
        assert torch.equal(g_a.view(torch.int32), g_b.view(torch.int32))


@pytest.mark.parametrize("idx_dtype", IDX)
def test_massmatrix_voronoi_hub_vertex(idx_dtype):
    v, f = fan_mesh(3000)
    x = t(v).requires_grad_(True)
    m = meshops.massmatrix_voronoi(x, t(f).to(idx_dtype))
    m.sum().backward()
    assert torch.isfinite(m).all() and torch.isfinite(x.grad).all()
    v64 = v.astype(np.float64)
    area = 0.5 * np.linalg.norm(np.cross(v64[f[:, 1]] - v64[f[:, 0]], v64[f[:, 2]] - v64[f[:, 0]]), axis=1).sum()
    assert abs(float(m.detach().double().sum()) - area) <= 1e-5 * area


def test_massmatrix_voronoi_edge_cases():
    v = torch.randn(10, 3, device=DEV)
    f = torch.tensor([[0, 1, 2], [2, 3, 4]], device=DEV)
    x = v.clone().requires_grad_(True)
    m = meshops.massmatrix_voronoi(x, f[:0])                      # no faces: zero mass, zero gradient
    assert torch.equal(m, torch.zeros(10, device=DEV))
    m.sum().backward()
    assert torch.equal(x.grad, torch.zeros(10, 3, device=DEV))
    assert meshops.massmatrix_voronoi(v[:0], f[:0]).shape == (0,)
    with pytest.raises(IndexError):
        meshops.massmatrix_voronoi(v, torch.tensor([[0, 1, 10]], device=DEV))
    with pytest.raises(IndexError):
        meshops.massmatrix_voronoi(v, torch.tensor([[0, -1, 2]], dtype=torch.int32, device=DEV))
    with pytest.raises(ValueError):
        meshops.massmatrix_voronoi(v[:, :2], f)
    with pytest.raises(ValueError):
        meshops.massmatrix_voronoi(v, f.reshape(-1))
    with pytest.raises(TypeError):
        meshops.massmatrix_voronoi(v.double(), f)
    with pytest.raises(TypeError):
        meshops.massmatrix_voronoi(v, f.to(torch.int16))
    with pytest.raises(RuntimeError):
        meshops.massmatrix_voronoi(v.cpu(), f)
    with pytest.raises(RuntimeError):
        meshops.massmatrix_voronoi(v, f.cpu())
