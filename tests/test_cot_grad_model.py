"""CPU: the float64 numpy model of the cotangent assembly's gradient (tests/cot_grad_model.py), the oracle of the GPU tests
on large meshes, against the reference's own float64 gradients (tests/golden/cot_grad.npz, make_golden_cot.py), and its
matrix against the reference's float32 values."""
import os

import numpy as np
import pytest

import cot_grad_model as model
from conftest import GOLDEN, rel_l2

MESHES = ["ico2", "bunny", "grid", "plane", "degen"]
LOSSES = ["l19", "a095", "td", "reg_bi", "reg_lap"]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(GOLDEN, "cot_grad.npz"))


@pytest.mark.parametrize("mesh", MESHES)
def test_model_pattern_matches_reference(golden, mesh):
    v, f = model.golden_mesh(golden, mesh)
    rows, cols, _ = model.matrix(v, f, 1.0, 19.0)
    idx = golden[f"{mesh}.idx"]
    np.testing.assert_array_equal(rows, idx[0])
    np.testing.assert_array_equal(cols, idx[1])


@pytest.mark.parametrize("mesh", ["ico2", "bunny"])
def test_model_values_match_reference(golden_assembly, mesh):
    """The model's matrix against the reference's float32 cotangent matrices of assembly.npz (make_golden.py)."""
    g = golden_assembly
    v, f = g[f"{mesh}.verts"], g[f"{mesh}.faces"]
    for case, shift, scale in (("cot_l19", 1.0, 19.0), ("cot_a09", 0.1, 0.9)):
        rows, cols, vals = model.matrix(v, f, shift, scale)
        np.testing.assert_array_equal(np.stack([rows, cols]), g[f"{mesh}.{case}.idx"])
        ref = g[f"{mesh}.{case}.val"]
        assert np.abs(vals - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("mesh", MESHES)
def test_model_gradient_matches_reference_float64(golden, mesh, loss):
    """Against the reference's float64 gradient, which the fixture stores rounded to float32 (rel-L2 change <= 2^-24)."""
    v, f = model.golden_mesh(golden, mesh)
    w = model.golden_weights(golden, mesh, loss)
    got = model.loss_grad(v, f, loss, W=w, G=w)
    ref = golden[f"{mesh}.{loss}.grad"]
    assert np.isfinite(ref).all() and np.isfinite(got).all()
    assert rel_l2(got, ref) < 1e-7, rel_l2(got, ref)
