"""CPU: tests/glue_model.py against the reference's own numbers in tests/golden/glue.npz -- the float64 loss and gradient of
the loop's glue, and the float32 forwards."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_l2
import glue_model as M


@pytest.fixture(scope="module")
def glue():
    return np.load(os.path.join(GOLDEN, "glue.npz"))


@pytest.mark.parametrize("mesh", ["ico2", "bunny"])
def test_float64_loss_and_gradient(glue, mesh):
    g = glue
    args = (g[f"{mesh}.v_unique"], g[f"{mesh}.f_unique"], g[f"{mesh}.dup"], g[f"{mesh}.W1"], g[f"{mesh}.W2"], g[f"{mesh}.W3"])
    loss, grad, _, _ = M.loop_loss(*args)
    ref = float(g[f"{mesh}.f64.loss"])
    assert abs(loss - ref) <= 1e-10 * abs(ref), (loss, ref)
    assert rel_l2(grad, g[f"{mesh}.f64.grad"]) < 1e-10


@pytest.mark.parametrize("mesh", ["ico2", "bunny"])
def test_float32_forwards(glue, mesh):
    g = glue
    v, f, dup = g[f"{mesh}.v_unique"], g[f"{mesh}.f_unique"], g[f"{mesh}.dup"]
    x, ft = torch.from_numpy(v), torch.from_numpy(f)
    fn = M.face_normals(x, ft)
    n = M.vertex_normals(x, ft, fn)
    eps = np.finfo(np.float32).eps
    # unit vectors: a few float32 roundings of 1 apart
    np.testing.assert_allclose(fn.numpy(), g[f"{mesh}.f32.face_normals"], rtol=0, atol=8 * eps)
    np.testing.assert_allclose(n.numpy(), g[f"{mesh}.f32.vertex_normals"], rtol=0, atol=16 * eps)
    np.testing.assert_array_equal(M.gather(n, dup).numpy(), n.numpy()[dup])
    np.testing.assert_allclose(M.gather(n, dup).numpy(), g[f"{mesh}.f32.n_opt"], rtol=0, atol=16 * eps)


def test_parts_are_consistent(glue):
    """The split VJP adds up to the loop's gradient: face-normal path (through g_fn) + angle path + gathers."""
    g = glue
    v, f, dup = g["ico2.v_unique"], g["ico2.f_unique"], g["ico2.dup"]
    W1, W2, W3 = g["ico2.W1"], g["ico2.W2"], g["ico2.W3"]
    _, grad, fn, _ = M.loop_loss(v, f, dup, W1, W2, W3)
    gout = np.zeros((len(v), 3))
    np.add.at(gout, dup, W2.astype(np.float64))
    p = M.vertex_normal_paths(v, f, fn, gout)
    _, g_face = M.face_normal_vjp(v, f, W3.astype(np.float64) + p["g_fn"])
    g_gather = np.zeros((len(v), 3))
    np.add.at(g_gather, dup, W1.astype(np.float64))
    assert rel_l2(g_face + p["g_angle"] + g_gather, grad) < 1e-12
    # the norms are those of the three edge fields
    fl = f.astype(np.int64)
    v64 = v.astype(np.float64)
    e = [v64[fl[:, 1]] - v64[fl[:, 0]], v64[fl[:, 2]] - v64[fl[:, 0]], v64[fl[:, 2]] - v64[fl[:, 1]]]
    np.testing.assert_allclose(p["norms"], [np.linalg.norm(x) for x in e], rtol=1e-14)
