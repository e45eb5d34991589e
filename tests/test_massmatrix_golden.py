"""CPU: tests/golden/mass.npz (the reference's massmatrix_voronoi, scripts/geometry.py:35-89, run by make_golden_mass.py) is
self-consistent: the Voronoi areas add up to the surface area, the reference's float32 and float64 runs agree, and the
degenerate mesh has NaN exactly where the reference puts it."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN, rel_l2
from largesteps_b200 import meshops

MESHES = ["ico2", "bunny", "grid", "plane"]


@pytest.fixture(scope="module")
def mass():
    return np.load(os.path.join(GOLDEN, "mass.npz"))


def surface_area(v, f):
    v = v.astype(np.float64)
    return 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1).sum()


def test_fixture_is_small_and_complete(mass):
    assert os.path.getsize(os.path.join(GOLDEN, "mass.npz")) < 1 << 20
    for m in MESHES + ["degen"]:
        V = len(mass[f"{m}.verts"])
        assert mass[f"{m}.faces"].dtype == np.int64 and mass[f"{m}.verts"].dtype == np.float32
        assert mass[f"{m}.f32.mass"].shape == (V,) and mass[f"{m}.f64.grad"].shape == (V, 3) and mass[f"{m}.W"].shape == (V,)


@pytest.mark.parametrize("mesh", MESHES)
def test_mass_sums_to_the_surface_area(mass, mesh):
    area = surface_area(mass[f"{mesh}.verts"], mass[f"{mesh}.faces"])
    assert abs(mass[f"{mesh}.f64.mass"].sum() - area) <= 1e-9 * area
    assert abs(mass[f"{mesh}.f32.mass"].astype(np.float64).sum() - area) <= 1e-5 * area
    assert (mass[f"{mesh}.f32.mass"] > 0).all()


@pytest.mark.parametrize("mesh", MESHES)
def test_float32_and_float64_runs_agree(mass, mesh):
    assert rel_l2(mass[f"{mesh}.f32.mass"], mass[f"{mesh}.f64.mass"]) < 1e-6
    assert np.isfinite(mass[f"{mesh}.f64.grad"]).all()
    assert rel_l2(mass[f"{mesh}.f32.grad"], mass[f"{mesh}.f64.grad"]) < 1e-5


def test_meshes_cover_the_override_branches(mass):
    def cosines(m):
        v, f = mass[f"{m}.verts"].astype(np.float64), mass[f"{m}.faces"]
        l = np.stack([np.linalg.norm(v[f[:, (k + 1) % 3]] - v[f[:, (k + 2) % 3]], axis=1) for k in range(3)], 1)
        return np.stack([(l[:, (k + 1) % 3] ** 2 + l[:, (k + 2) % 3] ** 2 - l[:, k] ** 2) / (2 * l[:, (k + 1) % 3] * l[:, (k + 2) % 3])
                         for k in range(3)], 1)
    c = cosines("grid")
    assert ((c == 0).sum(axis=1) == 1).all()                   # one exact right angle per face, at every corner position
    assert all((c[:, k] == 0).any() for k in range(3))
    c = cosines("plane")
    assert (c < 0).any(axis=1).sum() > 10                      # obtuse faces
    assert (np.abs(c).min(axis=1) < 1e-2).sum() > 10           # near-right faces


def test_degenerate_mesh(mass):
    m32, g64 = mass["degen.f32.mass"], mass["degen.f64.grad"]
    np.testing.assert_array_equal(np.nonzero(np.isnan(m32))[0], [0, 2])          # face [0, 0, 2]: zero-length edge
    np.testing.assert_array_equal(np.nonzero(np.isnan(mass["degen.f64.mass"]))[0], [0, 2])
    assert m32[3] == 0.0 and m32[7] == 0.0                      # only in the collinear face; isolated
    np.testing.assert_array_equal(np.nonzero(~np.isfinite(g64).all(axis=1))[0], [0, 2, 3, 4, 5])
    np.testing.assert_array_equal(g64[7], 0.0)


def test_safe_acos():
    x = torch.tensor([-2.0, -1.0, 0.25, 1.0, 3.0])
    assert torch.equal(meshops.safe_acos(x), torch.acos(x.clamp(-1, 1)))
