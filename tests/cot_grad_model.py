"""float64 numpy model of the cotangent assembly's gradient (csrc/ls_assemble.cu, ls_laplacian_cot_bwd_f32) and of the
products taken with the matrix, written from the reference's formulas (largesteps/geometry.py:3-63, 96-133).  It is the
oracle of the GPU tests on meshes too large for a golden fixture; tests/test_cot_grad_model.py pins it to the reference's
float64 gradients in tests/golden/cot_grad.npz."""
import os

import numpy as np


def _faces(verts, faces):
    v = np.asarray(verts, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64)
    p = [v[f[:, a]] for a in range(3)]
    e = [p[1] - p[2], p[0] - p[2], p[0] - p[1]]        # lengths A, B, C (geometry.py:25-27)
    l = [np.linalg.norm(x, axis=1) for x in e]
    s = 0.5 * (l[0] + l[1] + l[2])
    t = [s - x for x in l]
    P = s * t[0] * t[1] * t[2]
    area = np.sqrt(np.maximum(P, 1e-12))                # geometry.py:33
    sq = [x * x for x in l]
    num = [sq[1] + sq[2] - sq[0], sq[0] + sq[2] - sq[1], sq[0] + sq[1] - sq[2]]
    return f, e, l, s, t, P, area, num


def laplacian(verts, faces):
    """The cotangent Laplacian, coalesced: (rows, cols, vals float64), the diagonal always present."""
    V = len(verts)
    f, _, _, _, _, _, area, num = _faces(verts, faces)
    r, c, w = [np.arange(V)], [np.arange(V)], [np.zeros(V)]
    for k in range(3):
        i, j, wk = f[:, (k + 1) % 3], f[:, (k + 2) % 3], num[k] / area / 4
        r += [i, j, i, j]
        c += [j, i, i, j]
        w += [-wk, -wk, wk, wk]
    key = np.concatenate(r) * V + np.concatenate(c)
    ukey, inv = np.unique(key, return_inverse=True)
    vals = np.zeros(len(ukey))
    np.add.at(vals, inv, np.concatenate(w))
    return ukey // V, ukey % V, vals


def matrix(verts, faces, shift, scale):
    """M = shift I + scale L on L's pattern."""
    rows, cols, vals = laplacian(verts, faces)
    return rows, cols, scale * vals + shift * (rows == cols)


def cot_vjp(verts, faces, rows, cols, gval, scale):
    """d(sum_e gval[e] M.values[e]) / d verts, (V, 3) float64, for M = shift I + scale L on the coalesced pattern (rows, cols)."""
    V = len(verts)
    key = np.asarray(rows, np.int64) * V + np.asarray(cols, np.int64)
    gval = np.asarray(gval, dtype=np.float64)

    def G(i, j):
        pos = np.searchsorted(key, i * V + j)
        assert np.array_equal(key[pos], i * V + j)
        return gval[pos]

    f, e, l, s, t, P, area, num = _faces(verts, faces)
    gsq, garea = [0.0, 0.0, 0.0], 0.0
    for k in range(3):
        i, j = f[:, (k + 1) % 3], f[:, (k + 2) % 3]
        wbar = np.where(i == j, 0.0, scale * (G(i, i) + G(j, j) - G(i, j) - G(j, i)))
        gnum = wbar / 4 / area
        garea = garea - gnum * num[k] / area
        gsq[(k + 1) % 3] = gsq[(k + 1) % 3] + gnum
        gsq[(k + 2) % 3] = gsq[(k + 2) % 3] + gnum
        gsq[k] = gsq[k] - gnum
    gl = [2 * gsq[k] * l[k] for k in range(3)]
    gP = np.where(P >= 1e-12, garea / (2 * area), 0.0)   # the clamp passes the gradient where P >= 1e-12
    gt = [gP * s * t[1] * t[2], gP * s * t[0] * t[2], gP * s * t[0] * t[1]]
    gs = gP * t[0] * t[1] * t[2] + gt[0] + gt[1] + gt[2]
    gv = np.zeros((V, 3))
    with np.errstate(invalid="ignore", divide="ignore"):
        ge = [(gl[k] + 0.5 * gs - gt[k])[:, None] * np.where(l[k][:, None] == 0, 0.0, e[k] / l[k][:, None]) for k in range(3)]
    for a, contrib in ((0, ge[1] + ge[2]), (1, ge[0] - ge[2]), (2, -ge[0] - ge[1])):
        np.add.at(gv, f[:, a], contrib)
    return gv


def spmm_grad_values(rows, cols, gy, x):
    """gval[e] = sum_k gy[row_e, k] x[col_e, k]: the gradient of (A @ x) w.r.t. A's values, float64."""
    return (np.asarray(gy, np.float64)[rows] * np.asarray(x, np.float64)[cols]).sum(axis=1)


def loss_grad(verts, faces, loss, W=None, G=None):
    """Gradient w.r.t. verts of the losses of tests/golden/make_golden_cot.py, float64."""
    v = np.asarray(verts, dtype=np.float64)
    V = len(v)
    if loss in ("l19", "a095"):
        scale = 19.0 if loss == "l19" else 0.95
        rows, cols, _ = laplacian(verts, faces)
        return cot_vjp(verts, faces, rows, cols, W, scale)
    import scipy.sparse as sp
    scale = 19.0 if loss == "td" else 1.0
    rows, cols, vals = matrix(verts, faces, 1.0 if loss == "td" else 0.0, scale)
    A = sp.csr_matrix((vals, (rows, cols)), shape=(V, V))
    Av = A @ v
    if loss == "td":
        gy, direct = np.asarray(G, np.float64), 0.0
    elif loss == "reg_bi":
        gy, direct = 2 * Av / Av.size, 0.0
    else:
        gy, direct = v / Av.size, Av / Av.size
    return cot_vjp(verts, faces, rows, cols, spmm_grad_values(rows, cols, gy, v), scale) + A.T @ gy + direct


def golden_mesh(golden, name):
    """(verts float32, faces int64) of mesh `name` of tests/golden/cot_grad.npz; the bunny is bunny_mesh.npz's."""
    if name == "bunny":
        d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bunny_mesh.npz"))
        return d["verts"], d["faces"].astype(np.int64)
    return golden[f"{name}.verts"], golden[f"{name}.faces"]


def golden_weights(golden, name, loss):
    """The seeded integer weights of a loss as float32: W (nnz,) for l19 / a095, G (V, 3) for td, else None."""
    if loss in ("l19", "a095"):
        return golden[f"{name}.{loss}.W"].astype(np.float32)
    return golden[f"{name}.G"].astype(np.float32) if loss == "td" else None
