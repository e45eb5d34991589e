"""torch model (CPU, any dtype) of the loop glue in csrc/ls_glue.cu, written from the reference's formulas
(scripts/geometry.py:91-147, scripts/main.py:176-180): face normals, vertex normals with the global edge-field norms, and
the row gather.  Gradients come from autograd.  In float64 it is the oracle of tests/test_glue_host.py and
tests/test_gpu_glue_paths.py; run in float32 it measures the rounding error a float32 evaluation of the same formulas
makes, which scales their bounds.  tests/test_glue_model.py pins it to the reference's numbers in tests/golden/glue.npz."""
import numpy as np
import torch

# corner i of a face divides d0 = v[i+1] - v[i] by A_i and d1 = v[i+2] - v[i] by B_i, where A_i and B_i are two of the
# global norms N = (|E01|, |E02|, |E12|) of the edge fields E01 = v1 - v0, E02 = v2 - v0, E12 = v2 - v1
CORNER_A = (0, 2, 1)
CORNER_B = (1, 0, 2)


def as_tensor(x, dtype):
    return x.to(dtype) if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x)).to(dtype)


def gather(x, idx):
    return x[torch.as_tensor(idx).long()]


def face_normals(verts, faces):
    """(3, F): c / |c| with c = (v1 - v0) x (v2 - v0)."""
    f = faces.long()
    v0, v1, v2 = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    c = torch.linalg.cross(v1 - v0, v2 - v0, dim=1)
    return (c / c.norm(dim=1, keepdim=True)).T


def edge_norms(verts, faces):
    """The three global Frobenius norms (|E01|, |E02|, |E12|)."""
    f = faces.long()
    v0, v1, v2 = verts[f[:, 0]], verts[f[:, 1]], verts[f[:, 2]]
    return torch.stack([(v1 - v0).square().sum().sqrt(), (v2 - v0).square().sum().sqrt(), (v2 - v1).square().sum().sqrt()])


def corner_cos(verts, faces, norms):
    """(F, 3): q = d0 . d1 per corner, d0 and d1 divided by the corner's global norms."""
    f = faces.long()
    q = []
    for i in range(3):
        pi, pj, pk = verts[f[:, i]], verts[f[:, (i + 1) % 3]], verts[f[:, (i + 2) % 3]]
        q.append(((pj - pi) / norms[CORNER_A[i]] * ((pk - pi) / norms[CORNER_B[i]])).sum(1))
    return torch.stack(q, 1)


def vertex_normals(verts, faces, fn, parts=None):
    """(V, 3): N_v = sum over the corners at v of fn * acos(clamp(q, -1, 1)), n_v = N_v / |N_v|.  `parts`, a dict, receives
    the intermediate tensors (norms, q, theta, N)."""
    norms = edge_norms(verts, faces)
    q = corner_cos(verts, faces, norms)
    theta = torch.acos(q.clamp(-1, 1))
    f = faces.long()
    N = torch.zeros((verts.shape[0], 3), dtype=verts.dtype)
    for i in range(3):
        N = N.index_add(0, f[:, i], fn.T * theta[:, i:i + 1])
    if parts is not None:
        parts.update(norms=norms, q=q, theta=theta, N=N)
    return N / N.norm(dim=1, keepdim=True)


def vertex_normal_paths(verts, faces, fn, gout, dtype=torch.float64):
    """The vector-Jacobian product of compute_vertex_normals for the cotangent gout, split as the kernels split it.

    Returns a dict of numpy arrays: n (V, 3); g_fn (3, F), the gradient reaching the face normals; g_angle (V, 3), the
    gradient reaching the positions through the corner angles with fn held constant; norms, the three global norms; and T,
    the three sums T_i = sum_f g_q(f, i) q(f, i) of the backward's first pass."""
    x = as_tensor(verts, dtype).requires_grad_(True)
    fnt = as_tensor(fn, dtype).requires_grad_(True)
    f = as_tensor(faces, torch.int64)
    parts = {}
    n = vertex_normals(x, f, fnt, parts)
    parts["q"].retain_grad()
    (n * as_tensor(gout, dtype)).sum().backward()
    q = parts["q"]
    T = (q.grad * q.detach()).sum(0)
    return dict(n=n.detach().numpy(), g_fn=fnt.grad.numpy(), g_angle=x.grad.numpy(), norms=parts["norms"].detach().numpy(),
                T=T.numpy())


def face_normal_vjp(verts, faces, gn, dtype=torch.float64):
    """(fn (3, F), d(sum gn * fn) / d verts (V, 3))."""
    x = as_tensor(verts, dtype).requires_grad_(True)
    fn = face_normals(x, as_tensor(faces, torch.int64))
    (fn * as_tensor(gn, dtype)).sum().backward()
    return fn.detach().numpy(), x.grad.numpy()


def loop_loss(verts, faces, dup, W1, W2, W3, dtype=torch.float64):
    """The loop's glue under the loss sum(W1 v_opt) + sum(W2 n_opt) + sum(W3 fn) (scripts/main.py:176-180), with
    v_opt = x[dup], n_opt = n[dup].  Returns (loss, grad (V, 3), fn, n) as numpy."""
    x = as_tensor(verts, dtype).requires_grad_(True)
    f = as_tensor(faces, torch.int64)
    d = as_tensor(dup, torch.int64)
    fn = face_normals(x, f)
    n = vertex_normals(x, f, fn)
    loss = (gather(x, d) * as_tensor(W1, dtype)).sum() + (gather(n, d) * as_tensor(W2, dtype)).sum() \
        + (fn * as_tensor(W3, dtype)).sum()
    loss.backward()
    return loss.item(), x.grad.numpy(), fn.detach().numpy(), n.detach().numpy()


# ---- meshes on which the paths differ in kind ------------------------------------------------------------------------------
def small_meshes():
    """name -> (verts float32 (V, 3), faces int64 (F, 3)).  With F <= 20 the global norms are of the order of one edge, so
    the corner angles are far from pi/2 and the angle path is as large as the others; on one triangle every vertex normal
    is the face normal, so the angle path is exactly zero; 'isolated' has a vertex that no face uses."""
    from largesteps_b200 import workloads
    iv, if_ = workloads.icosahedron()
    out = {
        "triangle": ([[0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [0.3, 0.8, 0.2]], [[0, 1, 2]]),
        "two_triangles": ([[0.0, 0.0, 0.0], [1.0, 0.0, 0.0], [0.4, 0.9, 0.1], [0.5, -0.7, 0.6]], [[0, 1, 2], [1, 0, 3]]),
        "tetrahedron": ([[0.0, 0.0, 0.0], [1.0, 0.1, 0.0], [0.1, 0.9, 0.05], [0.2, 0.15, 1.1]],
                        [[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]]),
        "icosahedron": (iv, if_),
        "isolated": (np.concatenate([iv, [[2.0, 0.0, 0.0]]]), if_),
    }
    return {k: (np.asarray(v, np.float32), np.asarray(f, np.int64)) for k, (v, f) in out.items()}
