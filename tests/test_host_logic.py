"""CPU: host-side logic of the operator surface (error behaviour, caches, sharding) -- no GPU compute."""
import gc
import os
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT, PKG
from largesteps_b200 import workloads, distributed
from largesteps_b200 import geometry, parameterize, solvers, optimize


def test_reference_import_names_resolve():
    from largesteps.geometry import compute_matrix, laplacian_cot, laplacian_uniform          # noqa: F401
    from largesteps.parameterize import to_differential, from_differential                    # noqa: F401
    from largesteps.solvers import Solver, CholeskySolver, ConjugateGradientSolver, solve, DifferentiableSolve  # noqa: F401
    from largesteps.optimize import AdamUniform                                                # noqa: F401
    assert compute_matrix is geometry.compute_matrix
    assert from_differential is parameterize.from_differential


def test_alpha_validation_matches_reference(golden_assembly):
    v = torch.zeros(4, 3)
    f = torch.zeros(1, 3, dtype=torch.long)
    for bad in (1.0, -0.1, 1.5):
        with pytest.raises(ValueError) as e:
            geometry.compute_matrix(v, f, 1.0, alpha=bad)
        assert str(e.value).startswith(f"Invalid value for alpha: {bad}")
    assert str(golden_assembly["alpha_error"]) == \
        "Invalid value for alpha: 1.0 : it should take values between 0 (included) and 1 (excluded)"


def test_no_cpu_fallback():
    v = torch.zeros(4, 3)
    f = torch.tensor([[0, 1, 2]])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        geometry.compute_matrix(v, f, 1.0)
    M = torch.sparse_coo_tensor(torch.tensor([[0, 1], [0, 1]]), torch.ones(2), (2, 2)).coalesce()
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        parameterize.from_differential(M, torch.zeros(2, 3))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        parameterize.to_differential(M, torch.zeros(2, 3))
    p = torch.nn.Parameter(torch.zeros(3, 3))
    p.grad = torch.zeros(3, 3)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        optimize.AdamUniform([p]).step()


def test_unknown_method_message(golden_solve):
    M = torch.sparse_coo_tensor(torch.tensor([[0, 1], [0, 1]]), torch.ones(2), (2, 2)).coalesce()
    with pytest.raises(ValueError) as e:
        parameterize.from_differential(M, torch.zeros(2, 3), method="nope")
    assert str(e.value) == str(golden_solve["method_error"]) == "Unknown solver type 'nope'."


def test_solver_base_class_contract():
    with pytest.raises(NotImplementedError):
        solvers.Solver(None).solve(torch.zeros(1, 1))


def test_cache_is_weak_like_the_reference():
    class Dummy:
        pass
    a = Dummy()
    parameterize.cache_put(("k", "m"), "solver", a)
    assert ("k", "m") in parameterize._cache
    del a
    gc.collect()
    assert ("k", "m") not in parameterize._cache


def test_workload_sizes_match_survey():
    v, f = workloads.icosphere(4)
    assert v.shape == (2562, 3) and f.shape == (5120, 3)
    assert np.allclose(np.linalg.norm(v, axis=1), 1.0, atol=1e-6)
    v, f = workloads.plane(100, seed=0)
    assert v.shape == (10000, 3) and f.shape == (2 * 99 * 99, 3)
    e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
    E = len(np.unique(e[:, 0] * 10000 + e[:, 1]))
    assert 10000 + 2 * E == 7 * 100 * 100 - 8 * 100 + 2      # nnz(M) = 7n^2 - 8n + 2 (6992002 at n=1000)
    assert 7 * 1000 * 1000 - 8 * 1000 + 2 == 6992002


def test_bunny_subdivision_sizes(bunny_mesh):
    v, f = bunny_mesh
    assert v.shape == (3301, 3) and f.shape == (6598, 3)
    v2, f2 = workloads.subdivide(*workloads.subdivide(v, f))
    assert v2.shape[0] == 52786 and f2.shape[0] == 105568


def test_assign_round_robin():
    assert distributed.assign(8, 0, 1) == list(range(8))
    assert distributed.assign(8, 1, 2) == [1, 3, 5, 7]
    assert distributed.assign(8, 7, 8) == [7]
    assert distributed.assign(3, 3, 4) == []
    got = sorted(sum((distributed.assign(11, r, 4) for r in range(4)), []))
    assert got == list(range(11))
    with pytest.raises(ValueError):
        distributed.assign(4, 2, 2)


def _gloo_worker(rank, world, port, out_dir):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, PKG)
    import torch.distributed as dist
    import oracle
    from largesteps_b200 import workloads as W, distributed as D
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        # two independent planes, one per rank (config 4 shape, tiny): each rank solves only its own mesh
        mine = D.assign(world, rank, world)
        assert mine == [rank]
        v, f = W.plane(24, seed=rank)
        r, c, val, V = oracle.compute_matrix(v, f, 1.0, alpha=0.95)
        x = oracle.DirectSolver(r, c, val, V).solve(oracle.to_differential(r, c, val, V, v)).astype(np.float32)
        allx = D.gather_solutions(torch.from_numpy(x))
        assert allx.shape == (world, V, 3)
        t = D.max_over_ranks(1.0 + rank)
        n = D.sum_over_ranks(3)
        D.barrier()
        if rank == 0:
            np.savez(os.path.join(out_dir, "gloo.npz"), allx=allx.numpy(), t=t, n=n)
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_sharding(tmp_path):
    import torch.multiprocessing as mp
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_gloo_worker, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    d = np.load(os.path.join(str(tmp_path), "gloo.npz"))
    assert d["t"] == 2.0 and d["n"] == 6.0
    # rank r's slot holds the solution of plane(seed=r): from_differential(to_differential(v)) == v
    for r in range(2):
        v, _ = workloads.plane(24, seed=r)
        assert np.linalg.norm(d["allx"][r] - v) / np.linalg.norm(v) < 1e-5


def test_bench_reference_arm_contract():
    """`bench.py --impl reference` (the CPU arm that runs next to the GPU arm) prints one JSON line with the contract's
    keys; exercised on BASELINE config 1 so it finishes in seconds."""
    import json
    import subprocess
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "icosphere",
                          "--steps", "3", "--warmup", "1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    line = json.loads(out.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and line["metric"] == "from_differential solves/sec @1M verts"
    for key in ("value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "dtype",
                "data", "config", "cpu_baseline", "e2e"):
        assert key in line
    assert line["value"] > 0 and line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
    assert line["e2e"]["h2d_bytes_per_step"] == 0 and line["config"]["workload"] == "icosphere"
    # non-zero ranks of a torchrun launch exit quietly
    env = dict(os.environ, RANK="1", WORLD_SIZE="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--workload", "icosphere",
                          "--steps", "1"], capture_output=True, text=True, timeout=120, env=env)
    assert out.returncode == 0 and out.stdout.strip() == ""


def test_pattern_layout_model(bunny_mesh):
    """CPU model of the opt-in pattern-only matrix copy (csrc/ls_pcg.cu pat_fill_kernel + the PAT phase A of
    ls_pcg_fused.cuh): slots, self-pointing padding and the diagonal pay-back reproduce M @ p to fp32 rounding,
    including slices wider than the 4 register pairs (bunny: valence up to 10+) and narrower than 3."""
    import numpy as np
    import scipy.sparse as sp
    import oracle
    f32 = np.float32
    U = 4

    def run(v, f, lam):
        rows, cols, vals, V = oracle.compute_matrix(np.asarray(v, np.float64), np.asarray(f), lambda_=lam)
        A = sp.csr_matrix((vals.astype(f32), (rows, cols)), shape=(V, V))
        A.sort_indices()
        rp, ci, va = A.indptr, A.indices, A.data
        off = va[ci != np.repeat(np.arange(V), np.diff(rp))]
        assert off.min() == off.max()            # what pat_detect_kernel establishes (bitwise)
        c = f32(off[0])
        Vp = (V + 31) // 32 * 32
        p = np.zeros((Vp, 3), f32)
        p[:V] = np.random.default_rng(0).normal(size=(V, 3)).astype(f32)
        y = np.zeros((Vp, 3), f32)
        widths = set()
        for s in range(Vp // 32):
            rws = range(32 * s, 32 * s + 32)
            w2 = (max(int(np.sum(ci[rp[r]:rp[r + 1]] != r)) if r < V else 0 for r in rws) + 1) // 2
            widths.add(w2)
            for r in rws:
                slots, d = [], f32(0)
                if r < V:
                    for e in range(rp[r], rp[r + 1]):
                        if ci[e] == r:
                            d = va[e]
                        else:
                            slots.append(int(ci[e]))
                used = len(slots)
                slots += [r] * (2 * w2 - used)                       # unused stored slots point at the row itself ...
                dp = f32(d - c * f32(2 * w2 - used)) if r < V else f32(0)   # ... and are paid back in the diagonal
                pairs = [(slots[2 * m], slots[2 * m + 1]) for m in range(w2)]
                UB = 3 if w2 <= 3 else 4
                chunk = pairs[:UB] + [(r, r)] * (UB - min(w2, UB))   # register slots past the width: same trick
                dp = f32(dp - c * f32(2 * (UB - min(w2, UB))))
                sm = np.zeros(3, f32)
                for a, b in chunk:
                    sm = (sm + (p[a] + p[b]).astype(f32)).astype(f32)
                j = U
                while j < w2:
                    for a, b in pairs[j:j + U] + [(r, r)] * max(0, j + U - w2):
                        sm = (sm + (p[a] + p[b]).astype(f32)).astype(f32)
                    dp = f32(dp - c * f32(2 * max(0, j + U - w2)))
                    j += U
                y[r] = (dp * p[r] + c * sm).astype(f32)
        ref = A.astype(np.float64) @ p[:V].astype(np.float64)
        return np.linalg.norm(y[:V] - ref) / np.linalg.norm(ref), widths

    from largesteps_b200 import workloads
    err, widths = run(*bunny_mesh, 19.0)
    assert err < 5e-7 and max(widths) == 4
    n = 21                                            # a fan: one vertex of valence 21 -> 11 pairs, three passes of the wide-slice loop
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False)
    fv = np.vstack([[0, 0, 0], np.stack([np.cos(ang), np.sin(ang), 0 * ang], 1)])
    ff = np.array([[0, 1 + i, 1 + (i + 1) % n] for i in range(n)])
    err, widths = run(fv, ff, 3.0)
    assert err < 5e-7 and max(widths) > 2 * U
    err, widths = run(*workloads.plane(12), 5.0)
    assert err < 5e-7 and min(widths) <= 3           # exercises the 3-pair body and its pay-back


def test_meshops_and_remesh_reject_cpu_tensors_and_bad_arguments():
    """No CPU fallback anywhere: the loop glue and the re-parameteriser raise on CPU tensors, like every other operator."""
    import pytest
    import torch
    from largesteps_b200 import meshops
    from largesteps_b200.remesh import Reparameterizer, Arena
    v = torch.rand(5, 3)
    f = torch.tensor([[0, 1, 2], [2, 3, 4]])
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        meshops.compute_face_normals(v, f)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        meshops.compute_vertex_normals(v, f, torch.zeros(3, 2))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        meshops.gather_rows(v, torch.tensor([0, 1]))
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        Reparameterizer(lambda_=19.0).update(v, f)
    with pytest.raises(ValueError, match="Unknown solver type"):
        Reparameterizer(method="QR")
    # setup-time helpers are plain torch and keep the reference's semantics (scripts/geometry.py:3-35)
    vd = torch.tensor([[0., 0, 0], [1, 0, 0], [0, 1, 0], [1, 0, 0]])
    fd = torch.tensor([[0, 1, 2], [0, 2, 3]])
    vu, fu, inv = meshops.remove_duplicates(vd, fd)
    assert vu.shape == (3, 3) and torch.equal(vu[inv], vd) and torch.equal(vu[fu], vd[fd])
    assert abs(float(meshops.average_edge_length(vd, fd)) - (2 + 2 ** 0.5) / 3) < 1e-6
    a = Arena()
    with pytest.raises(MemoryError):
        a.take(16, torch.device("cpu"))
