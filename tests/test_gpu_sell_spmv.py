"""GPU: the solver's stand-alone SpMM, y = A x and the p.Ap epilogue, row by row against an exact model, for every launch
variant and column count.

This engine (csrc/ls_sell_kernel.cuh, launched by launch_spmm / launch_sell_tma in csrc/ls_pcg.cu) is the graph-mode
solver's SpMV and the kernel behind bench.py's HBM figure of record.  The test reads what those very launches write: the
input goes in with PCGSolver.spmv_put, the launches are the timing harness's own (solvers.bench_kernels, bench_spmm), the
output comes back with PCGSolver.spmv_get.  spmv_put sets the output rows and the dot products to NaN, so a row that a
launch skips cannot pass on a previous launch's value.

  * SELL-32 engine, bitwise: every SELL kernel (register prefetch, or TMA with any ring depth, warps per CTA, CTAs per SM,
    with or without programmatic dependent launch) runs each row as one fmaf chain over the row's entries and then its slice
    padding {own row, 0.0f}; oracle.sell_spmv_f32 is that chain on the CPU (pinned in rational arithmetic by
    tests/test_sell_model.py), so y must equal it bit for bit, per column.
  * Rounding bound, every engine: |y_i - (A x)_i| <= gamma_{w_i} (|A| |x|)_i row by row, fp64 reference, gamma_n = n u /
    (1 - n u), u = 2^-24, w_i the row's padded width (the CSR row length for the CSR engine).
  * CSR engine (spmm_tma_kernel): it also sums each row in CSR order with one fmaf per entry; its passes pad with
    {own row, 0.0f} at other places than the SELL copy, which can only change the sign of a zero, so y equals the same model
    as a float (-0 == +0).
  * Dot: ctrl->pAp[k] against the fp64 sum of x_ik y_ik over the device's own y, to 1e-9 of sum |x_ik y_ik| (every product is
    exact in fp64); bitwise the same after repeated launches (the grid reduction's ticket is reset) and after launches with
    another column count on the same handle.

The right-hand sides are random-normal: a smooth one would hide a wrong neighbour."""
import math
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import oracle
from largesteps_b200 import workloads
from largesteps_b200.geometry import compute_matrix, csr_of, order_of
from largesteps_b200.solvers import PCGSolver, bench_kernels
from gpu_util import DEV, fan_mesh, to_dev
from test_gpu_pattern_share import with_isolated

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24

# LS_SELL_TMA -> (warps per CTA, ring depth, CTAs per SM) of spmm_sell_tma_kernel (launch_sell_tma, csrc/ls_pcg.cu); 0 is the
# register-prefetch spmm_sell_kernel; >= 10: the same kernel launched without programmatic dependent launch.  2 and 4 .. 7
# exist for K = 3 only (other K take the 32 x 2 x 1 kernel).
TMA_GEOM = {1: (32, 3, 1), 2: (24, 4, 1), 3: (32, 2, 1), 4: (16, 6, 1), 5: (16, 3, 2), 6: (24, 2, 2), 7: (16, 2, 2),
            13: (32, 2, 1)}
VARIANTS = {3: (0, 1, 2, 3, 4, 5, 6, 7, 13), 1: (0, 1, 3, 13), 2: (0, 1, 3, 13), 4: (0, 1, 3, 13)}
RELOAD = 33               # a warp re-reads its window of 32 slice offsets from its 33rd slice on


def _bunny(levels):
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "bunny_mesh.npz"))
    v, f = d["verts"], d["faces"].astype(np.int64)
    for _ in range(levels):
        v, f = workloads.subdivide(v, f)
    return v.astype(np.float32), f


def one_triangle():
    return np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float32), np.array([[0, 1, 2]], np.int64)


UNI = dict(lambda_=1.0, alpha=0.95)           # bench.py's plane workloads
MESHES = {
    "triangle": lambda: (*one_triangle(), dict(lambda_=10.0)),                  # one slice of 3 rows, one CTA
    "ico1": lambda: (*workloads.icosphere(1), dict(lambda_=10.0)),              # 42 rows: a partial second slice, grid < SMs
    "fan": lambda: (*fan_mesh(100), dict(lambda_=10.0)),                        # a 101-entry row: columns past a ring slot's 8
    "bunny": lambda: (*_bunny(1), dict(lambda_=19.0, cotan=True)),              # irregular widths around 8
    "bunny2": lambda: (*_bunny(2), dict(lambda_=19.0, cotan=True)),             # BASELINE config 2, 52786 rows
    "isolated": lambda: (*with_isolated(*workloads.icosphere(4)), dict(lambda_=10.0)),   # rows with only a diagonal
    "shuffled": lambda: (*workloads.shuffle_vertices(*workloads.plane(100, seed=3)), UNI),   # re-ordered copy (forced)
    "plane300": lambda: (*workloads.plane(300, seed=1), UNI),
    "plane1000": lambda: (*workloads.plane(1000, seed=0), UNI),                 # bench.py's workload
    "plane2000": lambda: (*workloads.plane(2000, seed=0), UNI),                 # bench.py's 4e6-row SpMV
    "plane2200": lambda: (*workloads.plane(2200, seed=0), UNI),                 # > 32 slices per warp: the window reload
    "plane2600": lambda: (*workloads.plane(2600, seed=0), UNI),                 # ... also at 24 warps x 2 CTAs per SM
    "fan3000": lambda: (*fan_mesh(3000), dict(lambda_=10.0)),                   # no SELL copy (padding over capacity): CSR
}

ENV_KEYS = ("LS_PCG_MODE", "LS_PCG_CLUSTER", "LS_PCG_RES", "LS_PCG_ONECTA", "LS_PCG_CLRES", "LS_PCG_SMALLCTA", "LS_PCG_PATTERN",
            "LS_PCG_PROFILE", "LS_PCG_CHEB_M", "LS_SPMM_ENGINE", "LS_SELL_TMA", "LS_SELL_PF", "LS_FORCE_REORDER")


def set_env(monkeypatch, env):
    for k_ in ENV_KEYS:
        monkeypatch.delenv(k_, raising=False)
    for k_, v_ in env.items():
        monkeypatch.setenv(k_, v_)


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


class System:
    """M on the device and the CSR the solver received (caller's numbering) on the host, with the model's results"""

    def __init__(self, name):
        v, f, kw = MESHES[name]()
        self.name = name
        self.M = compute_matrix(*to_dev(v, f), **kw)
        rowptr, col, val = (a.cpu().numpy() for a in csr_of(self.M))
        self.V = int(self.M.shape[0])
        self.A = sp.csr_matrix((val, col, rowptr), shape=(self.V, self.V))
        order = order_of(self.M)
        self.perm = None if order is None else order.cpu().numpy().astype(np.int64)
        self._x, self._model, self._ref = {}, {}, {}

    def x(self, k, seed=0):
        if (k, seed) not in self._x:
            self._x[(k, seed)] = np.random.default_rng(1000 * seed + k).normal(size=(self.V, k)).astype(np.float32)
        return self._x[(k, seed)]

    def copy(self, reordered):
        """the matrix copy the device holds, its row numbering: A, or P A P^T with each row sorted by new column
        (k_perm_rows), and perm[new] = old"""
        if not reordered:
            return self.A, None
        assert self.perm is not None
        Ap = self.A[self.perm][:, self.perm].tocsr()
        Ap.sort_indices()
        return Ap, self.perm

    def model(self, k, reordered, seed=0):
        """(exact SELL-32 result, padded width of every row), both in the caller's numbering"""
        key = (k, reordered, seed)
        if key not in self._model:
            A, perm = self.copy(reordered)
            x = self.x(k, seed)
            xs = x if perm is None else x[perm]
            y = oracle.sell_spmv_f32(A.indptr, A.indices, A.data, xs)
            w = oracle.sell32(A.indptr, A.indices)
            if perm is not None:
                y_, w_ = np.empty_like(y), np.empty_like(w)
                y_[perm], w_[perm] = y, w
                y, w = y_, w_
            self._model[key] = (y, w)
        return self._model[key]

    def ref(self, k, seed=0):
        """(A x, |A| |x|) in fp64"""
        if (k, seed) not in self._ref:
            A64, x64 = self.A.astype(np.float64), self.x(k, seed).astype(np.float64)
            self._ref[(k, seed)] = (A64 @ x64, abs(A64) @ np.abs(x64))
        return self._ref[(k, seed)]


_cache = {}


def system(name):
    if name not in _cache:
        _cache.clear()
        _cache[name] = System(name)
    return _cache[name]


# ---------------------------------------------------------------- checks (each returns a list of failure strings)
def bitwise(tag, y, ym):
    bad = np.flatnonzero((bits(y) != bits(ym)).any(axis=1))
    return [f"{tag}: {bad.size} rows differ from the exact model, first {bad[:6].tolist()}"] if bad.size else []


def rounding_bound(tag, sysm, k, w, y, seed=0):
    """|y - A x| <= gamma_w (|A| |x|), row by row and column by column (NaN fails)"""
    ref, mag = sysm.ref(k, seed)
    wu = w.astype(np.float64)[:, None] * U32
    err = np.abs(y.astype(np.float64) - ref)
    bad = np.flatnonzero((~(err <= wu / (1.0 - wu) * mag)).any(axis=1))
    return [f"{tag}: {bad.size} rows outside the rounding bound, first {bad[:6].tolist()}"] if bad.size else []


def dot_check(tag, x, y, dot):
    p = x.astype(np.float64) * y.astype(np.float64)      # exact
    ref, scale = p.sum(axis=0), np.abs(p).sum(axis=0)
    if not (np.abs(dot - ref) <= 1e-9 * scale).all():
        return [f"{tag}: dot {dot.tolist()} vs fp64 {ref.tolist()} (scale {scale.tolist()})"]
    return []


def launch(s, k, which, n=1):
    """`n` launches of the timing harness (which 0: SpMM + p.Ap, 4: SpMM without the epilogue; 'spmm': ls_pcg_bench_spmm)"""
    if which == "spmm":
        s.bench_spmm(k, n)
    else:
        bench_kernels([s], which, n, k=k)


def run(s, k, x, which, n=1):
    s.spmv_put(t(x))
    launch(s, k, which, n)
    y, dot = s.spmv_get(k)
    return y.cpu().numpy(), dot.cpu().numpy()


def slices_per_warp(nslices, sms, nw, minb):
    """most slices any warp of spmm_sell_tma_kernel owns: grid min(nslices, SMs x MINB), contiguous chunks per CTA, warps
    interleaved over the chunk (launch_sell_tma_t, ls_sell_kernel.cuh)"""
    G = max(1, min(nslices, sms * minb))
    return max(math.ceil((nslices * (c + 1) // G - nslices * c // G) / nw) for c in range(G))


def sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def check_variant(sysm, variant, ks, fails, env=None, expect_reordered=None, record=None):
    """one handle built with LS_SELL_TMA = variant: every k of `ks` through which 0, 4 and ls_pcg_bench_spmm, repeated
    launches, and the first k again after the others"""
    s = PCGSolver(sysm.M)
    d = s.describe()
    assert d["sell_engine"] in (1, 2), d                     # the SELL-32 engine (1: general, 2: the pattern copy beside it)
    reordered = bool(d["reordered"])
    if expect_reordered is not None:
        assert reordered == expect_reordered, d
    tma = variant % 10 != 0
    first = None
    for k in ks:
        tag = f"{sysm.name} LS_SELL_TMA={variant}{' ' + str(env) if env else ''} k={k}"
        x = sysm.x(k)
        ym, w = sysm.model(k, reordered)
        y0, dot0 = run(s, k, x, 0)
        fails += bitwise(tag + " which=0", y0, ym)
        fails += rounding_bound(tag + " which=0", sysm, k, w, y0)
        fails += dot_check(tag + " which=0", x, y0, dot0)
        # repeated launches: the same y and dot bits (a ticket left non-zero would leave the dot at NaN)
        y1, dot1 = run(s, k, x, 0, n=3)
        if not (np.array_equal(bits(y1), bits(y0)) and np.array_equal(dot1.view(np.uint64), dot0.view(np.uint64))):
            fails.append(f"{tag}: 3 launches differ from 1 (dot {dot1.tolist()} vs {dot0.tolist()})")
        # without the epilogue (DOT = false for K = 3 on the TMA kernel: the dot stays unwritten), and the profiling entry
        y4, dot4 = run(s, k, x, 4)
        fails += bitwise(tag + " which=4", y4, ym)
        if np.isnan(dot4).all() != (k == 3 and tma):
            fails.append(f"{tag} which=4: dot {dot4.tolist()}: the {'DOT=false' if k == 3 and tma else 'DOT=true'} kernel did not run")
        y5, dot5 = run(s, k, x, "spmm")
        fails += bitwise(tag + " bench_spmm", y5, ym)
        if not np.array_equal(dot5.view(np.uint64), dot0.view(np.uint64)):
            fails.append(f"{tag} bench_spmm: dot {dot5.tolist()} vs {dot0.tolist()}")
        if first is None:
            first = (k, x, y0, dot0)
    if len(ks) > 1:   # after launches with other column counts (other partial layouts) on the same handle
        k, x, y0, dot0 = first
        y, dot = run(s, k, x, 0)
        if not (np.array_equal(bits(y), bits(y0)) and np.array_equal(dot.view(np.uint64), dot0.view(np.uint64))):
            fails.append(f"{sysm.name} LS_SELL_TMA={variant} k={k} after k={list(ks[1:])}: y or dot changed")
    if record is not None and tma:
        nw, _, minb = TMA_GEOM[variant]
        record[variant] = slices_per_warp((sysm.V + 31) // 32, sms(), nw, minb)
    del s


def variant_plan():
    """(variant, column counts) for a full sweep: every variant at k = 3, the ones with other instantiations at k = 1, 2, 4"""
    return [(v, tuple(k for k in (3, 1, 2, 4) if v in VARIANTS[k])) for v in VARIANTS[3]]


SWEEP = ["triangle", "ico1", "fan", "bunny", "isolated", "shuffled", "plane2200"]


@pytest.mark.parametrize("name", SWEEP)
def test_every_sell_variant_is_the_exact_model(name, monkeypatch):
    sysm = system(name)
    fails, spw = [], {}
    extra = {"LS_FORCE_REORDER": "1"} if name == "shuffled" else {}
    for variant, ks in variant_plan():
        set_env(monkeypatch, {"LS_SELL_TMA": str(variant), **extra})
        check_variant(sysm, variant, ks, fails, expect_reordered=True if name == "shuffled" else None, record=spw)
    if name == "plane2200":
        # the window reload must run: every TMA geometry whose grid leaves some warp >= 33 slices on this mesh does.  24 warps
        # x 2 CTAs per SM (variant 6) leaves 24 per warp on 132 SMs; plane2600 below covers it.
        print(f"plane2200 (V = {sysm.V}, {sms()} SMs): most slices per warp by LS_SELL_TMA: {spw}")
        for variant, n in spw.items():
            nw, _, minb = TMA_GEOM[variant]
            assert n >= RELOAD or (nw, minb) == (24, 2), (variant, n)
        assert sum(n >= RELOAD for n in spw.values()) >= 7, spw
    assert not fails, fails


def test_window_reload_at_24_warps_two_ctas_per_sm(monkeypatch):
    """LS_SELL_TMA = 6 (24 warps, 2 CTAs per SM) on a plane large enough for its warps to own more than 32 slices"""
    sysm = system("plane2600")
    fails, spw = [], {}
    set_env(monkeypatch, {"LS_SELL_TMA": "6"})
    check_variant(sysm, 6, (3,), fails, record=spw)
    print(f"plane2600 (V = {sysm.V}, {sms()} SMs): most slices per warp, LS_SELL_TMA=6: {spw[6]}")
    assert spw[6] >= RELOAD, spw
    assert not fails, fails


def test_prefetch_halo_does_not_change_a_bit(monkeypatch):
    """LS_SELL_PF = 0 (no bulk L2 prefetch of p) and a halo larger than the mesh (clamped to the vector): the same bits"""
    sysm = system("bunny2")
    fails = []
    for pf in ("0", "100000000"):
        for variant in (3, 5, 13):
            set_env(monkeypatch, {"LS_SELL_TMA": str(variant), "LS_SELL_PF": pf})
            check_variant(sysm, variant, (3, 1) if variant != 5 else (3,), fails, env={"LS_SELL_PF": pf})
    assert not fails, fails


def test_the_bench_sequence(monkeypatch):
    """bench.py's roofline launches as it issues them (time_kernels: 8 then 400 back-to-back launches from C rotating over 4
    handles of the 10^6-row plane, which = 0 and 4; one handle of the 4 10^6-row plane, which = 4), then every handle's y and
    dot are checked"""
    set_env(monkeypatch, {})
    fails = []
    sysm = system("plane1000")
    hs = [PCGSolver(sysm.M) for _ in range(4)]
    xs = [sysm.x(3, seed=i) for i in range(4)]
    single = []
    for i, (s, x) in enumerate(zip(hs, xs)):
        assert not s.describe()["reordered"]
        single.append(run(s, 3, x, 0)[1])                       # one launch alone: the dot's reference bits
    for which in (0, 4):
        for s, x in zip(hs, xs):
            s.spmv_put(t(x))
        bench_kernels(hs, which, 8)
        bench_kernels(hs, which, 400)
        torch.cuda.synchronize()
        for i, (s, x) in enumerate(zip(hs, xs)):
            tag = f"plane1000 handle {i} which={which}"
            y, dot = (a.cpu().numpy() for a in s.spmv_get(3))
            ym, w = sysm.model(3, False, seed=i)
            fails += bitwise(tag, y, ym)
            fails += rounding_bound(tag, sysm, 3, w, y, seed=i)
            if which == 0:
                fails += dot_check(tag, x, y, dot)
                if not np.array_equal(dot.view(np.uint64), single[i].view(np.uint64)):
                    fails.append(f"{tag}: dot after 102 launches {dot.tolist()} vs one launch {single[i].tolist()}")
            elif not np.isnan(dot).all():
                fails.append(f"{tag}: the dot was written")
    del hs
    sysm = system("plane2000")
    s4 = PCGSolver(sysm.M)
    x = sysm.x(3)
    s4.spmv_put(t(x))
    bench_kernels([s4], 4, 8)
    bench_kernels([s4], 4, 400)
    y, _ = (a.cpu().numpy() for a in s4.spmv_get(3))
    ym, w = sysm.model(3, bool(s4.describe()["reordered"]))
    fails += bitwise("plane2000 which=4", y, ym)
    fails += rounding_bound("plane2000 which=4", sysm, 3, w, y)
    assert not fails, fails


@pytest.mark.parametrize("name,env", [("fan3000", {}), ("bunny", {"LS_SPMM_ENGINE": "csr"}),
                                      ("plane300", {"LS_SPMM_ENGINE": "csr"})], ids=["fan3000", "bunny-csr", "plane300-csr"])
def test_csr_engine(name, env, monkeypatch):
    """the TMA-staged CSR kernel: within the rounding bound of its CSR row lengths, and equal to the model as a float"""
    set_env(monkeypatch, env)
    sysm = system(name)
    s = PCGSolver(sysm.M)
    d = s.describe()
    assert d["algo"] == "graph" and d["sell_engine"] == 0, d
    reordered = bool(d["reordered"])
    A, _ = sysm.copy(reordered)
    lens = np.diff(A.indptr)
    if reordered:
        lens_ = np.empty_like(lens)
        lens_[sysm.perm] = lens
        lens = lens_
    fails = []
    for k in (1, 2, 3, 4):
        tag = f"{name} CSR k={k}"
        x = sysm.x(k)
        ym, _ = sysm.model(k, reordered)
        for which in (0, 4, "spmm"):
            y, dot = run(s, k, x, which)
            fails += rounding_bound(f"{tag} which={which}", sysm, k, lens, y)
            if not np.array_equal(y, ym):
                bad = np.flatnonzero((y != ym).any(axis=1))
                fails.append(f"{tag} which={which}: {bad.size} rows differ from the sequential fmaf chain, first {bad[:6].tolist()}")
            fails += dot_check(f"{tag} which={which}", x, y, dot)   # the CSR engine always runs its epilogue
        y1, dot1 = run(s, k, x, 0, n=3)
        if not np.array_equal(dot1.view(np.uint64), dot.view(np.uint64)):
            fails.append(f"{tag}: 3 launches give dot {dot1.tolist()}, 1 gives {dot.tolist()}")
    if name == "fan3000":
        assert int(lens.max()) == 3001
    assert not fails, fails


@pytest.mark.parametrize("mode", ["fused", "graph"])
def test_a_handle_solves_the_same_after_the_diagnostics(mode, monkeypatch):
    """spmv_put / the launches / spmv_get overwrite the solver's p and Ap planes and its p.Ap: the next solve re-initialises
    them and returns the same bits as before"""
    set_env(monkeypatch, {"LS_PCG_MODE": "graph"} if mode == "graph" else {})
    sysm = system("bunny2")
    s = PCGSolver(sysm.M)
    assert s.describe()["algo"] == mode
    b = t(np.random.default_rng(7).normal(size=(sysm.V, 3)).astype(np.float32))
    x1 = s.solve(b).cpu().numpy()
    for k in (3, 4, 1):
        run(s, k, sysm.x(k), 0)
    x2 = s.solve(b).cpu().numpy()
    assert np.array_equal(bits(x1), bits(x2))


def test_the_spmv_diagnostics_validate_their_arguments():
    sysm = system("ico1")
    s = PCGSolver(sysm.M)
    with pytest.raises(ValueError):
        s.spmv_put(t(np.zeros((sysm.V, 5), np.float32)))
    with pytest.raises(ValueError):
        s.spmv_put(t(np.zeros((sysm.V + 1, 3), np.float32)))
    with pytest.raises(ValueError):
        s.spmv_get(0)
    for which in (-1, 1, 2, 3, 5):   # the harness launches the SpMM alone: 0 with the p.Ap epilogue, 4 without
        with pytest.raises(ValueError):
            bench_kernels([s], which, 1)
