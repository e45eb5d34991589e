"""GPU: the TMA-staged CSR SpMM (spmm_tma_kernel, csrc/ls_spmm_kernel.cuh) row by row, at the shapes where it changes path,
in both of its layouts.

  * Public layout (ls_spmm_csr_f32, behind to_differential, parameterize.spmm and the gradient of L @ v w.r.t. v): x and y
    are (V, k) row-major with leading dimensions ldx and ldy, k > 4 runs in chunks of 4 columns, the rows are split evenly
    over the grid, and the producer warp finds the block boundaries on the fly.
  * Solver layout (the graph-mode solver's CSR engine, LS_PCG_MODE=graph LS_SPMM_ENGINE=csr): an nnz-balanced row partition
    (k_partition) and a per-CTA block plan of at most SPMM_BMAX = 64 blocks, which the producer reads from two descriptor
    registers (blocks 1..32 and 33..64).  If any CTA needs more, the whole grid runs the on-the-fly producer over the
    partition (describe()["planned"] == 0).  Input, launches and output are the timing harness's (spmv_put, bench_kernels
    which 0 and 4, bench_spmm, spmv_get), as in test_gpu_sell_spmv.py.

Value model: each row is one fmaf chain over its entries in CSR order, from 0.  oracle.sell_spmv_f32 is that chain (its
SELL padding only changes the sign of a zero when x is finite), so y must equal it as a float.  y must also be within
gamma_w (|A| |x|) of the fp64 product, row by row, w the CSR row length.

Planner model: partition() and plan() restate k_partition, spmm_block_extent and spmm_plan_kernel at the default stage
capacity: at most 256 rows per block, and a block fits when e_nz - (s_nz & ~3) <= cap - 4 with cap = 2048.  Every case
asserts that it reaches the path it was built for, and the solver's overflow bit must agree with the model.

The matrices are foreign (not built by compute_matrix): prescribed row lengths, random distinct columns, random-normal
values and, where the solver needs one, a positive diagonal.  The right-hand sides are random-normal."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import oracle
import largesteps_b200._native as N
from largesteps_b200 import workloads
from largesteps_b200.geometry import compute_matrix, csr_of
from largesteps_b200.parameterize import spmm, spmm_grad_values, to_differential
from largesteps_b200.solvers import PCGSolver
from gpu_util import DEV, to_dev
from test_gpu_sell_spmv import U32, UNI, bits, dot_check, rounding_bound, run, set_env, t

pytestmark = pytest.mark.gpu

NT, CAP, BMAX = 256, 256 * 8, 64      # SPMM_NT, the default stage capacity (LS_SPMM_CAPMUL = 8), SPMM_BMAX
FIT = CAP - 4                          # most entries a block may span from its 16-byte aligned start
DIRECT = 2100                          # a row this long never fits a stage
SOLVER = {"LS_PCG_MODE": "graph", "LS_SPMM_ENGINE": "csr"}
SENTINEL = np.uint32(0x7FC0DEAD)       # a NaN payload no kernel writes


@pytest.fixture(autouse=True)
def default_stage_config():
    # the planner model is for the default stages and capacity (spmm_config reads these once per process)
    assert not [k for k in os.environ if k.startswith("LS_SPMM_") and k != "LS_SPMM_ENGINE"], "LS_SPMM_* tuning set"


# ------------------------------------------------------------------------------------------------------------ matrices
class Foreign:
    """A (V, V) CSR with row i holding lens[i] entries: the diagonal (positive) where diag[i], and distinct random columns.
    The same matrix lives on the device as a coalesced torch sparse COO tensor."""

    def __init__(self, name, lens, diag=True, seed=0):
        lens = np.asarray(lens, np.int64)
        V = lens.shape[0]
        diag = np.broadcast_to(np.asarray(diag, bool), (V,)) & (lens > 0)
        m = lens - diag                               # off-diagonal entries per row, at offsets 1 .. V-1 from the row
        assert (m <= V - 1).all(), name
        rng = np.random.default_rng(seed)
        gmax = np.repeat((V - 1) // np.maximum(m, 1), m)
        gaps = rng.integers(1, gmax + 1)              # increasing offsets, at most m * gmax <= V - 1: distinct columns
        cs = np.cumsum(gaps)
        first = np.repeat(np.cumsum(m) - m, m)
        off = cs - (cs - gaps)[first]
        r_off = np.repeat(np.arange(V), m)
        d = np.flatnonzero(diag)
        rows = np.concatenate([d, r_off])
        cols = np.concatenate([d, (r_off + off) % V])
        vals = np.concatenate([np.abs(rng.normal(size=d.size)) + 1.0, rng.normal(size=r_off.size)]).astype(np.float32)
        o = np.argsort(rows * V + cols, kind="stable")
        rows, cols, vals = rows[o], cols[o], vals[o]
        self.name, self.V, self.lens = name, V, lens
        self.rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        self.col, self.val = cols.astype(np.int32), vals
        self.A = sp.csr_matrix((vals, cols, self.rowptr), shape=(V, V))
        self.M = torch.sparse_coo_tensor(torch.from_numpy(np.stack([rows, cols])).to(DEV), t(vals), (V, V)).coalesce()
        rp, cl, _ = csr_of(self.M)
        assert np.array_equal(rp.cpu().numpy(), self.rowptr) and np.array_equal(cl.cpu().numpy(), self.col), name
        self._x, self._ref = {}, {}

    def x(self, k, seed=0):
        if (k, seed) not in self._x:
            self._x[(k, seed)] = np.random.default_rng(1000 * seed + k).normal(size=(self.V, k)).astype(np.float32)
        return self._x[(k, seed)]

    def model(self, k, seed=0):
        return oracle.sell_spmv_f32(self.rowptr, self.col, self.val, self.x(k, seed))

    def ref(self, k, seed=0):
        """(A x, |A| |x|) in fp64"""
        if (k, seed) not in self._ref:
            A64, x64 = self.A.astype(np.float64), self.x(k, seed).astype(np.float64)
            self._ref[(k, seed)] = (A64 @ x64, abs(A64) @ np.abs(x64))
        return self._ref[(k, seed)]


def values(tag, F, k, y, seed=0):
    """y against the fmaf-chain model (as floats: +-0 may differ) and the rounding bound"""
    fails = rounding_bound(tag, F, k, F.lens, y, seed)
    bad = np.flatnonzero((y != F.model(k, seed)).any(axis=1))
    if bad.size:
        fails.append(f"{tag}: {bad.size} rows differ from the sequential fmaf chain, first {bad[:6].tolist()}")
    return fails


# ------------------------------------------------------------------------------------------------------- planner model
def partition(rowptr, G):
    """k_partition: part[c] = the first row r with 2 rowptr[r] + 5 r >= (2 nnz + 5 V) c / G, part[G] = V"""
    V = rowptr.shape[0] - 1
    w = 2 * rowptr.astype(np.int64) + 5 * np.arange(V + 1, dtype=np.int64)
    return np.append(np.searchsorted(w, w[-1] * np.arange(G, dtype=np.int64) // G, side="left"), V)


def even_split(V, G):
    """the public layout's rows of CTA c: [V c / G, V (c + 1) / G)"""
    return np.array([V * c // G for c in range(G + 1)], np.int64)


def public_grid(V):
    """spmm_grid_for: min(ceil(V / 64), SMs x CTAs per SM), so ceil(V / 64) while V <= 64 SMs"""
    assert V <= 64 * torch.cuda.get_device_properties(DEV).multi_processor_count
    return max(1, (V + 63) // 64)


def plan(rowptr, part):
    """spmm_block_extent over every CTA's rows, as spmm_plan_kernel and the on-the-fly producer walk them: per CTA the list
    of blocks (r0, nr, direct, s_nz, e_nz)"""
    rp = rowptr.tolist()
    out = []
    for c in range(len(part) - 1):
        r, r_end = int(part[c]), int(part[c + 1])
        s = rp[r] if r < r_end else 0
        blocks = []
        while r < r_end:
            nr = min(NT, r_end - r)
            e, s_a, direct = rp[r + nr], s & ~3, 0
            if e - s_a > FIT:
                lo = int(np.searchsorted(rowptr[r:r + nr + 1], s_a + FIT, side="right")) - 1   # rows that fit
                nr, direct = (1, 1) if lo == 0 else (lo, 0)
                e = rp[r + nr]
            blocks.append((r, nr, direct, s, e))
            r, s = r + nr, e
        out.append(blocks)
    return out


def block_at(blocks, r0):
    hit = [b for cta in blocks for b in cta if b[0] == r0]
    assert len(hit) == 1, (r0, hit)
    return hit[0]


# ---------------------------------------------------------------------------------------------- the cases' row lengths
def lens_stage(seed=11, G=40, Z=4400):
    """Stage-capacity edges, one group per 64-row segment, each group right after a direct row that opens the segment, so
    that it starts a block:
      rows of L entries starting at s_nz with L + (s_nz & 3) = 2043, 2044 (fit) and 2045 (a direct row), s_nz & 3 = 0..3;
      runs of 46 rows spanning exactly 2044 (one block) and 2045 entries (the last row starts the next block).
    Filler rows hold >= 2 entries, so no row can join a 2043-entry one.  Every segment holds Z entries: then k_partition's
    weights hit their targets at rows 64 c, and the solver's partition is the public layout's even split (V = 64 G).
    Returns (lens, rows [(r, off, T)], runs [(r, n, off, S)])."""
    rng = np.random.default_rng(seed)
    lens = np.zeros((G, 64), np.int64)
    groups = [("row", off, T) for off in range(4) for T in (FIT - 1, FIT, FIT + 1)] + \
             [("run", off, S) for off in range(4) for S in (FIT, FIT + 1)]
    rows, runs = [], []
    for c in range(G):
        seg = lens[c]
        used = 0
        if 1 <= c <= len(groups):
            kind, off, T = groups[c - 1]
            seg[0] = DIRECT + (off - DIRECT) % 4            # c Z = 0 mod 4, so s_nz of row 64 c + 1 is off mod 4
            if kind == "row":
                seg[1] = T - off
                rows.append((64 * c + 1, off, T))
                used = 2
            else:
                n = 46
                seg[1:n] = rng.integers(30, 45, n - 1)
                seg[n] = T - off - seg[1:n].sum()
                runs.append((64 * c + 1, n, off, T))
                used = n + 1
        rest = Z - seg[:used].sum()
        f = 64 - used
        seg[used:] = 2 + rng.multinomial(rest - 2 * f, np.full(f, 1.0 / f))
    assert (lens.sum(axis=1) == Z).all()
    return lens.ravel(), rows, runs


def lens_direct(G=40):
    """direct rows first and last in the matrix, first and last in a CTA of the even split, and two in a row"""
    lens = np.random.default_rng(12).integers(1, 30, 64 * G)
    at = [0, 64 * 3, 64 * 5 + 63, 64 * 7 + 10, 64 * 7 + 11, 64 * G - 1]
    for i, r in enumerate(at):
        lens[r] = DIRECT + i
    return lens, at


def lens_empty(G=40):
    """(public layout only) empty rows first, last, at CTA starts, right after a direct row, and one CTA of nothing but"""
    V = 64 * (G - 1) + 2
    lens = np.random.default_rng(13).integers(1, 30, V)
    part = even_split(V, G)
    lens[[0, V - 1, part[2], part[5], 301]] = 0
    lens[300] = DIRECT
    lens[part[10]:part[11]] = 0
    return lens, part


def lens_rows256(seed=14, H=2500):
    """(solver layout) runs of 256 and 257 one-entry rows, each after a direct row, starting at every row offset mod 4: the
    256-row block limit and the rowptr stage alignment at it.  Eight segments of 314 rows, G = 40: four pairs of H-entry rows,
    each pair of k_partition weight Wc = 2 (2 H + 5), then 306 light rows of weight Wc too.  The partition's targets are the
    multiples of Wc, so its fifth CTA of a segment holds all the light rows.  Returns (lens, runs [(r, n)])."""
    rng = np.random.default_rng(seed)
    Wc, segs, runs = 2 * (2 * H + 5), [], []
    for s, (n, off) in enumerate([(n, off) for off in range(4) for n in (NT, NT + 1)]):
        base = 314 * s
        q = (off - (base + 9)) % 4                 # light rows before the direct row: the run starts at off mod 4
        light = np.ones(306, np.int64)
        light[q] = DIRECT
        f = 306 - q - 1 - n                        # filler rows after the run
        nnz_light = (Wc - 5 * 306) // 2
        light[q + 1 + n:] = 1 + rng.multinomial(nnz_light - light[:q + 1 + n].sum() - f, np.full(f, 1.0 / f))
        segs += [np.full(8, H), light]
        runs.append((base + 8 + q + 1, n))
    lens = np.concatenate(segs)
    assert (lens.shape[0] + 63) // 64 == 40 and 2 * lens.sum() + 5 * lens.shape[0] == 40 * Wc
    return lens, runs


def lens_hub(V, p, seed):
    """(solver layout) a share p of rows with ~1030 entries, each its own block (two never fit a stage), then short rows:
    the nnz-balanced partition gives the CTAs of the first part ~64 p blocks"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(3, 9, V)
    n = int(V * p)
    lens[:n] = rng.integers(1025, 1036, n)
    return lens


def lens_overflow(seed=15):
    """(solver layout) ~6,300 rows: 30 % with ~1030 entries (one block each) and 70 % direct rows of ~2100.  A CTA of the
    first kind gets far more than 64 blocks: the plan overflows."""
    rng = np.random.default_rng(seed)
    V = 6300
    lens = rng.integers(2095, 2106, V)
    n = int(0.3 * V)
    lens[:n] = rng.integers(1025, 1036, n)
    return lens


_cache = {}


def foreign(name, fn, **kw):
    if name not in _cache:
        _cache.clear()
        out = fn()
        lens = out[0] if isinstance(out, tuple) else out
        _cache[name] = (Foreign(name, lens, **kw), out)
    return _cache[name]


# ---------------------------------------------------------------------------------------------------- the two layouts
def public_checks(F, ks=(1, 2, 3, 4), G=None):
    """spmm for every k of ks; returns the failures and, when the grid is known, the blocks of the even split"""
    fails = []
    for k in ks:
        y = spmm(F.M, t(F.x(k))).cpu().numpy()
        fails += values(f"{F.name} public k={k}", F, k, y)
    blocks = plan(F.rowptr, even_split(F.V, G)) if G else None
    return fails, blocks


def solver_checks(F, monkeypatch, ks=(1, 2, 3, 4)):
    """the graph-mode CSR engine on F for every k of ks, through which 0, 4 and bench_spmm; three launches give the same bits
    as one.  Returns the failures, describe() and the model's blocks for the solver's grid and partition."""
    set_env(monkeypatch, SOLVER)
    s = PCGSolver(F.M)
    d = s.describe()
    assert d["algo"] == "graph" and d["sell_engine"] == 0 and not d["reordered"], d
    blocks = plan(F.rowptr, partition(F.rowptr, d["spmm_grid"]))
    most = max(len(b) for b in blocks)
    assert bool(d["planned"]) == (most <= BMAX), (d, most)          # the device's overflow bit agrees with the model
    fails = []
    for k in ks:
        tag = f"{F.name} solver k={k}"
        x = F.x(k)
        for which in (0, 4, "spmm"):
            y, dot = run(s, k, x, which)
            fails += values(f"{tag} which={which}", F, k, y)
            fails += dot_check(f"{tag} which={which}", x, y, dot)     # the CSR engine always runs its epilogue
            if which == 0:
                y0, dot0 = y, dot
        y3, dot3 = run(s, k, x, 0, n=3)
        if not (np.array_equal(bits(y3), bits(y0)) and np.array_equal(dot3.view(np.uint64), dot0.view(np.uint64))):
            fails.append(f"{tag}: 3 launches give dot {dot3.tolist()}, 1 gives {dot0.tolist()}")
    del s
    return fails, d, blocks


def stage_edges_reached(F, blocks, rows, runs):
    for r, off, T in rows:
        r0, nr, direct, s, e = block_at(blocks, r)
        assert s & 3 == off and nr == 1 and direct == (T > FIT), (r, off, T, block_at(blocks, r))
        if T <= FIT:
            assert e - (s & ~3) == T, (r, off, T)
    for r, n, off, S in runs:
        r0, nr, direct, s, e = block_at(blocks, r)
        assert s & 3 == off and not direct, (r, n, off, S)
        if S == FIT:
            assert nr == n and e - (s & ~3) == FIT, (r, n, S, block_at(blocks, r))
        else:
            assert nr == n - 1 and e - (s & ~3) < FIT, (r, n, S, block_at(blocks, r))


# ----------------------------------------------------------------------------------------------------- public layout
def test_public_column_chunks():
    """k = 1..4 and the 4-column chunk loop at k = 5, 7, 8, 9, through spmm and to_differential"""
    F, (lens, rows, runs) = foreign("stage", lens_stage)
    fails, _ = public_checks(F, ks=(1, 2, 3, 4, 5, 7, 8, 9))
    for k in (3, 9):
        y = to_differential(F.M, t(F.x(k))).cpu().numpy()
        fails += values(f"stage to_differential k={k}", F, k, y)
    assert not fails, fails


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 9])
def test_public_leading_dimensions(k):
    """ldx > k and ldy > k through the C entry point: the extra x columns are NaN and must not be read; the extra y columns
    and one row past V hold a sentinel that must survive; every row < V is written (it starts as the sentinel too)"""
    F, _ = foreign("stage", lens_stage)
    ldx, ldy = k + 3, k + 2
    rowptr, col, val = csr_of(F.M)
    xb = np.full((F.V, ldx), np.nan, np.float32)
    xb[:, :k] = F.x(k)
    yb = np.full((F.V + 1, ldy), SENTINEL, np.uint32).view(np.float32)
    x_d, y_d = t(xb), t(yb)
    rc = N.lib().ls_spmm_csr_f32(F.V, N.ptr(rowptr), N.ptr(col), N.ptr(val), N.ptr(x_d), ldx, N.ptr(y_d), ldy, k,
                                 N.stream_ptr(DEV))
    assert rc == N.LS_OK, N.last_error()
    out = y_d.cpu().numpy()
    fails = values(f"ldx={ldx} ldy={ldy} k={k}", F, k, np.ascontiguousarray(out[:F.V, :k]))
    assert (out[:F.V, k:].view(np.uint32) == SENTINEL).all(), "a column past k was written"
    assert (out[F.V].view(np.uint32) == SENTINEL).all(), "row V was written"
    assert not fails, fails


def test_public_stage_capacity_edges():
    F, (lens, rows, runs) = foreign("stage", lens_stage)
    G = public_grid(F.V)
    fails, blocks = public_checks(F, G=G)
    stage_edges_reached(F, blocks, rows, runs)
    for r in [g[0] for g in rows + runs]:   # the direct row before each group opens a CTA of the even split
        assert r - 1 in even_split(F.V, G) and block_at(blocks, r - 1)[1:3] == (1, 1)
    assert not fails, fails


def test_public_direct_rows_at_cta_edges():
    F, (lens, at) = foreign("direct", lens_direct)
    G = public_grid(F.V)
    fails, blocks = public_checks(F, G=G)
    part = even_split(F.V, G)
    for r in at:
        assert block_at(blocks, r)[1:3] == (1, 1), (r, block_at(blocks, r))
    first = {int(p) for p in part[:-1]}
    last = {int(p) - 1 for p in part[1:]}
    assert {0, 64 * 3} <= first and {64 * 5 + 63, F.V - 1} <= last
    assert not fails, fails


def test_public_empty_rows():
    """empty rows first, last, at CTA starts and block starts, a CTA of empty rows only (rows without a diagonal too), and a
    matrix with no entry at all through the C entry point"""
    F, (lens, part) = foreign("empty", lens_empty, diag=np.random.default_rng(3).random(64 * 39 + 2) < 0.5)
    G = public_grid(F.V)
    assert G == len(part) - 1
    fails, blocks = public_checks(F, ks=(1, 2, 3, 4, 5), G=G)
    for r in (0, part[2], part[5], 301):      # an empty row opens a block (301: after the direct row 300)
        assert lens[r] == 0 and block_at(blocks, r)
    assert block_at(blocks, 300)[1:3] == (1, 1)
    assert blocks[10] and all(b[3] == b[4] for b in blocks[10])          # blocks with nothing to copy
    assert blocks[-1][-1][0] + blocks[-1][-1][1] == F.V and lens[F.V - 1] == 0
    assert not fails, fails
    # every row empty: the kernel streams rowptr only
    V = 200
    rowptr = torch.zeros(V + 1 + 8, dtype=torch.int32, device=DEV)
    pad = torch.zeros(8, dtype=torch.int32, device=DEV)
    for k in (1, 3, 6):
        x = t(np.random.default_rng(k).normal(size=(V, k)).astype(np.float32))
        y = torch.full((V, k), float("nan"), device=DEV)
        rc = N.lib().ls_spmm_csr_f32(V, N.ptr(rowptr), N.ptr(pad), N.ptr(pad), N.ptr(x), k, N.ptr(y), k, k, N.stream_ptr(DEV))
        assert rc == N.LS_OK, N.last_error()
        assert (y.cpu().numpy() == 0).all()


@pytest.mark.parametrize("V", [1, 2, 3, 37, 63, 64, 65, 4095, 4096, 4097, 4098])
def test_public_sizes(V):
    """one CTA (V < 64), V = 64 G - 1, 64 G, 64 G + 1, and V = 0..3 mod 4 (the last rowptr stage copy)"""
    rng = np.random.default_rng(V)
    diag = rng.random(V) < 0.5
    lens = rng.integers(0, 40, V)
    lens[rng.random(V) < 0.01] = DIRECT
    lens = np.minimum(lens, np.where(diag, V, V - 1))
    F = Foreign(f"V{V}", lens, diag=diag, seed=V)
    fails, _ = public_checks(F, ks=(1, 2, 3, 4, 6))
    assert not fails, fails


def test_public_plane2000():
    """the 4 * 10^6-row plane: every CTA owns thousands of rows, so its two-stage ring wraps many times"""
    v, f = workloads.plane(2000, seed=0)
    M = compute_matrix(*to_dev(v, f), **UNI)
    rowptr, col, val = (a.cpu().numpy() for a in csr_of(M))
    V = int(M.shape[0])
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    assert V // (sms * (2048 // (NT + 32))) >= 16 * NT       # at most 7 CTAs of 288 threads per SM
    A = sp.csr_matrix((val, col, rowptr), shape=(V, V)).astype(np.float64)
    fails = []
    for k in (3, 1):
        x = np.random.default_rng(k).normal(size=(V, k)).astype(np.float32)
        y = spmm(M, t(x)).cpu().numpy()
        bad = np.flatnonzero((y != oracle.sell_spmv_f32(rowptr, col, val, x)).any(axis=1))
        if bad.size:
            fails.append(f"plane2000 k={k}: {bad.size} rows differ from the fmaf chain, first {bad[:6].tolist()}")
        w = np.diff(rowptr).astype(np.float64)[:, None] * U32
        err = np.abs(y - A @ x.astype(np.float64))
        if not (err <= w / (1 - w) * (abs(A) @ np.abs(x.astype(np.float64)))).all():
            fails.append(f"plane2000 k={k}: outside the rounding bound")
    assert not fails, fails


# ----------------------------------------------------------------------------------------------------- solver layout
def test_solver_stage_capacity_edges(monkeypatch):
    F, (lens, rows, runs) = foreign("stage", lens_stage)
    fails, d, blocks = solver_checks(F, monkeypatch)
    assert d["planned"] == 1
    stage_edges_reached(F, blocks, rows, runs)
    assert not fails, fails


def test_solver_direct_rows(monkeypatch):
    F, (lens, at) = foreign("direct", lens_direct)
    fails, d, blocks = solver_checks(F, monkeypatch)
    for r in at:
        assert block_at(blocks, r)[1:3] == (1, 1), (r, block_at(blocks, r))
    assert not fails, fails


def test_solver_256_row_blocks(monkeypatch):
    """blocks of exactly 256 rows (and a 257th row in a block of its own) starting at every row offset mod 4"""
    F, (lens, runs) = foreign("rows256", lens_rows256)
    fails, d, blocks = solver_checks(F, monkeypatch)
    assert d["planned"] == 1 and d["spmm_grid"] == 40
    for r, n in runs:
        assert block_at(blocks, r)[1:3] == (NT, 0), (r, block_at(blocks, r))
        if n == NT + 1:
            assert block_at(blocks, r + NT)[0] == r + NT
    assert {r & 3 for r, n in runs} == {0, 1, 2, 3}
    fails += public_checks(F)[0]
    assert not fails, fails


def test_solver_second_descriptor_register(monkeypatch):
    """a CTA with 33..64 planned blocks: blocks 33 and up come from the producer's second descriptor register"""
    F, lens = foreign("hub", lambda: lens_hub(4096, 0.75, 16))
    fails, d, blocks = solver_checks(F, monkeypatch)
    most = max(len(b) for b in blocks)
    print(f"hub: V={F.V} nnz={F.rowptr[-1]} grid={d['spmm_grid']} most blocks per CTA={most}")
    assert d["planned"] == 1 and 40 <= most <= BMAX, most
    assert not fails, fails


def test_solver_plan_overflow(monkeypatch):
    """a CTA with more than 64 blocks: no plan, and the on-the-fly producer walks the nnz-balanced partition"""
    F, lens = foreign("overflow", lens_overflow)
    fails, d, blocks = solver_checks(F, monkeypatch)
    most = max(len(b) for b in blocks)
    print(f"overflow: V={F.V} nnz={F.rowptr[-1]} grid={d['spmm_grid']} most blocks per CTA={most}")
    assert d["planned"] == 0 and most > BMAX
    assert sum(b[2] for cta in blocks for b in cta) > 1000         # direct rows in the same launch
    assert not fails, fails


# -------------------------------------------------------------------------------------------------- the public API
def _random_coo(shape, nnz, seed):
    rng = np.random.default_rng(seed)
    key = np.unique(rng.integers(0, shape[0] * shape[1], nnz))
    idx = np.stack([key // shape[1], key % shape[1]])
    return torch.sparse_coo_tensor(torch.from_numpy(idx).to(DEV), t(rng.normal(size=key.size).astype(np.float32)),
                                   shape).coalesce()


@pytest.mark.parametrize("shape", [(300, 200), (200, 300)], ids=["tall", "wide"])
def test_non_square_matrix_is_rejected(shape):
    """the C ABI has one V for the rows of L, x and y: a non-square L raises before anything reaches the device"""
    A = _random_coo(shape, 2000, 1)
    x = t(np.ones((shape[1], 3), np.float32))
    gy = t(np.ones((shape[0], 3), np.float32))
    n0 = N.launch_count()
    with pytest.raises(ValueError):
        spmm(A, x)
    with pytest.raises(ValueError):
        to_differential(A, x)
    with pytest.raises(ValueError):
        spmm_grad_values(A, gy, x)
    assert N.launch_count() == n0


def test_non_symmetric_gradient():
    """d/dx of sum(g * (A x)) is A^T g for a foreign non-symmetric A; the gradient w.r.t. A's values is unchanged"""
    rng = np.random.default_rng(21)
    F = Foreign("nonsym", rng.integers(1, 24, 700), diag=rng.random(700) < 0.5, seed=21)
    At = F.A.T.tocsr()
    At.sort_indices()
    assert abs(F.A - At).max() > 0
    for k in (1, 3, 4, 6):
        x = t(F.x(k)).requires_grad_(True)
        g = np.random.default_rng(100 + k).normal(size=(F.V, k)).astype(np.float32)
        (to_differential(F.M, x) * t(g)).sum().backward()
        gx = x.grad.cpu().numpy()
        assert np.array_equal(gx, oracle.sell_spmv_f32(At.indptr, At.indices, At.data, g)), k
        # against torch's own L @ v backward: both within gamma_w of the fp64 A^T g, w the column counts of A
        xt = t(F.x(k)).requires_grad_(True)
        (torch.sparse.mm(F.M, xt) * t(g)).sum().backward()
        ref = At.astype(np.float64) @ g.astype(np.float64)
        mag = abs(At.astype(np.float64)) @ np.abs(g.astype(np.float64))
        wu = np.diff(At.indptr).astype(np.float64)[:, None] * U32
        gam = wu / (1 - wu) * mag
        assert (np.abs(gx - ref) <= gam).all(), k
        assert (np.abs(gx - xt.grad.cpu().numpy()) <= 2 * gam).all(), k
    # with A's values requiring grad: the values gradient is the sampled product, as before
    A = F.M.detach().clone().requires_grad_(True)
    x = t(F.x(3)).requires_grad_(True)
    g = t(np.random.default_rng(7).normal(size=(F.V, 3)).astype(np.float32))
    (to_differential(A, x) * g).sum().backward()
    assert torch.equal(A.grad.coalesce().values(), spmm_grad_values(F.M, g, t(F.x(3))))
    assert np.array_equal(x.grad.cpu().numpy(), oracle.sell_spmv_f32(At.indptr, At.indices, At.data, g.cpu().numpy()))


def test_non_finite_x():
    """+-inf and NaN in chosen rows of x, in rows with and without a diagonal and with lengths = 0 and != 0 mod 8: the NaN /
    +-inf / finite pattern of y and its signs are torch's A @ x, and the finite rows are the fmaf chain"""
    rng = np.random.default_rng(31)
    V = 512
    lens = rng.choice([5, 8, 11, 13, 16, 19], V)
    diag = rng.random(V) < 0.5
    F = Foreign("nonfinite", lens, diag=diag, seed=31)
    for k in (1, 3, 4, 5):
        x = F.x(k).copy()
        pick = rng.choice(V, 24, replace=False)
        x[pick[:8]] = np.inf
        x[pick[8:16]] = -np.inf
        x[pick[16:]] = np.nan
        x[pick[0], 0] = 1.0                       # a row of x with both finite and non-finite entries
        y = spmm(F.M, t(x)).cpu().numpy()
        yt = torch.sparse.mm(F.M, t(x)).cpu().numpy()
        assert np.array_equal(np.isnan(y), np.isnan(yt)), k
        assert np.array_equal(np.isposinf(y), np.isposinf(yt)) and np.array_equal(np.isneginf(y), np.isneginf(yt)), k
        fin = np.isfinite(yt)
        model = oracle.sell_spmv_f32(F.rowptr, F.col, F.val, np.where(np.isfinite(x), x, 0).astype(np.float32))
        assert np.array_equal(y[fin], model[fin]), k
        # the rows the padding used to poison: x[row] not finite, no entry in column row, length not a multiple of 8
        own = np.zeros(V, bool)
        own[pick] = True
        poisoned = own & ~diag & (lens % 8 != 0) & fin.all(axis=1)
        assert poisoned.any(), k


def test_empty_matrix():
    """nnz = 0: zeros of shape (V, k), an empty values gradient, and zero gradients"""
    V = 100
    A = torch.sparse_coo_tensor(torch.zeros((2, 0), dtype=torch.int64, device=DEV), torch.zeros(0, device=DEV), (V, V)).coalesce()
    for k in (1, 3, 5):
        x = t(np.random.default_rng(k).normal(size=(V, k)).astype(np.float32))
        y = spmm(A, x)
        assert y.shape == (V, k) and (y == 0).all()
        assert spmm_grad_values(A, x, x).shape == (0,)
    y1 = spmm(A, x[:, 0])
    assert y1.shape == (V,) and (y1 == 0).all()
    xg = x.clone().requires_grad_(True)
    (to_differential(A, xg) * x).sum().backward()
    assert (xg.grad == 0).all()
