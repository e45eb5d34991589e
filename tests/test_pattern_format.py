"""CPU model of the pattern-only matrix copy's storage (csrc/ls_pcg.cu pat_width_kernel / pat_fill_kernel, the layout of
csrc/ls_sell_kernel.cuh): pairs of signed 16-bit column offsets in compact slices, plain column pairs in the slices that need
them (bit 0 of the slice offset), and the diagonal classes that replace the per-row D^-1 and corrected diagonal."""
import numpy as np
import scipy.sparse as sp

import oracle
from largesteps_b200 import workloads

f32 = np.float32


def pattern_copy(rp, ci, va, V):
    """(poff, words, cls, table) as the fill kernel writes them, vectorised over rows."""
    Vp = (V + 31) // 32 * 32
    rows = np.repeat(np.arange(V), np.diff(rp))
    off = ci != rows
    c = f32(va[off][0])
    used = np.zeros(Vp, np.int64)
    used[:V] = np.bincount(rows[off], minlength=V)
    far = np.zeros(Vp, bool)
    far[:V] = np.bincount(rows[off], weights=(np.abs(ci[off] - rows[off]) > 32767), minlength=V) > 0
    w2 = (used.reshape(-1, 32).max(1) + 1) // 2
    wide = far.reshape(-1, 32).any(1)
    cnt = np.where(wide, 64, 32) * w2
    poff = np.zeros(len(cnt) + 1, np.int64)
    poff[1:] = np.cumsum(cnt)
    assert (poff % 32 == 0).all()                     # wide pairs stay 8-byte aligned
    words = np.zeros(poff[-1], np.uint32)
    d = np.zeros(Vp, f32)
    d[rows[~off]] = va[~off]
    for s in range(len(cnt)):
        for lane in range(32):
            r = 32 * s + lane
            slots = list(ci[rp[r]:rp[r + 1]][off[rp[r]:rp[r + 1]]]) if r < V else []
            slots += [r] * (2 * w2[s] - len(slots))   # unused slots: the row itself (offset 0)
            for m in range(w2[s]):
                a, b = slots[2 * m], slots[2 * m + 1]
                if wide[s]:
                    words[poff[s] + 2 * (32 * m + lane)] = a
                    words[poff[s] + 2 * (32 * m + lane) + 1] = b
                else:
                    words[poff[s] + 32 * m + lane] = ((a - r) & 0xFFFF) | (((b - r) & 0xFFFF) << 16)
    k = (2 * np.repeat(w2, 32) - used).astype(np.float64)
    dp = np.where(np.arange(Vp) < V, (d.astype(np.float64) - np.float64(c) * k).astype(f32), f32(0))
    di = np.zeros(Vp, f32)
    di[:V] = f32(1) / d[:V]
    keys = (di.view(np.uint32).astype(np.uint64) << np.uint64(32)) | dp.view(np.uint32).astype(np.uint64)
    table, cls = np.unique(keys, return_inverse=True)
    flagged = poff[:-1] | wide.astype(np.int64)
    return flagged, poff[-1], words, w2, cls, table, di, dp


def decode(flagged, total, words, s, lane):
    """columns of row 32 s + lane, pair by pair, as the solver reads them (lsk::pat_slice / pat_load / pat_cols)."""
    p0, p1 = int(flagged[s]), int(flagged[s + 1]) if s + 1 < len(flagged) else int(total)
    wide, o0 = p0 & 1, p0 & ~1
    w2 = ((p1 & ~1) - o0) >> (6 if wide else 5)
    r = 32 * s + lane
    out = []
    for m in range(w2):
        if wide:
            out += [int(words[o0 + 2 * (32 * m + lane)]), int(words[o0 + 2 * (32 * m + lane) + 1])]
        else:
            w = int(words[o0 + 32 * m + lane])
            lo, hi = w & 0xFFFF, w >> 16
            out += [r + (lo - 65536 if lo >= 32768 else lo), r + (hi - 65536 if hi >= 32768 else hi)]
    return out


def csr(v, f, **kw):
    rows, cols, vals, V = oracle.compute_matrix(np.asarray(v, np.float64), np.asarray(f), **kw)
    A = sp.csr_matrix((vals.astype(f32), (rows, cols)), shape=(V, V))
    A.sort_indices()
    return A.indptr, A.indices, A.data, V


def test_compact_and_wide_slices_decode_to_the_columns():
    v, f = workloads.plane(200, seed=0)
    V = v.shape[0]
    # move 1000 vertices to the far end of the numbering: their slices (and their neighbours') need full columns
    perm = np.arange(V)
    perm[:1000], perm[V - 1000:] = np.arange(V - 1000, V), np.arange(1000)
    rp, ci, va, V = csr(v, perm[f], lambda_=1.0, alpha=0.95)
    flagged, total, words, w2, cls, table, di, dp = pattern_copy(rp, ci, va, V)
    wide = flagged & 1
    assert 0 < wide.sum() < len(wide)
    for s in list(np.flatnonzero(wide)[:4]) + list(np.flatnonzero(wide == 0)[:4]) + [len(wide) - 1]:
        for lane in range(32):
            r = 32 * s + lane
            got = decode(flagged, total, words, s, lane)
            want = list(ci[rp[r]:rp[r + 1]][ci[rp[r]:rp[r + 1]] != r]) if r < V else []
            assert got[:len(want)] == want and all(x == r for x in got[len(want):]), (s, lane)
    # the compact copy costs 4 bytes per pair: half of the wide layout
    assert total == sum((64 if w else 32) * n for w, n in zip(wide, w2))


def test_diagonal_classes_are_few_and_exact(bunny_mesh):
    for v, f, kw in ((*workloads.plane(120, seed=0), dict(lambda_=1.0, alpha=0.95)),
                     (*workloads.subdivide(*bunny_mesh), dict(lambda_=19.0)),
                     (*workloads.icosphere(3), dict(lambda_=10.0))):
        rp, ci, va, V = csr(v, f, **kw)
        flagged, total, words, w2, cls, table, di, dp = pattern_copy(rp, ci, va, V)
        assert len(table) <= 256                       # what the 1-byte class can address
        assert (flagged & 1).sum() == 0                # native order: every slice compact
        # a class lookup gives back the very floats the row had
        assert ((table[cls] >> np.uint64(32)).astype(np.uint32) == di.view(np.uint32)).all()
        assert ((table[cls] & np.uint64(0xFFFFFFFF)).astype(np.uint32) == dp.view(np.uint32)).all()

