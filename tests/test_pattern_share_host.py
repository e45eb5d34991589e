"""CPU model of the shared pattern-only copy (csrc/ls_sell_kernel.cuh pat_word / pat_slice and csrc/ls_pcg_copies.cu
pat_hash_kernel .. pat_share_copy_kernel): bits 1-4 of a slice offset carry its pairs per row (15: up to the next slice's
offset), and identical compact slices point at one stored copy, the one of their lowest slice index."""
import numpy as np
import pytest

from largesteps_b200 import workloads

ESC = 15


def pat_word(o0, w2, wide):
    assert o0 % 32 == 0
    return o0 | (min(w2, ESC) << 1) | int(wide)


def pat_slice(poff, s):
    p0 = int(poff[s])
    wide, o0, f = p0 & 1, p0 & ~31, (p0 >> 1) & 15
    w2 = f if f < ESC else ((int(poff[s + 1]) & ~31) - o0) >> (6 if wide else 5)
    return o0, w2, bool(wide)


def structure(f, V):
    """structural CSR (sorted columns, no diagonal) of the mesh's vertex adjacency"""
    e = np.asarray(f, np.int64)[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2)
    key = np.unique(np.concatenate([e[:, 0] * V + e[:, 1], e[:, 1] * V + e[:, 0]]))
    rows, cols = key // V, key % V
    rp = np.zeros(V + 1, np.int64)
    rp[1:] = np.cumsum(np.bincount(rows, minlength=V))
    return rp, rows, cols


def slices(rp, rows, cols, V):
    """per slice: pairs per row, wide, and the stored words (compact: 16-bit offset pairs; wide: columns) in load order"""
    Vp = (V + 31) // 32 * 32
    ns = Vp // 32
    used = np.zeros(Vp, np.int64)
    used[:V] = np.diff(rp)
    w2 = (used.reshape(ns, 32).max(1) + 1) // 2
    far = np.zeros(Vp, bool)
    far[:V] = np.bincount(rows, weights=np.abs(cols - rows) > 32767, minlength=V) > 0
    wide = far.reshape(ns, 32).any(1)
    W = max(int(w2.max()), 1)
    slot = np.tile(np.arange(Vp)[:, None], (1, 2 * W))          # unused slots: the row itself
    slot[rows, np.arange(len(rows)) - rp[rows]] = cols
    r = np.arange(Vp)[:, None]
    off = (slot - r) & 0xFFFF
    compact = (off[:, 0::2] | (off[:, 1::2] << 16)).astype(np.uint32)   # (Vp, W)
    words = []
    for s in range(ns):
        n = int(w2[s])
        if wide[s]:
            words.append(slot[32 * s:32 * s + 32, :2 * n].reshape(32, n, 2).transpose(1, 0, 2).reshape(-1).astype(np.uint32))
        else:
            words.append(compact[32 * s:32 * s + 32, :n].T.reshape(-1))
    return w2, wide, words


def unshared(w2, wide, words):
    sizes = np.array([len(x) for x in words], np.int64)
    start = np.concatenate([[0], np.cumsum(sizes)])
    poff = np.array([pat_word(int(start[s]), int(w2[s]), wide[s]) for s in range(len(w2))] + [int(start[-1])], np.int64)
    return poff, np.concatenate(words) if len(words) else np.zeros(0, np.uint32)


def share(w2, wide, words):
    """the device build's result: (poff, stored words, slices stored)"""
    ns = len(w2)
    esc = w2 >= ESC
    shareable = ~wide & ~esc & ~np.concatenate([[False], esc[:-1]])
    rep = np.arange(ns)
    first = {}
    for s in range(ns):
        if shareable[s]:
            rep[s] = first.setdefault((int(w2[s]), words[s].tobytes()), s)
    stored = rep == np.arange(ns)
    sizes = np.array([len(words[s]) if stored[s] else 0 for s in range(ns)], np.int64)
    start = np.concatenate([[0], np.cumsum(sizes)])
    if stored.all():
        return (*unshared(w2, wide, words), ns)
    poff = np.array([pat_word(int(start[rep[s]]), int(w2[s]), wide[s]) for s in range(ns)] + [int(start[-1])], np.int64)
    pc = np.concatenate([words[s] for s in range(ns) if stored[s]])
    return poff, pc, int(stored.sum())


def decode_rows(poff, pc, ns):
    """columns of every row, as the solver reads them (pat_slice, pat_load, pat_cols); (Vp, 2 max w2), padded with the row"""
    ws = [pat_slice(poff, s) for s in range(ns)]
    W = max([w for _, w, _ in ws] + [1])
    out = np.tile(np.arange(32 * ns)[:, None], (1, 2 * W))
    for s, (o0, w2, wide) in enumerate(ws):
        r = 32 * s + np.arange(32)
        for m in range(w2):
            if wide:
                blk = pc[o0 + 64 * m:o0 + 64 * m + 64].reshape(32, 2).astype(np.int64)
                out[r, 2 * m], out[r, 2 * m + 1] = blk[:, 0], blk[:, 1]
            else:
                w = pc[o0 + 32 * m:o0 + 32 * m + 32].astype(np.int64)
                out[r, 2 * m] = r + (w & 0xFFFF).astype(np.int16)
                out[r, 2 * m + 1] = r + (w >> 16).astype(np.int16)
    return out


def expected_rows(rp, cols, V, W):
    Vp = (V + 31) // 32 * 32
    out = np.tile(np.arange(Vp)[:, None], (1, 2 * W))
    rows = np.repeat(np.arange(V), np.diff(rp))
    out[rows, np.arange(len(rows)) - rp[rows]] = cols
    return out


def test_offset_word_round_trip():
    for o0 in (0, 32, 4096, (1 << 30) - 32):
        for w2 in range(0, 15):
            for wide in (False, True):
                p = np.array([pat_word(o0, w2, wide), o0 + 999 * 32], np.int64)    # the next offset is not read
                assert pat_slice(p, 0) == (o0, w2, wide)
        for w2, wide in ((15, False), (16, False), (40, False), (15, True), (40, True)):   # escape: width from the next offset
            p = np.array([pat_word(o0, w2, wide), o0 + w2 * (64 if wide else 32)], np.int64)
            assert pat_slice(p, 0) == (o0, w2, wide)


def test_share_model_keeps_every_row_and_escape_neighbours_apart():
    # a plane with fan vertices of valence 40 (escape slices) and a block of far-numbered vertices (wide slices)
    v, f = workloads.plane(200, seed=0)
    V = v.shape[0]
    perm = np.arange(V)
    perm[:1000], perm[V - 1000:] = np.arange(V - 1000, V), np.arange(1000)
    f = perm[f]
    hubs = np.array([15000, 19000, 19031])
    extra = np.array([[h, (h + 7 * k + 1) % V, (h + 7 * k + 4) % V] for h in hubs for k in range(20)])
    f = np.concatenate([f, extra])
    rp, rows, cols = structure(f, V)
    w2, wide, words = slices(rp, rows, cols, V)
    assert (w2 >= ESC).any() and wide.any() and (~wide).any()
    poff, pc, stored = share(w2, wide, words)
    ns = len(w2)
    assert stored < ns and len(pc) < sum(len(x) for x in words)
    got = decode_rows(poff, pc, ns)
    assert (got == expected_rows(rp, cols, V, got.shape[1] // 2)).all()
    # an escape slice's end is the next slice's start: neither is shared
    for s in np.flatnonzero(w2 >= ESC):
        o0, n, wd = pat_slice(poff, s)
        assert (int(poff[s + 1]) & ~31) == o0 + n * (64 if wd else 32)
    # stored slices keep their order: the copies, taken in order of first use, lie at increasing offsets
    starts = np.array([int(p) & ~31 for p in poff[:-1]])
    _, first = np.unique(starts, return_index=True)
    assert (np.diff(starts[np.sort(first)]) > 0).all()
    unsh, pcu = unshared(w2, wide, words)
    assert (decode_rows(unsh, pcu, ns) == got).all()


@pytest.mark.parametrize("n, distinct", [(500, 16), (1000, 12), (2000, 10)])
def test_distinct_slices_of_the_plane(n, distinct):
    v, f = workloads.plane(n, seed=0)
    V = v.shape[0]
    rp, rows, cols = structure(f, V)
    w2, wide, words = slices(rp, rows, cols, V)
    assert not wide.any() and w2.max() < ESC
    keys = {(int(a), w.tobytes()) for a, w in zip(w2, words)}
    assert len(keys) == distinct
    if n <= 1000:
        poff, pc, stored = share(w2, wide, words)
        assert stored == distinct
        assert 4 * len(pc) < 8192                      # stored columns: a few KB instead of ~12 MB at n = 1000
        got = decode_rows(poff, pc, len(w2))
        assert (got == expected_rows(rp, cols, V, got.shape[1] // 2)).all()
