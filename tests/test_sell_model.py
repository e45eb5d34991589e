"""CPU: the exact model of the solver's SELL-32 SpMV (oracle.sell_spmv_f32, oracle/cg_port.c) against an exact evaluation of
the same chain in rational arithmetic, and the padded widths (oracle.sell32) against a direct count.

tests/test_gpu_sell_spmv.py compares the device's SpMV with this model bit for bit; here the model itself is pinned: every
row is the fmaf chain over the row's CSR entries and then its slice padding {own row, 0.0f}, from acc = +0, each step the
exact value of val * x + acc rounded once to float32 (round to nearest even, gradual underflow, IEEE signs of zero)."""
import math
from fractions import Fraction

import numpy as np

import oracle


def pow2(e):
    return Fraction(2 ** e) if e >= 0 else Fraction(1, 2 ** -e)


def round_f32(q):
    """the float32 nearest to the rational q != 0 (ties to even), with the sign of q when it rounds to zero"""
    s = -1 if q < 0 else 1
    a = abs(q)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if a < pow2(e):
        e -= 1
    quantum = pow2(max(e - 23, -149))        # 24-bit significand; below 2^-126 the spacing stays 2^-149
    t = a / quantum
    m = t.numerator // t.denominator
    rem = t - m
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and m % 2 == 1):
        m += 1
    assert m * quantum < pow2(128), "overflow: the test data must stay finite"
    return np.float32(s * float(m * quantum)) if m else np.float32(math.copysign(0.0, s))


def fma_f32(a, b, c):
    """fmaf(a, b, c) of float32 values, exactly: one rounding of a b + c"""
    p = Fraction(float(a)) * Fraction(float(b))
    s = p + Fraction(float(c))
    if s != 0:
        return round_f32(s)
    # an exact zero: -0 only if both addends are zeros of negative sign (round to nearest)
    p_neg = math.copysign(1.0, float(a)) * math.copysign(1.0, float(b)) < 0
    return np.float32(-0.0) if (p == 0 and p_neg and float(c) == 0 and math.copysign(1.0, float(c)) < 0) else np.float32(0.0)


def sell_chain(rowptr, col, val, x):
    V, K = x.shape
    w = oracle.sell32(rowptr, col)
    y = np.empty((V, K), np.float32)
    for i in range(V):
        for k in range(K):
            acc = np.float32(0.0)
            for j in range(int(w[i])):
                e = rowptr[i] + j
                acc = fma_f32(val[e], x[col[e], k], acc) if e < rowptr[i + 1] else fma_f32(np.float32(0.0), x[i, k], acc)
            y[i, k] = acc
    return y


def mixed_csr(V=300, seed=0):
    """rows of 1 .. 12 entries with magnitudes from 1e-22 to 1e17 and both signs (products from the subnormal range to 1e34),
    one 101-entry row, rows whose chain cancels to +0, rows whose products underflow to -0 and a row of subnormals; x to match"""
    rng = np.random.default_rng(seed)
    mag = lambda n: (10.0 ** rng.uniform(-22, 17, n)) * rng.choice([-1.0, 1.0], n)
    x = mag(V * 3).astype(np.float32).reshape(V, 3)
    rows = []
    for i in range(V):
        n = int(rng.integers(1, 13))
        c = np.sort(rng.choice(V, size=n, replace=False)).astype(np.int32)
        rows.append((c, mag(n).astype(np.float32)))
    rows[37] = (np.sort(rng.choice(V, size=101, replace=False)).astype(np.int32), mag(101).astype(np.float32))
    # cancellation to +0: two columns with equal x, opposite weights (the same x in every column of the right-hand side)
    x[10] = x[11]
    rows[5] = (np.array([10, 11], np.int32), np.array([2.0, -2.0], np.float32))   # exact products: fmaf cancels them
    # products below half the smallest subnormal: every step rounds to a zero of the product's sign; the padding's
    # 0 * x[own row] then decides the sign of a -0 row (x[50] < 0 keeps it, x[51] > 0 turns it into +0)
    x[50], x[51] = -np.abs(x[50]), np.abs(x[51])
    tiny = np.float32(1e-30)
    x[60] = tiny
    rows[50] = (np.array([60], np.int32), np.array([-tiny], np.float32))
    rows[51] = (np.array([60], np.int32), np.array([-tiny], np.float32))
    # a chain of subnormal products and sums (gradual underflow, rounded to the 2^-149 grid)
    x[62], x[63] = np.float32(1e-21), np.float32(-2.7e-21)
    rows[52] = (np.array([62, 63], np.int32), np.array([1e-20, 3.1e-20], np.float32))
    rowptr = np.zeros(V + 1, np.int32)
    rowptr[1:] = np.cumsum([len(c) for c, _ in rows])
    col = np.concatenate([c for c, _ in rows]).astype(np.int32)
    val = np.concatenate([v for _, v in rows]).astype(np.float32)
    return rowptr, col, val, x


def test_exact_rounding_agrees_with_float32_sums_and_products():
    """IEEE float32 addition and multiplication round the exact result once, as fmaf does: 1 * a + b and a * b + (-0)"""
    rng = np.random.default_rng(5)
    a, b = [(10.0 ** rng.uniform(-25, 18, 3000) * rng.choice([-1, 1], 3000)).astype(np.float32) for _ in range(2)]
    with np.errstate(under="ignore"):
        for p, q in zip(a, b):
            assert fma_f32(np.float32(1.0), p, q).view(np.uint32) == (p + q).view(np.uint32), (p, q)
            assert fma_f32(p, q, np.float32(-0.0)).view(np.uint32) == (p * q).view(np.uint32), (p, q)


def test_sell_model_is_the_exact_fmaf_chain():
    rowptr, col, val, x = mixed_csr()
    assert int(np.diff(rowptr).max()) == 101
    want = sell_chain(rowptr, col, val, x)
    for K in (1, 2, 3):
        got = oracle.sell_spmv_f32(rowptr, col, val, x[:, :K])
        assert np.array_equal(got.view(np.uint32), want[:, :K].view(np.uint32)), np.flatnonzero(
            (got.view(np.uint32) != want[:, :K].view(np.uint32)).any(axis=1))
    # the edges the data was built for are there
    assert (want[5] == 0).all() and not np.signbit(want[5]).any()
    assert (want[50] == 0).all() and np.signbit(want[50]).all()                 # -0 survives: 0 * x[50] is -0
    assert (want[51] == 0).all() and not np.signbit(want[51]).any()             # -0 + (+0) from the padding = +0
    assert (np.abs(want[52]) < np.float32(1.2e-38)).all() and (want[52] != 0).all()   # subnormal results
    # and it is not a plain sum: the rows of the 101-entry row's slice run 101 steps, most of them padding
    w = oracle.sell32(rowptr, col)
    assert (w[32:64] == 101).all()


def test_sell32_widths_match_a_direct_count():
    for V, seed in ((1, 0), (31, 1), (32, 2), (33, 3), (300, 4), (1000, 5)):
        rng = np.random.default_rng(seed)
        lens = rng.integers(0, 20, V)
        lens[rng.integers(0, V)] = 101
        rowptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        col = np.zeros(int(rowptr[-1]), np.int32)
        w = oracle.sell32(rowptr, col)
        assert w.shape == (V,)
        for i in range(V):
            s = i // 32
            assert w[i] == max(lens[32 * s:min(V, 32 * s + 32)])
