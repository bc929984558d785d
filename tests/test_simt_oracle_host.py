"""The SIMT GEMM emulation (tests/simt_oracle.py) against exact rational arithmetic.  No device needed.

fma32 is checked against fractions.Fraction rounded to fp32 by hand (round to nearest, ties to even, with subnormals
and overflow) on random triples over the whole exponent range, on constructed cases where the float64 sum lands
exactly on an fp32 midpoint (with and without a rounding error below it), on subnormal products and addends, and on
large cancellations.  The GEMM, the row norm and the epilogues are then checked as compositions of it."""
from fractions import Fraction

import numpy as np

import simt_oracle as so

F32 = np.float32
_MAX_MID = Fraction(2) ** 128 - Fraction(2) ** 103  # halfway between FLT_MAX and 2^128


def _round_f32(q):
    """The fp32 nearest to the rational q, ties to even, as a Python float (exactly representable)."""
    if q == 0:
        return 0.0
    sign = -1.0 if q < 0 else 1.0
    q = abs(q)
    if q >= _MAX_MID:  # FLT_MAX has an odd significand, so the tie goes to 2^128 = inf
        return sign * float("inf")
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    elif Fraction(2) ** (e + 1) <= q:
        e += 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    n = q / ulp
    k = n.numerator // n.denominator
    rem = n - k
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and k % 2 == 1):
        k += 1
    return sign * float(k * ulp)


def _exact_fma(a, b, c):
    if not all(np.isfinite([a, b, c])):  # inf and NaN operands: IEEE's rules, the same in any precision
        return float(np.float64(a) * np.float64(b) + np.float64(c))
    return _round_f32(Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c)))


def _check(a, b, c):
    a, b, c = (v.ravel() for v in np.broadcast_arrays(*(np.asarray(v, dtype=F32) for v in (a, b, c))))
    got = so.fma32(a, b, c)
    for i in range(a.size):
        want = _exact_fma(a[i], b[i], c[i])
        assert got[i] == want or (np.isnan(got[i]) and np.isnan(want)), (a[i], b[i], c[i], got[i], want)
    return got


def _random_f32(rng, n, emin, emax):
    m = rng.uniform(1.0, 2.0, n)
    e = rng.integers(emin, emax, n)
    s = rng.choice([-1.0, 1.0], n)
    return (s * np.ldexp(m, e)).astype(F32)


def test_fma32_random_triples():
    rng = np.random.default_rng(0)
    n = 4000
    for emin, emax in ((-3, 4), (-60, 60), (-140, -100), (60, 64)):
        a, b = _random_f32(rng, n, emin, emax), _random_f32(rng, n, emin, emax)
        # addends at the product's scale (cancellation and carries) and far from it
        c = np.concatenate([_random_f32(rng, n // 2, 2 * emin, 2 * emax),
                            (-(a[: n // 2].astype(np.float64) * b[: n // 2]) *
                             rng.uniform(0.999, 1.001, n // 2)).astype(F32)])
        _check(a, b, c)


def _near_products(rng, target, n):
    """fp32 pairs (a, b) whose product is within 2^-33 of ``target`` (relative) but not equal to it: a random,
    b = fl32(target / a), kept when the product lands that close (about one try in 2^8)."""
    a = rng.uniform(1.0, 2.0, 1 << 16).astype(F32)
    b = (target / a.astype(np.float64)).astype(F32)
    p = a.astype(np.float64) * b.astype(np.float64)
    keep = (np.abs(p - target) < 2.0 ** -33 * target) & (p != target)
    assert keep.sum() >= n
    return a[keep][:n], b[keep][:n]


def _double_rounded(a, b, c):
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)


def test_fma32_midpoint_ties():
    """c + a b with c in [s, 2 s) and a b within 5 2^-57 s of an odd number of c's half-ulps: the float64 sum is
    exactly an fp32 midpoint while the exact sum lies just above or below it, so rounding the float64 sum again breaks
    the tie the wrong way about half the time.  Then products that are exactly the odd half-ulps (ties to even)."""
    rng = np.random.default_rng(1)
    wrong_if_double_rounded = 0
    for scale in (1.0, 2.0 ** -30, 2.0 ** 40, 2.0 ** -100):
        for odd in (1, 3, 5):
            target = odd * 2.0 ** -24 * scale
            a, b = _near_products(rng, target, 64)
            c = (rng.integers(1 << 23, 1 << 24, a.size) * 2.0 ** -23 * scale).astype(F32)
            for sc, sp in ((1, 1), (-1, -1), (1, -1), (-1, 1)):
                cc, bb = (sc * c).astype(F32), (sp * b).astype(F32)
                got = _check(a, bb, cc)
                wrong_if_double_rounded += int((got != _double_rounded(a, bb, cc)).sum())
            at = np.full(8, F32(odd * scale), dtype=F32)
            bt = np.full(8, F32(2.0 ** -24), dtype=F32)
            _check(at, bt, c[:8])
            _check(at, -bt, c[:8])
            _check(at, bt, -c[:8])
    assert wrong_if_double_rounded > 300, wrong_if_double_rounded


def test_fma32_subnormals_and_cancellation():
    rng = np.random.default_rng(2)
    tiny = np.ldexp(rng.uniform(1.0, 2.0, 500), rng.integers(-149, -126, 500)).astype(F32)  # subnormal fp32
    a, b = _random_f32(rng, 500, -80, -60), _random_f32(rng, 500, -80, -60)  # products far below fp32's range
    _check(a, b, tiny)
    _check(a, b, -tiny)
    _check(a, b, np.zeros(500, dtype=F32))
    _check(tiny, F32(1.5), tiny)
    _check(_random_f32(rng, 500, -70, -60), _random_f32(rng, 500, -70, -60), np.zeros(500, dtype=F32))
    # c = -fl32(a b): the result is the rounding error of the product, exactly
    a, b = _random_f32(rng, 2000, -20, 20), _random_f32(rng, 2000, -20, 20)
    c = -(a.astype(np.float64) * b).astype(F32)
    got = _check(a, b, c)
    assert (got != 0).mean() > 0.9
    # overflow: just below, at and above the fp32 rounding threshold, and NaN / inf operands
    big = F32(np.finfo(F32).max)
    _check(np.full(4, big), np.array([1.0, 1.0, -1.0, 2.0], dtype=F32),
           np.array([F32(2.0 ** 103), F32(2.0 ** 102), F32(-2.0 ** 103), F32(0.0)]))
    _check(np.array([np.nan, np.inf, 1.0], dtype=F32), np.array([1.0, 1.0, 1.0], dtype=F32),
           np.array([0.0, 0.0, np.nan], dtype=F32))


def _exact_chain(A, B):
    """fmaf chains of gemm_nt, each fma rounded exactly from rationals."""
    out = np.zeros((A.shape[0], B.shape[0]))
    for m in range(A.shape[0]):
        for n in range(B.shape[0]):
            acc = 0.0
            for k in range(A.shape[1]):
                acc = _exact_fma(A[m, k], B[n, k], acc)
            out[m, n] = acc
    return out


def test_gemm_and_row_sqnorm_compose_exact_fmas():
    rng = np.random.default_rng(3)
    A = _random_f32(rng, 5 * 37, -4, 4).reshape(5, 37)
    B = _random_f32(rng, 3 * 37, -4, 4).reshape(3, 37)
    assert np.array_equal(so.gemm_nt(A, B), _exact_chain(A, B))
    # the row norm: 32 lane chains (lane l: k = l, l + 32), then the xor butterfly.  Its last step adds lane 1's value
    # to lane 0's, so lane 0 ends with (sum over even lanes) + (sum over odd lanes), each split the same way by the
    # next bit, down to the pairs (l, l + 16) the first step adds
    X = _random_f32(rng, 4 * 37, -4, 4).reshape(4, 37)
    for r in range(4):
        lanes = [0.0] * 32
        for k in range(37):
            lanes[k % 32] = _exact_fma(X[r, k], X[r, k], lanes[k % 32])

        def tree(idx):
            if len(idx) == 1:
                return lanes[idx[0]]
            return _round_f32(Fraction(tree(idx[0::2])) + Fraction(tree(idx[1::2])))
        assert so.row_sqnorm(X[r:r + 1])[0] == tree(list(range(32)))


def test_sqdist_epilogue_cases():
    """Exact zero for identical rows, the clamp of a negative d2, NaN passing the clamp, squared = 0 and 1."""
    x = np.array([[1.5, -2.25, 3.0], [1e3 + 0.1, 1e3, 1e3 - 0.1]], dtype=F32)
    M = so.sqdist(x, x)
    assert M[0, 0] == 0 and M[1, 1] == 0 and M[0, 1] == M[1, 0] > 0
    dot, a, b = F32(1.0), F32(0.75), F32(1.0)  # d2 = 1.75 - 2 < 0
    assert so.sqdist_epilogue(dot, a, b, 1) == 0 and so.sqdist_epilogue(dot, a, b, 0) == 0
    assert np.isnan(so.sqdist_epilogue(F32(np.nan), a, b, 1))
    r = so.sqdist_epilogue(F32(0.0), F32(2.0), F32(0.0), 0)
    assert r == np.sqrt(F32(2.0)) and so.sqdist_epilogue(F32(0.0), F32(2.0), F32(0.0), 1) == r * r != 2.0
    assert so.cost_max(np.array([[np.nan, 3.0], [0.0, 2.0]], dtype=F32)) == 3.0
    assert so.cost_max(np.array([[np.nan]], dtype=F32)) == 0.0


def test_bias_act_pre_time_column():
    rng = np.random.default_rng(4)
    acc, bias, tcol = (_random_f32(rng, n, -3, 3) for n in (12, 4, 4))
    acc = acc.reshape(3, 4)
    t = F32(0.37)
    got = so.bias_act_pre(acc, bias, t, tcol)
    for m in range(3):
        for n in range(4):
            v = _round_f32(Fraction(float(acc[m, n])) + Fraction(float(bias[n])))
            assert got[m, n] == _exact_fma(t, tcol[n], v)
    assert np.array_equal(so.bias_act_pre(acc, bias), (acc + bias[None, :]).astype(F32))
