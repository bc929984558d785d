"""NumPy emulation of the SIMT fp32 GEMM core's arithmetic (csrc/gemm_simt.cuh) and of the two epilogues built on it,
operation for operation, so that the device results can be checked bit for bit.

* gemm_nt:    acc[m, n] = fmaf chain over k = 0, 1, ..., K-1 of A[m, k] * B[n, k], starting from +0.  The kernel's K
              padding adds fmaf(0, 0, acc) = acc, which changes no bit, so it is not emulated.
* row_sqnorm: row_sqnorm_kernel (csrc/sqdist.cu): lane l of a warp accumulates fmaf(x_k, x_k, s) over k = l, l + 32,
              ..., then warp_sum (csrc/common.cuh) adds v[lane ^ o] for o = 16, 8, 4, 2, 1; lane 0 holds the norm.
* sqdist:     SqDistEpilogue::one: d2 = (a + b) - 2 dot (2 dot is exact, so a contraction cannot change it), clamp
              d2 < 0 to 0 (NaN passes), __fsqrt_rn, and r * r when squared.
* bias_act:   BiasActEpilogue (csrc/mlp.cu) up to the activation: acc + bias, then fmaf(t, tcol, .).

fma32 is a correctly rounded fp32 fused multiply-add: the float64 product of two fp32 values is exact; the float64 sum
s of it and the addend is rounded, and TwoSum recovers that rounding error e exactly.  Rounding s to fp32 is then the
correctly rounded result except when s lies exactly on an fp32 midpoint (any value strictly between the exact sum and
s would be a float64 closer to the sum than s), and there the sign of e decides.  The library is built without fast
math, so the device's fmaf, adds, multiplies and square roots are IEEE round-to-nearest-even with subnormals."""
import numpy as np

F32 = np.float32
F64 = np.float64


def _f32_neighbours(s):
    """(lo, hi): the fp32 values below and above the float64 s (equal where s is an fp32 value)."""
    r = s.astype(F32)
    r64 = r.astype(F64)
    up = r64 < s
    dn = r64 > s
    lo = np.where(dn, np.nextafter(r, F32(-np.inf)), r)
    hi = np.where(up, np.nextafter(r, F32(np.inf)), r)
    return lo, hi


def _as_value(v):
    """float64 value of an fp32 array, with +-inf standing for +-2^128 (the rounding neighbour past FLT_MAX)."""
    d = v.astype(F64)
    return np.where(np.isinf(d), np.copysign(2.0 ** 128, d), d)


def fma32(a, b, c):
    """Correctly rounded fp32 fmaf(a, b, c), elementwise on broadcastable fp32 arrays."""
    a, b, c = (np.asarray(v, dtype=F32) for v in (a, b, c))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a.astype(F64) * b.astype(F64)  # exact: 48 significant bits, no under- or overflow in float64
        cc = c.astype(F64)
        s = p + cc
        bb = s - p
        e = (p - (s - bb)) + (cc - bb)  # TwoSum: s + e == p + c exactly
        r = s.astype(F32)
        tie = np.isfinite(s) & (e != 0)
        if not tie.any():
            return r
        lo, hi = _f32_neighbours(s)
        mid = tie & (lo != hi) & (0.5 * (_as_value(lo) + _as_value(hi)) == s)
        return np.where(mid, np.where(e > 0, hi, lo), r).astype(F32)


def gemm_nt(A, B):
    """(M, N) fp32: the kernel's accumulator for A (M, K) and B (N, K), one fmaf per k in ascending order from +0."""
    A = np.asarray(A, dtype=F32)
    B = np.asarray(B, dtype=F32)
    acc = np.zeros((A.shape[0], B.shape[0]), dtype=F32)
    for k in range(A.shape[1]):
        acc = fma32(A[:, k, None], B[None, :, k], acc)
    return acc


def row_sqnorm(X):
    """(rows,) fp32 |x_r|^2 in the order of row_sqnorm_kernel: 32 lane-strided fmaf chains and the xor butterfly."""
    X = np.asarray(X, dtype=F32)
    rows, d = X.shape
    # lanes >= d hold +0 (and every lane holds +0, a positive value or NaN), so butterfly steps o >= p, with p the
    # power of two >= min(d, 32), add +0 to every lane value and change no bit: only the first p lanes are kept
    p = 1 << (min(d, 32) - 1).bit_length()
    lanes = np.zeros((rows, p), dtype=F32)
    for k in range(d):
        lanes[:, k % 32] = fma32(X[:, k], X[:, k], lanes[:, k % 32])
    idx = np.arange(p)
    o = p // 2
    while o:
        lanes = (lanes + lanes[:, idx ^ o]).astype(F32)
        o //= 2
    return lanes[:, 0]


def sqdist_epilogue(dot, a, b, squared):
    """SqDistEpilogue::one for the accumulator ``dot`` and the row norms a (rows, 1) and b (1, cols)."""
    dot, a, b = (np.asarray(v, dtype=F32) for v in (dot, a, b))
    with np.errstate(invalid="ignore", over="ignore"):
        d2 = ((a + b) - F32(2.0) * dot).astype(F32)
        v = np.where(d2 < 0, F32(0.0), d2).astype(F32)
        r = np.sqrt(v).astype(F32)
        return (r * r).astype(F32) if squared else r


def sqdist(x0, x1, squared=1):
    """The cost matrix cfm_sqdist_f32 computes on the SIMT path (algo 1)."""
    return sqdist_epilogue(gemm_nt(x0, x1), row_sqnorm(x0)[:, None], row_sqnorm(x1)[None, :], squared)


def cost_max(M):
    """The kernel's cost_max: atomic max of the non-negative entries from 0, so NaN entries never enter it."""
    M = np.asarray(M, dtype=F32)
    ok = ~np.isnan(M)
    return F32(M[ok].max()) if ok.any() and M[ok].max() > 0 else F32(0.0)


def bias_act_pre(acc, bias, t=None, tcol=None):
    """BiasActEpilogue before its activation: acc + bias, then fmaf(t, tcol, .) for the first layer's time column."""
    v = (np.asarray(acc, dtype=F32) + np.asarray(bias, dtype=F32)[None, :]).astype(F32)
    if tcol is not None:
        v = fma32(F32(t), np.asarray(tcol, dtype=F32)[None, :], v)
    return v
