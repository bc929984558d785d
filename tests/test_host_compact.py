"""NumPy emulation of the 3-byte fixed-point cost format of the factored Sinkhorn sweep (sinkhorn_v2.cu):
the float64 encode of the exponent e = M*c2 - kappa, the 12-byte packing of 4 columns, and the decode through the
bit pattern 0x4B000000 | q (the float 2^23 + q) in fp32.  The decoded exponent must be within half a quantum
(span * 2^-24) plus one fp32 ulp of the exact one, for spans up to the factored path's limit of 40."""
import numpy as np
import pytest

LOG2E = np.float32(1.4426950408889634)
QMAX = 8388607  # 2^23 - 1


def _constants(reg, cmax):
    """c2, kappa as the kernel forms them (normalised cost): fp32 arithmetic."""
    c2 = np.float32(-LOG2E / np.float32(np.float32(reg) * np.float32(cmax)))
    kappa = np.float32(c2 * np.float32(cmax))
    return c2, kappa


def _encode(M, c2, kappa):
    qa = np.float32(np.float64(-kappa) / QMAX)
    qinv = 1.0 / np.float64(qa) if qa > 0 else 0.0
    e = M.astype(np.float64) * np.float64(c2) - np.float64(kappa)
    q = np.clip(np.rint(e * qinv), 0, QMAX).astype(np.uint32)
    q = q.reshape(-1, 4)
    w0 = q[:, 0] | (q[:, 1] << 24)
    w1 = (q[:, 1] >> 8) | (q[:, 2] << 16)
    w2 = (q[:, 2] >> 16) | (q[:, 3] << 8)
    return np.stack([w0, w1, w2], 1).astype(np.uint32), qa


def _funnel_r(lo, hi, s):
    return ((lo.astype(np.uint64) | (hi.astype(np.uint64) << 32)) >> s).astype(np.uint32)


def _decode(w, qa):
    w0, w1, w2 = w[:, 0], w[:, 1], w[:, 2]
    ent = np.stack([w0, _funnel_r(w0, w1, 24), _funnel_r(w1, w2, 16), w2 >> 8], 1)
    F = (np.uint32(0x4B000000) | (ent & np.uint32(0xFFFFFF))).view(np.float32)
    return ((F - np.float32(8388608.0)) * qa).astype(np.float32).reshape(-1)


@pytest.mark.parametrize("span", [1.0, 10.0, 28.85, 39.99])
def test_compact_cost_format_error_bound(span):
    rng = np.random.default_rng(int(span * 100))
    cmax = np.float32(1973.25)
    reg = float(LOG2E) / span  # normalised cost: span = log2(e) / reg
    c2, kappa = _constants(reg, cmax)
    assert abs(-float(kappa) - span) < 1e-4 * span
    quantum = float(cmax) / QMAX
    k = rng.integers(0, QMAX, size=2048).astype(np.float64)
    edges = np.array([0.0, cmax, np.nextafter(cmax, np.float32(0)), np.float32(quantum), np.float32(2 * quantum),
                      np.float32(cmax / 2), np.nextafter(np.float32(0), np.float32(1))], dtype=np.float32)
    M = np.concatenate([rng.uniform(0, cmax, 40000).astype(np.float32),
                        (k * quantum).astype(np.float32),          # values one quantum apart
                        ((k + 1) * quantum).astype(np.float32),
                        ((k + 0.5) * quantum).astype(np.float32),  # half-way between two codes
                        edges, np.zeros(1, np.float32)])
    M = np.minimum(M, cmax)
    M = np.concatenate([M, np.zeros((-len(M)) % 4, np.float32)])
    w, qa = _encode(M, c2, kappa)
    # byte 2 of each entry (group bytes 2, 5, 8, 11) has its top bit clear
    assert np.all((w[:, 0] >> 23) & 1 == 0) and np.all((w[:, 1] >> 15) & 1 == 0)
    assert np.all((w[:, 2] >> 7) & 1 == 0) and np.all(w[:, 2] >> 31 == 0)
    dec = _decode(w, qa)
    exact = M.astype(np.float64) * np.float64(c2) - np.float64(kappa)
    half_quantum = 0.5 * float(qa)
    assert half_quantum <= span * 2.0 ** -24 * (1 + 2.0 ** -20)
    ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
    err = np.abs(dec.astype(np.float64) - exact)
    assert np.all(err <= half_quantum + ulp), err.max()
    # the fp32 path's own exponent fl(M*c2 - kappa) has half an ulp; the compact one stays within a quantum of it
    fp32 = np.float32(M * c2 + np.float32(-kappa)).astype(np.float64)
    assert np.abs(dec - fp32).max() <= 2 * half_quantum + float(np.spacing(np.float32(span)))


def test_compact_cost_format_round_trips_the_codes():
    rng = np.random.default_rng(7)
    q = np.concatenate([rng.integers(0, QMAX + 1, 4000), [0, QMAX, 1, QMAX - 1]]).astype(np.uint32)
    q0, q1, q2, q3 = q.reshape(-1, 4).T
    w = np.stack([q0 | (q1 << 24), (q1 >> 8) | (q2 << 16), (q2 >> 16) | (q3 << 8)], 1).astype(np.uint32)
    dec = _decode(w, np.float32(1.0))  # qa = 1: the decode returns q itself, exactly
    assert np.array_equal(dec.astype(np.uint32), q)
