"""NumPy emulation of the 22-bit chunks of the Sinkhorn cost copy (sinkhorn_v2.cu, KG = 4): thread t's 16 entries
of a row (4 groups of 4 columns at 4 t + 2048 k) packed into the 11 words at word 11 t, entry i at bit 22 i, the
kernel's word-by-word packing loop, the decode of each field, and the rule that makes a chunk narrow: its smallest
cost encodes below 2^22 (the encode is monotone in M, so that code is the chunk's largest) and no cost is NaN."""
import numpy as np
import pytest

from test_host_compact import QMAX, _constants, _decode

NT, WORDS, LIMIT = 512, 11, 1 << 22


def _pack_row(q):
    """The kernel's prologue loop for one row: q[n1 = 8192] codes -> 512 * 11 words."""
    words = np.zeros((NT, WORDS), dtype=np.uint32)
    for t in range(NT):
        acc = 0
        for k in range(4):
            for c in range(4):
                qi = int(q[4 * t + 2048 * k + c])
                bit = 22 * (4 * k + c)
                sh = bit & 31
                acc |= (qi << sh) & 0xFFFFFFFF
                if sh + 22 >= 32:
                    words[t, bit >> 5] = acc
                    acc = qi >> (32 - sh) if sh + 22 > 32 else 0
    return words


def _field(w, i):
    """v2_q22_field: entry i of a thread's 11 words (rows of w), before the 22-bit mask."""
    bit = 22 * i
    wd, sh = bit >> 5, bit & 31
    if sh + 22 <= 32:
        return w[:, wd] >> np.uint32(sh)
    return ((w[:, wd].astype(np.uint64) | (w[:, wd + 1].astype(np.uint64) << np.uint64(32))) >> np.uint64(sh)).astype(np.uint32)


def _decode22(f, qa):
    F = (np.uint32(0x4B000000) | (f & np.uint32(0x3FFFFF))).view(np.float32)
    return ((F - np.float32(8388608.0)) * qa).astype(np.float32)


def _q(M, c2, kappa):
    """v2_encode in float64: the code of every entry."""
    qa = np.float32(np.float64(-kappa) / QMAX)
    qinv = 1.0 / np.float64(qa) if qa > 0 else 0.0
    e = M.astype(np.float64) * np.float64(c2) - np.float64(kappa)
    with np.errstate(invalid="ignore"):
        q = np.rint(e * qinv)
    return np.clip(np.nan_to_num(q, nan=0.0), 0, QMAX).astype(np.int64), qa


def cost_with_code(target, cmax, c2, kappa):
    """An fp32 cost whose code is exactly `target` (the codes are monotone in M: walk fp32 neighbours)."""
    m = np.float32(cmax * (1.0 - target / QMAX))
    for _ in range(64):
        qm = _q(np.array([m]), c2, kappa)[0][0]
        if qm == target:
            return m
        m = np.nextafter(m, np.float32(np.inf if qm > target else -np.inf))
    raise AssertionError(f"no fp32 cost with code {target}")


def test_narrow_layout_round_trips_and_decodes_like_the_3_byte_one():
    rng = np.random.default_rng(3)
    q = rng.integers(0, LIMIT, size=8192).astype(np.uint32)
    q[:16] = [0, LIMIT - 1, 1, LIMIT - 2, LIMIT - 1, 0, LIMIT - 1, LIMIT - 1, 0, 0, 1, LIMIT - 1, 2, 3, LIMIT - 1, 0]
    q[4 * 511 + 2048 * 3:] = LIMIT - 1  # the last thread's last group: its entry 15 ends exactly at word 10's top bit
    w = _pack_row(q)
    assert w.shape == (512, 11) and 512 * 11 * 4 == 22528
    cols = (4 * np.arange(NT)[:, None, None] + 2048 * np.arange(4)[None, :, None] + np.arange(4)[None, None, :]).reshape(NT, 16)
    qa = np.float32(28.853900817779268 / QMAX)
    # the 3-byte decode of the same codes, 4 columns per 12-byte group
    q4 = q.reshape(-1, 4)
    w3 = np.stack([q4[:, 0] | (q4[:, 1] << 24), (q4[:, 1] >> 8) | (q4[:, 2] << 16), (q4[:, 2] >> 16) | (q4[:, 3] << 8)],
                  1).astype(np.uint32)
    ref = _decode(w3, qa)
    for i in range(16):
        f = _field(w, i)
        assert np.array_equal(f & np.uint32(0x3FFFFF), q[cols[:, i]]), i
        # the same float as the 3-byte stream's decode: e' is bit-identical
        assert np.array_equal(_decode22(f, qa).view(np.uint32), ref[cols[:, i]].view(np.uint32)), i


def test_narrow_word_loads_are_free_of_bank_conflicts():
    for j in range(WORDS):
        banks = (WORDS * np.arange(32) + j) % 32
        assert len(set(banks.tolist())) == 32


def test_narrow_pitch_rule():
    """22-bit rows (512 x 44 bytes) only where they are shorter than the 3-byte pitch align16(3 n1): n1 > 7509."""
    n1 = np.arange(4096 + 4, 8193, 4)
    ldc = (3 * n1 + 15) // 16 * 16
    narrow = 22528 < ldc
    assert narrow[n1 == 7508].item() is False and narrow[n1 == 7512].item() is True
    assert np.array_equal(narrow, n1 > 7509)


@pytest.mark.parametrize("seed", range(6))
def test_width_rule_is_exact_on_random_chunks(seed):
    """The code of the chunk's smallest cost is the chunk's largest code, so one comparison decides the width."""
    rng = np.random.default_rng(seed)
    cmax = np.float32(rng.uniform(10.0, 3000.0))
    reg = rng.uniform(0.04, 0.5)
    c2, kappa = _constants(reg, cmax)
    for _ in range(200):
        lo = rng.uniform(0.0, 0.8)
        M = (cmax * rng.uniform(lo, 1.0, size=(2, 64))).astype(np.float32)
        if rng.random() < 0.3:  # a cost right at the boundary between the widths
            M[rng.integers(0, 2), rng.integers(0, 64)] = cost_with_code(LIMIT - 1 + rng.integers(0, 2), cmax, c2, kappa)
        q, _ = _q(M, c2, kappa)
        by_max = q.max() < LIMIT
        by_min = _q(np.array([M.min()]), c2, kappa)[0][0] < LIMIT
        assert by_max == by_min
    # NaN: the encode maps it to 0, so only the explicit flag makes its chunk wide
    M = np.full((2, 8), cmax, np.float32)
    M[1, 3] = np.nan
    assert _q(M, c2, kappa)[0].max() == 0 and np.isnan(M).any()


def test_boundary_codes_exist_in_fp32():
    """The GPU tests place costs whose codes are exactly 2^22 - 1 and 2^22: both exist at C2-like constants."""
    cmax = np.float32(2044.9)
    c2, kappa = _constants(0.05, cmax)
    for target in (LIMIT - 1, LIMIT):
        assert _q(np.array([cost_with_code(target, cmax, c2, kappa)]), c2, kappa)[0][0] == target
