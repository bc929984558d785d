"""The edge cases of the tensor-core samplers without a device (tests/tc_sampler_cases.py): the table reaches every
listed code path of the Hutchinson field, the dopri5 stage array, the SDE pair forward and the SDE step grid, on an
H100's 132 SMs and on parts with fewer; the restated launch arithmetic gives the launches the GPU tests are named
for; and the constants it restates are the sources'."""
import os
import re

import pytest

import tc_sampler_cases as tc

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cfm_b200", "csrc")


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_the_table_reaches_every_path(sms):
    reached = tc.reached(sms)
    missing = sorted(tc.REQUIRED - set(reached))
    assert not missing, (sms, missing)


def test_each_path_is_lost_with_the_cases_that_reach_it(monkeypatch):
    """Dropping every case that reaches a path (here: the multi-tile batches, the pair's S = 1 batch) loses it."""
    with monkeypatch.context() as mp:
        mp.setattr(tc, "FIELD_SHAPES", [s for s in tc.FIELD_SHAPES if not isinstance(s[0], str)])
        assert "CTA runs 2+ tiles: tangent hidden" not in tc.reached(132)
    monkeypatch.setattr(tc, "PAIR_SHAPES", [s for s in tc.PAIR_SHAPES if s[0] != 128])
    assert "pair: S = 1" not in tc.reached(132)


def test_launch_arithmetic_on_132_sms():
    sms = tc.H100_SMS
    # the MNIST-shape batch: 20 M tiles x 7 N tiles = 140 output-layer tiles on 132 CTAs, hidden layers 40 tiles
    B = tc.batch("128*ceil(SMs/7)+1", sms)
    assert B == 2433 and tc.gemm_launch(B, 784, sms) == (20, 7, 132) and tc.gemm_launch(B, 256, sms) == (20, 2, 40)
    assert tc.field_paths(B, 784, 256, sms) == {
        "partial output chunk: primal", "partial output chunk: tangent", "layer-0 K tail", "one-row last M tile",
        "CTA runs 2+ tiles: primal output", "CTA runs 2+ tiles: tangent output"}
    assert tc.field_paths(129, 40, 136, sms) >= {"8-column hidden N tile", "partial hidden chunk: tangent",
                                                 "hidden K tail", "layer-0 K tail", "partial output chunk: primal"}
    # dopri5's stage outputs: B (D + 1) = 1, 2, 3 mod 4
    assert [tc.stage_offsets(B, 64) for B in (129, 130, 131, 256)] == [[0, 4, 8, 12], [0, 8], [0, 4, 8, 12], [0]]
    # the pair: one slab per net; one slab per CTA; two CTAs with a second, score slab; S = SMs + 1
    assert tc.pair_slabs(128, sms)[:2] == (1, 2)
    assert tc.pair_slabs(64 * sms, sms)[:2] == (66, 132)
    S, grid, seqs = tc.pair_slabs(64 * sms + 1, sms)
    assert (S, grid) == (67, 132) and seqs[0] == [(0, 0, 128), (1, 65, 128)] and seqs[1] == [(0, 1, 128), (1, 66, 1)]
    S, grid, seqs = tc.pair_slabs(128 * sms + 1, sms)
    assert (S, grid) == (133, 132) and seqs[0] == [(0, 0, 128), (0, 132, 1), (1, 131, 128)]
    S, grid, seqs = tc.pair_slabs(3 * 128 * sms - 5, sms)
    assert (S, grid) == (396, 132) and seqs[131][2:4] == [(0, 395, 123), (1, 131, 128)]
    # the noise grid: four steps of 0.07, then one of 0.03
    g = tc.sde_grid(tc.NOISE_TS, tc.NOISE_DT)
    assert len(g) == 6 and abs(float(g[-1] - g[-2]) - 0.03) < 1e-6
    assert list(tc.noise_rows(300)) == [0, 1, 2, 127, 128, 255, 256, 297, 298, 299]


def test_restated_constants_are_the_sources():
    def src(name):
        with open(os.path.join(CSRC, name)) as f:
            return f.read()
    assert re.search(r"constexpr int kTM = (\d+), kTN = (\d+);", src("gemm_tc.cuh")).groups() == (str(tc.TM),
                                                                                                 str(tc.TN))
    assert re.search(r"constexpr int kHK = (\d+);", src("gemm_h3.cuh")).group(1) == str(tc.HK)
    assert re.search(r"p\.tiles_m = \(n0 \+ kTM - 1\) / kTM;", src("gemm_tc.cuh"))
    assert "const int tm = tile % p.tiles_m, tn = tile / p.tiles_m;" in src("gemm_tc.cuh")  # M-fastest
    assert "if (grid > sm_count()) grid = sm_count();" in src("gemm_tc.cuh")
    cnf = src("cnf_tc.cu")
    assert cnf.count(f"const bool full = col0 + {tc.CHUNK} <= n1;") == 2
    mlp = src("mlp_h3.cu")
    assert "int grid = 2 * ((batch + kTM - 1) / kTM);\n  if (grid > sm_count()) grid = sm_count();" in mlp
    assert "auto net_of = [&](int v) { return (NETS > 1 && v >= num_slabs) ? 1 : 0; };" in mlp
