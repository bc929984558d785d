"""The float64 restatement of the device's Sinkhorn loop (tests/sinkhorn_oracle.py) against POT's sinkhorn_log and on
tiny inputs whose every step can be checked by hand.  No device needed."""
import math

import numpy as np
import torch
from scipy.special import logsumexp

from oracle import ot as oot
from sinkhorn_oracle import FLAG_NONFINITE, FLAG_NOT_CONVERGED, mr_exact, mr_precise, sinkhorn_device_loop


def _cost(n0, n1, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.cdist(torch.randn(n0, 3, generator=g, dtype=torch.float64),
                       torch.randn(n1, 3, generator=g, dtype=torch.float64) + 0.2) ** 2


def test_restatement_equals_pot_sinkhorn_log():
    """With a float64 M and check_every = 10, the device loop computes POT's iterates: the same iteration count
    (niter + 1), potentials and err, both when stopThr stops the solve and when numItermax does (a last iteration that
    is no check)."""
    M = _cost(30, 45, 0)
    reg = 0.5
    for iters, thr in ((1000, 1e-9), (1000, 1e-5), (37, 0.0), (41, 0.0), (1, 0.0)):
        _, log = oot.sinkhorn_log(oot.unif(30), oot.unif(45), M.numpy(), reg, numItermax=iters, stopThr=thr,
                                  warn=False, log=True)
        r = sinkhorn_device_loop(-M / reg, iters, 10, thr)
        assert r.iters == log["niter"] + 1, (iters, thr)
        assert np.abs(r.u.numpy() - log["log_u"]).max() < 1e-12
        assert np.abs(r.v.numpy() - log["log_v"]).max() < 1e-12
        assert abs(r.err - log["err"]) < 1e-12
        assert bool(r.flags & FLAG_NOT_CONVERGED) == (thr == 0.0 or r.err >= thr)
    assert sinkhorn_device_loop(-M / reg, 1000, 10, 1e-9).iters < 1000


def _by_hand(Mr, v):
    """one row pass and one column pass of the device loop, in NumPy"""
    n0, n1 = Mr.shape
    u = -math.log(n0) - logsumexp(Mr + v[None, :], axis=1)
    return u, -math.log(n1) - logsumexp(Mr + u[:, None], axis=0)


def test_single_iteration_and_non_check_last_iteration_by_hand():
    Mr = np.array([[-1.0, -3.0, 0.5], [-2.0, 0.0, -0.25]])
    v0 = -math.log(3) - logsumexp(Mr, axis=0)  # prologue: u = 0
    u1, v1 = _by_hand(Mr, v0)
    r = sinkhorn_device_loop(torch.from_numpy(Mr), 1, 10)
    # one iteration: its row pass used v0, and v0 is what is returned (not the v1 the check computed)
    assert r.iters == 1 and r.flags == FLAG_NOT_CONVERGED and [c[0] for c in r.checks] == [0]
    np.testing.assert_allclose(r.u.numpy(), u1, rtol=0, atol=1e-15)
    np.testing.assert_allclose(r.v.numpy(), v0, rtol=0, atol=1e-15)
    assert abs(r.err - np.linalg.norm(np.expm1(v0 - v1) / 3)) < 1e-16
    # 5 iterations checked every 3: checks at 0 and 3; iteration 4 is the last and no check, so it updates u only
    v = v0
    us, vs = [], []
    for _ in range(5):
        u, vn = _by_hand(Mr, v)
        us.append(u), vs.append(v)
        v = vn
    r = sinkhorn_device_loop(torch.from_numpy(Mr), 5, 3)
    assert r.iters == 5 and [c[0] for c in r.checks] == [0, 3]
    np.testing.assert_allclose(r.u.numpy(), us[4], rtol=0, atol=1e-14)
    np.testing.assert_allclose(r.v.numpy(), vs[4], rtol=0, atol=1e-14)
    assert r.err == r.checks[-1][1] and abs(r.err - np.linalg.norm(np.expm1(vs[3] - vs[4]) / 3)) < 1e-16
    # 4 iterations checked every 3: the last is a check, and the v returned is the one its row pass used
    r = sinkhorn_device_loop(torch.from_numpy(Mr), 4, 3)
    assert r.iters == 4 and [c[0] for c in r.checks] == [0, 3]
    np.testing.assert_allclose(r.v.numpy(), vs[3], rtol=0, atol=1e-14)


def test_stop_threshold_stops_on_the_first_check_below_it():
    Mr = -_cost(6, 5, 1) / 0.7
    full = sinkhorn_device_loop(Mr, 200, 3)
    errs = [e for _, e in full.checks]
    k = 4
    thr = math.sqrt(errs[k - 1] * errs[k])
    r = sinkhorn_device_loop(Mr, 200, 3, thr)
    assert r.iters == full.checks[k][0] + 1 and r.flags == 0 and r.err == errs[k]
    assert sinkhorn_device_loop(Mr, 200, 3, 2 * errs[0]).iters == 1  # stops on the first iteration


def test_stall_rule():
    """Stops at the first check after the first one whose err improved by less than stall_tol while
    err * sqrt(n1) < 1e-5, and never without stall_tol."""
    Mr = -_cost(7, 9, 2) / 0.4
    full = sinkhorn_device_loop(Mr, 3000, 10)
    errs = [e for _, e in full.checks]
    assert full.iters == 3000 and full.flags == FLAG_NOT_CONVERGED
    # err falls by a factor of about 4.6 per check, then reaches exactly 0
    ratios = [errs[k] / errs[k - 1] for k in range(1, 20)]
    assert 0.15 < min(ratios) and max(ratios) < 0.3 and errs[-1] == 0.0
    # stall_tol = 0.9 fires on every check that has a predecessor, but only once err * sqrt(n1) < 1e-5: check 7
    first = next(k for k in range(len(errs)) if errs[k] * 3 < 1e-5)
    assert first == 7
    r = sinkhorn_device_loop(Mr, 3000, 10, 0.0, 0.9)
    assert r.iters == full.checks[first][0] + 1 and r.flags == 0 and r.err == errs[first]
    # stall_tol = 0.5: no check improves by less than half, and 0 > 0.5 * 0 is false
    assert sinkhorn_device_loop(Mr, 3000, 10, 0.0, 0.5).iters == 3000


def test_nan_cost():
    Mr = torch.tensor([[-1.0, float("nan"), 0.5], [-2.0, 0.0, -0.25]])
    r = sinkhorn_device_loop(Mr.double(), 1, 10)
    # the prologue makes v_1 NaN; every row sees column 1, so all of u is NaN after one iteration
    assert r.v.isnan().tolist() == [False, True, False] and r.u.isnan().all()
    r = sinkhorn_device_loop(Mr.double(), 25, 10, stop_thr=1.0, stall_tol=0.5)
    assert r.iters == 25 and r.flags == FLAG_NONFINITE | FLAG_NOT_CONVERGED and math.isnan(r.err)
    assert r.u.isnan().all() and r.v.isnan().all()


def test_exponent_forms():
    """mr_precise is NumPy's fp32 rounding of -(M / cmax) / reg; mr_exact the float64 quotient."""
    g = np.random.RandomState(3)
    M = (g.rand(64, 33) * 7).astype(np.float32)
    cmax, reg = np.float32(M.max()), np.float32(0.013)
    want = (-((M / cmax).astype(np.float32) / reg)).astype(np.float32)
    assert np.array_equal(mr_precise(torch.from_numpy(M), float(reg), float(cmax)).numpy(), want.astype(np.float64))
    want = (-(M / reg)).astype(np.float32)
    assert np.array_equal(mr_precise(torch.from_numpy(M), float(reg)).numpy(), want.astype(np.float64))
    got = mr_exact(torch.from_numpy(M), float(reg), float(cmax)).numpy()
    np.testing.assert_allclose(got, -M.astype(np.float64) / (float(reg) * float(cmax)), rtol=1e-15)
