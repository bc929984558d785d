"""Every Sinkhorn solver body (cfm_sinkhorn_log_f32) against the float64 restatement of the device loop
(tests/sinkhorn_oracle.py): iterates, stopping iteration, err and status word, through the C ABI so that
check_every, a null cost_max and a pitched or offset M can be passed.

Bodies (status[2] arithmetic, status[3] kernel variant):
    v2 factored (0, 3), v2 log-domain (0, 2), v2 on the 3-byte stream (0, 4)       sinkhorn_v2_kernel
    generic fp32 (0, 0), float64 (1, 0), mixed screened / unscreened (2, 0)         sinkhorn_kernel, sinkhorn_run
    seeded mixed (2, 1)                                                             sinkhorn_kernel, sinkhorn_run_seeded
Gates on the potentials, per arithmetic: float64 1e-6 absolute at |M/reg| ~ 1e4, mixed 4e-6, fp32 2e-5 on
gauge-fixed potentials (u + mean v, v - mean v).  err: float64 1e-9 relative (or its rounding floor), fp32 and mixed
the body's err floor, measured here as the largest err the body reports after many iterations.  A stop_thr is admitted only
at 100 x the floor (float64: the rounding floor of err from potentials as large as M/reg).  Shapes that depend on the
device (grid sizes, the 3-byte stream's L2 threshold) are computed from its properties by the launchers' rules."""
import math
import re
import subprocess

import numpy as np
import pytest
import torch

from cfm_b200 import _ffi
from sinkhorn_oracle import FLAG_NONFINITE, FLAG_NOT_CONVERGED, mr_exact, mr_precise, sinkhorn_device_loop

DEV = torch.device("cuda:0")
PREC = {"auto": -1, "fp32": 0, "fp64": 1, "fp32-generic": 2, "fp64-mixed": 3, "fp64-mixed-unscreened": 4}
GATE = {0: 2e-5, 1: 1e-6, 2: 4e-6}  # potentials, per status[2]
FLOOR_ITERS = (1400, 1600, 1800, 2000)  # the err floor: the largest err reported after these many iterations
WORST = {}                           # body -> largest potential error / gate seen (printed with -s)
ERR_RATIO = {}                       # body -> largest |err - restatement's err| / tolerance seen (printed with -s)


@pytest.fixture(scope="module", autouse=True)
def _report():
    """after the module: the largest errors of each body as fractions of their gates, for the record"""
    yield
    for k, v in sorted(WORST.items()):
        print(f"\n[potentials / gate] {k}: {v:.3f}   [err / tolerance] {ERR_RATIO.get(k, 0.0):.3f}")


# ---------------------------------------------------------------------------------------------------- helpers
def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _grid():
    """Both kernels' grid before the cap by n0.  v2: the SM count.  Generic: SMs x min(occupancy, 2), capped by 512;
    the occupancy is 1 because every sinkhorn_kernel instantiation takes more than 64 registers per thread, so 512
    threads fill more than half of an SM's 64K registers (test_compiled_sinkhorn_instantiations_are_the_tested_ones
    reads the register counts out of the library)."""
    return min(_sms(), 512)


def _streams(n0, n1):
    return n0 * n1 * 4 > torch.cuda.get_device_properties(DEV).L2_cache_size // 4 * 3


def _points(n0, n1, d, seed, offset=0.0):
    """squared distances (+ offset) of Gaussian points; low d spreads them, so that the solve converges slowly"""
    g = torch.Generator().manual_seed(seed)
    x0 = torch.randn(n0, d, generator=g, dtype=torch.float64).to(DEV)
    x1 = (torch.randn(n1, d, generator=g, dtype=torch.float64) + 0.1).to(DEV)
    return ((x0 * x0).sum(1)[:, None] + (x1 * x1).sum(1)[None, :] - 2 * x0 @ x1.T).clamp_min(0).add(offset).float()


def _blocks(n0, n1, seed):
    """uniform costs plus 0.5 between the first half of the rows and the last 60 % of the columns and between the
    other two blocks: a plan that must carry mass across the gap converges slowly enough to have err decrease by
    less than 100x per check over several checks"""
    g = torch.Generator().manual_seed(seed)
    M = torch.rand(n0, n1, generator=g).to(DEV) * 0.5
    cross = (torch.arange(n0, device=DEV) < n0 // 2)[:, None] != (torch.arange(n1, device=DEV) < 2 * n1 // 5)[None, :]
    return M + 0.5 * cross


def _place(M, ldm=None, offset=0):
    """M in an n0 x ldm buffer whose padding columns are NaN (a read of one poisons the solve), optionally
    starting `offset` floats into its allocation"""
    n0, n1 = M.shape
    ldm = ldm or (n1 + 3) // 4 * 4
    flat = torch.full((offset + n0 * ldm + 4,), float("nan"), dtype=torch.float32, device=DEV)
    view = flat[offset:offset + n0 * ldm].view(n0, ldm)
    view[:, :n1] = M
    return view


class Out:
    def __init__(self, lu, lv, st, err, launches):
        self.lu, self.lv, self.st, self.err, self.launches = lu, lv, st, err, launches


def _solve(M, n1, reg, cmax, normalize, precision, iters, stop_thr=0.0, check_every=10, stall_tol=0.0, ws=None):
    L = _ffi.lib()
    n0 = M.shape[0]
    lu = torch.full((n0,), 7.0, dtype=torch.float64, device=DEV)
    lv = torch.full((n1,), 7.0, dtype=torch.float64, device=DEV)
    st = torch.full((4,), -9, dtype=torch.int32, device=DEV)
    err = torch.zeros(1, dtype=torch.float64, device=DEV)
    if ws is None:
        ws = torch.zeros(L.cfm_sinkhorn_workspace_bytes(n0, n1), dtype=torch.uint8, device=DEV)
    before = L.cfm_launch_count()
    _ffi.check(L.cfm_sinkhorn_log_f32(
        _ffi.ptr(M), n0, n1, M.stride(0), float(reg), _ffi.ptr(cmax), int(normalize), iters, float(stop_thr),
        check_every, PREC[precision], float(stall_tol), _ffi.ptr(lu), _ffi.ptr(lv), _ffi.ptr(st), _ffi.ptr(err),
        _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(DEV)), "cfm_sinkhorn_log_f32")
    launches = L.cfm_launch_count() - before
    torch.cuda.synchronize()
    return Out(lu, lv, st.cpu().tolist(), float(err.item()), launches)


class Problem:
    """A cost matrix, its solve settings and the body they must reach; Mr in the form that body computes with."""

    def __init__(self, M, reg, normalize, precision, body, ldm=None, offset=0, null_cmax=False):
        self.n0, self.n1 = M.shape
        self.cmax = None if null_cmax else M.max().reshape(1).float()
        self.Mbuf = _place(M, ldm, offset)
        self.reg, self.normalize, self.precision, self.body = reg, normalize, precision, body
        scale = float(self.cmax) if normalize else None
        self.Mr = (mr_exact if body[0] == 0 else mr_precise)(M, reg, scale)

    def solve(self, iters, **kw):
        out = _solve(self.Mbuf, self.n1, self.reg, self.cmax, self.normalize, self.precision, iters, **kw)
        assert tuple(out.st[2:]) == self.body, (out.st, self.body)
        return out

    def ref(self, iters, **kw):
        return sinkhorn_device_loop(self.Mr, iters, **kw)


def _pot_err(out, ref, arith):
    """largest potential error, gauge-fixed for fp32"""
    lu, lv, ru, rv = out.lu, out.lv, ref.u, ref.v
    if arith == 0:
        lu, ru = lu + lv.mean(), ru + rv.mean()
        lv, rv = lv - lv.mean(), rv - rv.mean()
    return max((lu - ru).abs().max().item(), (lv - rv).abs().max().item())


def _f64_floor(p):
    """rounding floor of a float64 err: a few ulp of potentials as large as M/reg in each column's change of v"""
    return 64 * 2.0 ** -52 * p.Mr.abs().max().item() / math.sqrt(p.n1)


def _err_tol(p, ref_err, floor):
    if p.body[0] == 1:  # float64: 1e-9 relative, or its rounding floor
        return max(1e-9 * ref_err, floor)
    return floor


def _check(p, out, ref, floor, what):
    arith = p.body[0]
    e = _pot_err(out, ref, arith)
    WORST[p.name] = max(WORST.get(p.name, 0.0), e / GATE[arith])
    tol = _err_tol(p, ref.err, floor)
    ERR_RATIO[p.name] = max(ERR_RATIO.get(p.name, 0.0), abs(out.err - ref.err) / tol)
    assert e < GATE[arith], (what, e)
    assert abs(out.err - ref.err) <= tol, (what, out.err, ref.err)


# ------------------------------------------------------------------------------------------------ the bodies
def _v2_3byte_n0():
    return torch.cuda.get_device_properties(DEV).L2_cache_size // 4 * 3 // (4 * 4096) + 301


BODIES = {
    # name: (cost: None for _blocks or (point dimension, offset) for _points, n0, n1, reg, normalize, precision,
    # (status[2], status[3])).  The float64 body's costs are 2e4 + O(10) at reg 2: |M/reg| ~ 1e4 with a spread of a
    # few units.
    "v2_factored": (None, 768, 1024, 0.05, 1, "fp32", (0, 3)),
    "v2_log_domain": (None, 768, 1024, 0.03, 1, "fp32", (0, 2)),
    "v2_3byte": (None, _v2_3byte_n0, 4096, 0.05, 1, "fp32", (0, 4)),
    "generic_fp32": (None, 600, 1001, 0.05, 1, "fp32-generic", (0, 0)),
    "generic_f64": ((2, 2e4), 400, 515, 2.0, 0, "fp64", (1, 0)),
    "generic_mixed": ((16, 0.0), 64, 8200, 0.012, 1, "fp64-mixed", (2, 0)),
    "generic_mixed_unscreened": ((16, 0.0), 384, 512, 0.012, 1, "fp64-mixed-unscreened", (2, 0)),
    "seeded": ((16, 0.0), 512, 384, 0.012, 1, "auto", (2, 1)),
}
_CACHE = {}


def _cost(spec, n0, n1, seed):
    return _blocks(n0, n1, seed) if spec is None else _points(n0, n1, spec[0], seed, spec[1])


def _body(name, nan=False):
    key = (name, nan)
    if key not in _CACHE:
        d, n0, n1, reg, norm, prec, body = BODIES[name]
        n0 = n0() if callable(n0) else n0
        p = Problem(_cost(d, n0, n1, n0 + n1), reg, norm, prec, body)
        if nan:  # cost_max (taken above) stays finite, as the cost kernel leaves it
            p.Mbuf[3, 7] = float("nan")
            p.Mr[3, 7] = float("nan")
        p.name = name
        if name == "v2_3byte":
            assert _streams(n0, n1)
        _CACHE[key] = p
    return _CACHE[key]


def _floor(p):
    """the largest err the body reports at the end of long solves; float64: its rounding floor"""
    if p.body[0] == 1:
        return _f64_floor(p)
    if not hasattr(p, "floor"):
        p.floor = max(p.solve(k).err for k in FLOOR_ITERS)
        assert p.floor > 0
        print(f"\n[err floor] {p.name}: {p.floor:.3e}")
    return p.floor


FP32_MIXED = [n for n in BODIES if BODIES[n][6][0] != 1]


# ------------------------------------------------------------------ A. loop and stopping rule on every body
@pytest.mark.gpu
@pytest.mark.parametrize("check_every", [1, 3, 7, 10])
@pytest.mark.parametrize("name", list(BODIES))
def test_iterates_at_every_loop_edge(name, check_every):
    """stop_thr = 0: after max_iters in {1, 2, c - 1, c, c + 1, 3c, 3c + 1} the potentials, err (the last check's)
    and the status word are the restatement's; log_v is the v the last row pass used"""
    p = _body(name)
    floor = _floor(p)
    c = check_every
    for iters in sorted({1, 2, c - 1, c, c + 1, 3 * c, 3 * c + 1} - {0}):
        out = p.solve(iters, check_every=c)
        ref = p.ref(iters, check_every=c)
        assert out.st[1] == iters and out.st[0] == FLAG_NOT_CONVERGED, (iters, out.st)
        assert out.launches == (2 if p.precision == "auto" and p.body[1] != 0 else 1)
        _check(p, out, ref, floor, (iters, c))


def _stop_thresholds(p, c, floor):
    """stop_thr values at which a differing iteration count is a defect: every earlier check >= 1.5 thr, the
    stopping one <= thr / 1.5, thr >= 100 x the err floor (on every body, float64 included).  The first check
    (2 x its err) and the first and last admissible geometric means of consecutive checks."""
    errs = [e for _, e in p.ref(400, check_every=c).checks]
    out = [2 * errs[0]] if c == 10 and 2 * errs[0] >= 100 * floor else []
    ok = []
    for k in range(1, len(errs)):
        thr = math.sqrt(errs[k - 1] * errs[k])
        if min(errs[:k]) >= 1.5 * thr and errs[k] <= thr / 1.5 and thr >= 100 * floor:
            ok.append(thr)
    assert ok, (p.name, c)
    return out + sorted({ok[0], ok[-1]}, reverse=True)


@pytest.mark.gpu
@pytest.mark.parametrize("check_every", [3, 7, 10])
@pytest.mark.parametrize("name", list(BODIES))
def test_stop_threshold_stops_on_the_restatements_iteration(name, check_every):
    p = _body(name)
    floor = _floor(p)
    for thr in _stop_thresholds(p, check_every, floor):
        ref = p.ref(400, check_every=check_every, stop_thr=thr)
        out = p.solve(400, check_every=check_every, stop_thr=thr)
        assert ref.flags == 0 and out.st[0] == 0 and out.st[1] == ref.iters, (thr, out.st, ref.iters)
        _check(p, out, ref, floor, thr)  # log_v: the v of the stopping iteration


@pytest.mark.gpu
@pytest.mark.parametrize("name,reg", [(n, None) for n in FP32_MIXED] + [("seeded", 0.015)])
def test_stall_rule(name, reg):
    """stall_tol = 0.1 with an unreachable stop_thr: the solve ends on a check whose err * sqrt(n1) < 1e-5 and that
    improved on the previous check (rerun one check earlier) by less than 10 %; err is the float64 column error of
    the returned potentials within the floor; without stall_tol the solve runs to max_iters"""
    p = _body(name)
    if reg is not None:
        d, n0, n1, _, norm, prec, body = BODIES[name]
        p = Problem(_cost(d, n0, n1, n0 + n1), reg, norm, prec, body)
        p.name = f"{name}_reg{reg}"
    floor = _floor(p)
    c, big = 10, 4000
    out = p.solve(big, stop_thr=1e-14, stall_tol=0.1)
    it = out.st[1]
    assert out.st[0] == 0 and it < big and (it - 1) % c == 0, out.st
    assert out.err * math.sqrt(p.n1) < 1e-5
    prev = p.solve(it - c, stop_thr=1e-14)
    assert prev.st[1] == it - c and out.err > 0.9 * prev.err, (out.err, prev.err)
    v_next = -math.log(p.n1) - torch.logsumexp(p.Mr + out.lu[:, None], dim=0)
    col_err = torch.linalg.vector_norm(torch.expm1(out.lv - v_next) / p.n1).item()
    assert abs(col_err - out.err) <= floor, (col_err, out.err, floor)
    full = p.solve(it + 5 * c, stop_thr=1e-14, stall_tol=0.0)
    assert full.st[1] == it + 5 * c and full.st[0] == FLAG_NOT_CONVERGED


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BODIES))
def test_nan_cost(name):
    """A NaN cost: both flags, err NaN, all max_iters run although stop_thr and stall_tol are set, and the
    potentials NaN where the restatement's are"""
    p = _body(name, nan=True)
    for iters in (1, 25):
        out = p.solve(iters, stop_thr=1e-3, stall_tol=0.5)
        ref = p.ref(iters, stop_thr=1e-3, stall_tol=0.5)
        assert out.st[0] == FLAG_NONFINITE | FLAG_NOT_CONVERGED and out.st[1] == iters and math.isnan(out.err)
        assert ref.flags == out.st[0] and ref.iters == iters
        assert torch.equal(out.lu.isnan(), ref.u.isnan()) and torch.equal(out.lv.isnan(), ref.v.isnan()), iters
        assert ref.v.isnan().any()


# -------------------------------------------------- B. shapes and instantiations of the generic and v2 kernels
def _shape_case(n0, n1, precision, reg, normalize, body, d=16, ldm=None, offset=0, null_cmax=False, launches=1,
                M=None):
    """the status word, launch count, potentials and err against the restatement after 1, 11 and 12 iterations (the
    last checked every 10: a check, then a last iteration that is none)"""
    if M is None:
        M = _points(n0, n1, d, n0 + n1)
    p = Problem(M, reg, normalize, precision, body, ldm=ldm, offset=offset, null_cmax=null_cmax)
    p.name = "shapes"
    for iters in (1, 11, 12):
        out = p.solve(iters)
        ref = p.ref(iters)
        assert out.st[1] == iters and out.st[0] == FLAG_NOT_CONVERGED and out.launches == launches, (iters, out.st)
        e = _pot_err(out, ref, body[0])
        assert e < GATE[body[0]], (iters, e)
        if body[0] == 1:
            assert abs(out.err - ref.err) <= _err_tol(p, ref.err, _f64_floor(p))
        else:  # rounding noise of err: DV / sqrt(n1) for a noise of DV in each column's change of v
            assert abs(out.err - ref.err) <= DV[body[0]] / math.sqrt(n1), (out.err, ref.err)


DV = {0: 8e-6, 2: 1e-6}  # fp32: a few ulp of |v| ~ 20; mixed: fp32 exponentials


# the generic kernel's four modes; the f64 regime of normalised costs starts at reg < 1/64
GENERIC_MODES = {"fp32": ("fp32-generic", 0.05, (0, 0)), "fp64": ("fp64", 0.05, (1, 0)),
                 "mixed": ("fp64-mixed-unscreened", 0.012, (2, 0)), "seeded": ("fp64-mixed", 0.012, (2, 1))}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(GENERIC_MODES))
@pytest.mark.parametrize("n1,pitch,offset", [
    (2048, 0, 0), (4096, 0, 0), (6000, 0, 0),           # VEC, KG = 1, 2, 4
    (2047, 0, 0), (2049, 0, 0), (4095, 0, 0), (6001, 0, 0), (9001, 0, 0),  # n1 % 4 != 0
    (2048, 1, 0), (4096, 1, 0), (6000, 1, 0),           # row pitch n1 + 1
    (2048, 0, 1), (6000, 0, 1),                         # M at a storage offset of one float
    (12288, 0, 0), (14000, 0, 0)])                      # column panels; v not staged (n1p > 13653)
def test_generic_kernel_instantiations(mode, n1, pitch, offset):
    prec, reg, body = GENERIC_MODES[mode]
    if mode == "seeded" and n1 > 8192:
        body = (2, 0)  # more than one column panel: the generic mixed body, screened while v is staged
    _shape_case(200, n1, prec, reg, 1, body, ldm=n1 + pitch if pitch else None, offset=offset)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["v2", "fp32", "fp64", "seeded"])
@pytest.mark.parametrize("rows", ["1", "2", "grid-1", "grid", "grid+1", "2grid-1", "2grid+1", "3grid-1"])
def test_row_slabs_around_the_grid(kernel, rows):
    """n0 from 1 to three grids: one row per CTA, CTAs without rows, slabs that differ by one row"""
    G = _grid()
    n0 = {"1": 1, "2": 2, "grid-1": G - 1, "grid": G, "grid+1": G + 1, "2grid-1": 2 * G - 1, "2grid+1": 2 * G + 1,
          "3grid-1": 3 * G - 1}[rows]
    if kernel == "v2":
        _shape_case(n0, 256, "fp32", 0.05, 1, (0, 3))
    else:
        prec, reg, body = GENERIC_MODES[kernel]
        _shape_case(n0, 256, prec, reg, 1, body)


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", ["auto", "fp32", "fp64", "seeded"])
@pytest.mark.parametrize("n1", [1, 3, 4, 5, 17])
def test_few_columns_many_rows(kernel, n1):
    """n1 far below the grid: most CTAs own no column in the combine"""
    if kernel == "auto":  # the v2 kernel on aligned n1, with the generic kernel launched behind it; else generic fp32
        _shape_case(3000, n1, "auto", 0.05, 1, (0, 3) if n1 % 4 == 0 else (0, 0), launches=2 if n1 % 4 == 0 else 1)
    else:
        prec, reg, body = GENERIC_MODES[kernel]
        _shape_case(3000, n1, prec, reg, 1, body)


@pytest.mark.gpu
@pytest.mark.parametrize("path,reg,variant", [("factored", 0.05, 3), ("log_domain", 0.03, 2)])
@pytest.mark.parametrize("n1", [2048, 2052, 4096, 4100, 8188, 8192])
def test_v2_kernel_instantiations(path, reg, variant, n1):
    """<512, 1, 8> up to n1 = 2048, <512, 2, 4> up to 4096, <512, 4, 2> up to 8192; on both sweeps"""
    _shape_case(300, n1, "fp32", reg, 1, (0, variant))


@pytest.mark.gpu
@pytest.mark.parametrize("precision,body", [("fp32", (0, 2)), ("fp64", (1, 0))])
def test_null_cost_max(precision, body):
    """normalize = 0 without cost_max: the v2 kernel cannot form its factored span and runs the log-domain sweep"""
    g = torch.Generator().manual_seed(4)
    M = (torch.rand(500, 512, generator=g) * 0.5 + 0.5).to(DEV)
    _shape_case(500, 512, precision, 0.05, 0, body, null_cmax=True, M=M)


# ------------------------------------------------------------------- C. dispatch table and regime boundary
# (precision, normalize, regime, n1, row pitch, float offset, cost_max) -> (status[2], status[3], launches).
# cfm_sinkhorn_log_f32: precisions 0 and -1 try sinkhorn_v2_kernel first, which covers 16-byte aligned rows of
# n1 % 4 == 0 <= 8192; auto mode then launches the generic kernel behind it for the float64 regime.  v2 variant:
# 4 when M streams (fp32 larger than 3/4 of the L2) and the span allows factoring, 3 factored, 2 log-domain.  The
# generic kernel: mixed arithmetic (auto, 3, 4) with screening (not 4) and one column panel runs the seeded solver.
DISPATCH = [
    (-1, 1, "fp32", 256, 0, 0, True, (0, 3, 2)),
    (-1, 1, "f64", 256, 0, 0, True, (2, 1, 2)),
    (-1, 0, "span", 256, 0, 0, True, (0, 2, 2)),
    (-1, 1, "fp32", 257, 0, 0, True, (0, 0, 1)),
    (-1, 1, "f64", 257, 0, 0, True, (2, 1, 1)),
    (-1, 1, "fp32", 256, 1, 0, True, (0, 0, 1)),
    (-1, 1, "fp32", 256, 0, 1, True, (0, 0, 1)),
    (-1, 1, "fp32", 9000, 0, 0, True, (0, 0, 1)),
    (-1, 1, "f64", 9000, 0, 0, True, (2, 0, 1)),
    (-1, 1, "f64", 14000, 0, 0, True, (2, 0, 1)),
    (-1, 1, "fp32", 4096, 0, 0, True, (0, 4, 2)),
    (0, 1, "fp32", 256, 0, 0, True, (0, 3, 1)),
    (0, 1, "f64", 256, 0, 0, True, (0, 2, 1)),
    (0, 1, "fp32", 257, 0, 0, True, (0, 0, 1)),
    (0, 1, "fp32", 4096, 0, 0, True, (0, 4, 1)),
    (0, 0, "fp32", 256, 0, 0, False, (0, 2, 1)),
    (0, 0, "fp32", 257, 0, 0, False, (0, 0, 1)),
    (1, 1, "fp32", 256, 0, 0, True, (1, 0, 1)),
    (1, 0, "f64", 256, 0, 0, False, (1, 0, 1)),
    (2, 1, "fp32", 256, 0, 0, True, (0, 0, 1)),
    (2, 1, "f64", 256, 0, 0, True, (0, 0, 1)),
    (3, 1, "f64", 256, 0, 0, True, (2, 1, 1)),
    (3, 1, "f64", 9000, 0, 0, True, (2, 0, 1)),
    (3, 1, "f64", 14000, 0, 0, True, (2, 0, 1)),
    (4, 1, "f64", 256, 0, 0, True, (2, 0, 1)),
]


@pytest.mark.gpu
def test_dispatch_table():
    inv = {v: k for k, v in PREC.items()}
    for prec, norm, regime, n1, pitch, offset, has_cmax, want in DISPATCH:
        n0 = _v2_3byte_n0() if n1 == 4096 else 64
        M = _points(n0, n1, 16, n1)
        if not norm:
            M = M / M.max()  # max 1 (un-normalised regimes set by reg below)
        # normalised: reg 0.05 factors (span 29 log2 units), 0.01 is past |M/reg| = 64; un-normalised "span": M/reg
        # = 50, inside the fp32 regime but past the factored span of 40
        reg = {"fp32": 0.05, "f64": 0.01, "span": 0.02}[regime]
        Mb = _place(M, n1 + pitch if pitch else None, offset)
        cmax = M.max().reshape(1).float() if has_cmax else None
        out = _solve(Mb, n1, reg, cmax, norm, inv[prec], 1)
        assert (out.st[2], out.st[3], out.launches) == want, (prec, norm, regime, n1, pitch, offset, has_cmax)


@pytest.mark.gpu
@pytest.mark.parametrize("n1", [256, 257])
@pytest.mark.parametrize("normalize", [0, 1])
def test_regime_boundary_at_64(normalize, n1):
    """|cmax / reg| = 64 exactly is fp32; the next float above it is float64 potentials (mixed), on the v2-covered
    shape (n1 = 256) and the generic-only one (n1 = 257).  Powers of two make both quotients exact."""
    g = torch.Generator().manual_seed(n1)
    M = (torch.randint(0, 33, (200, n1), generator=g).float()).to(DEV)  # entries 0 .. 32
    M[0, 0] = 32.0
    for above in (False, True):
        if normalize:
            reg = np.nextafter(np.float32(2.0 ** -6), np.float32(0)) if above else np.float32(2.0 ** -6)
            Mc = M
        else:
            reg = np.float32(0.5)
            Mc = M.clone()
            if above:
                Mc[0, 0] = float(np.nextafter(np.float32(32.0), np.float32(64)))
        cmax = Mc.max().reshape(1).float()
        q = np.float32(1.0 if normalize else float(cmax)) / np.float32(reg)
        assert q > 64 if above else q == 64
        out = _solve(_place(Mc), n1, float(reg), cmax, normalize, "auto", 3)
        want = (2, 1) if above else (0, 2 if n1 == 256 else 0)
        assert (out.st[2], out.st[3]) == want, (above, out.st)
        assert out.launches == (2 if n1 == 256 else 1)


# ---------------------------------------------------------------------------- D. stale workspace on every body
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BODIES))
def test_stale_workspace(name):
    """0x00, 0xFF and the leftovers of a larger solve (more CTAs, a non-zero error ring, other per-CTA minima) in
    the workspace give the same bits; err only to 1e-14 (an atomicAdd in CTA arrival order)"""
    d, n0, n1, reg, norm, prec, body = BODIES[name]
    n0 = n0() if callable(n0) else n0
    small = name != "v2_3byte"
    if small:
        n0 = _sms() // 2 + 3  # a grid of fewer CTAs than the other solve's
    p = Problem(_cost(d, n0, n1, 1), reg, norm, prec, body)
    n0o = 2 * _sms() + 5 if small else n0
    other = Problem(_cost(d, n0o, n1, 2), reg, norm, prec, body)
    L = _ffi.lib()
    ws = torch.empty(max(L.cfm_sinkhorn_workspace_bytes(n0, n1), L.cfm_sinkhorn_workspace_bytes(n0o, n1)),
                     dtype=torch.uint8, device=DEV)
    for iters in (1, 2, 3, 11):
        got = []
        for history in ("zeros", "ones", "other"):
            if history == "zeros":
                ws.fill_(0x00)
            elif history == "ones":
                ws.fill_(0xFF)
            else:
                o = other.solve(23, ws=ws)
                assert o.st[1] == 23
            got.append(p.solve(iters, ws=ws))
        for g in got[1:]:
            assert torch.equal(g.lu, got[0].lu) and torch.equal(g.lv, got[0].lv) and g.st == got[0].st, iters
            assert abs(g.err - got[0].err) <= 1e-14 * abs(got[0].err), iters


# ---------------------------------------------------------------------------- E. the compiled instantiations
def test_compiled_sinkhorn_instantiations_are_the_tested_ones(lib_built):
    """Reads the kernels out of the library's cubin; no device needed.  A new sinkhorn_kernel or sinkhorn_v2_kernel
    instantiation needs cases in this file first."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout

    def args(kernel, pattern):
        syms = set(re.findall(r"\w*%s\w*" % kernel, out))
        parsed = {s: re.search(kernel + pattern, s) for s in syms}
        assert syms and all(parsed.values()), syms
        return {p.groups() for p in parsed.values()}

    # VEC x KG: test_generic_kernel_instantiations
    assert args("sinkhorn_kernel", r"ILb(\d)ELi(\d)EEEv") == {(v, k) for v in "01" for k in "124"}
    # <512, KG, R>: test_v2_kernel_instantiations
    assert args("sinkhorn_v2_kernel", r"ILi(\d+)ELi(\d+)ELi(\d+)EEEv") == {("512", "1", "8"), ("512", "2", "4"),
                                                                            ("512", "4", "2")}
    # _grid: more than 64 registers per thread leave room for one 512-thread CTA of sinkhorn_kernel per SM (64K
    # registers), so the launcher's SMs x min(occupancy, 2) is the SM count
    res = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", lib_built], capture_output=True, text=True,
                         check=True).stdout
    regs = {m.group(1): int(m.group(2)) for m in re.finditer(r"Function (\w*sinkhorn_kernel\w*):\s+REG:(\d+)", res)}
    assert len(regs) == 6 and all(64 < r <= 128 for r in regs.values()), regs
