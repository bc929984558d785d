"""The fused flow-pair kernel (csrc/flow.cu: cfm_flow_pairs_f32, flow_pairs_kernel<VEC>) and the row gather
(csrc/gather.cu: cfm_gather_rows, gather_rows_kernel<W>) on every path they take.

CPU: the kernel instantiations in the built library; every argument refusal of both entry points, which return before
any CUDA call; the torch layout rules behind the matchers' routing (randn_like and x[i] keep a transposed or
channels_last layout, so only contiguous batches may take the fused path, whose eps is contiguous).
GPU:
  (a) cfm_flow_pairs_f32 through the C ABI: every kind on both instantiations, with and without pair indices, with
      per-row and scalar sigma, at 1 thread, exactly one grid pass, one more and at least three passes.  Against the
      same closed form written as one fp32 torch op per rounded kernel op in the kernel's order (bit for bit, NaN
      where it is NaN), and against the float64 matcher formulas of oracle.coupling within a few ulps of the terms;
  (b) the five matcher classes against their unfused subclasses (the reference's torch-op chain) at t = 0 and 1,
      integer sigma = 0, caller-supplied and float64 t, odd rows, offset, transposed and channels_last inputs, and
      guided labels of four dtypes and three shapes;
  (c) cfm_gather_rows at each word width it picks, reached by row bytes and by pointer offset, at element sizes 1, 2,
      4 and 8, at every grid-pass class, and on a byte-path source past 2^31 bytes, against index_select bit for bit;
  (d) OTPlanSampler._gather's torch fallback, and sample_plan on host inputs.

Which kernel ran: every GPU case records the arguments of each entry-point call (a proxy of the library stands in for
it) and derives the instantiation from them by the dispatch rule (row bytes and pointer alignment).  The dispatch tests
read the kernel names and grids of one launch of every dispatch class from torch.profiler traces, which pins that rule
to what the library launches.  Those traces are taken in a child process: with torch 2.11, once a process has taken a
trace, kernels go missing from its later traces, and the profiler-based tests of other files would lose theirs.

Sizes follow from the device's SM count (the kernels cap their grid at 16 CTAs of 256 threads per SM), so the pass
classes keep their meaning on a part with a different SM count."""
import ctypes
import itertools
import json
import math
import os
import pathlib
import re
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from oracle import coupling as oc

import cfm_b200
from cfm_b200 import _ffi
from cfm_b200.optimal_transport import OTPlanSampler

DEV = "cuda:0"
TESTS = os.path.dirname(os.path.abspath(__file__))
gpu = pytest.mark.gpu
BLOCK = 256
CTAS_PER_SM = 16

_KERNEL_RE = re.compile(r"cfm::(flow_pairs|gather_rows)_kernel<([^>]+)>")
# gather_rows_kernel<W> by word bytes: (W as the profiler names it, W as its mangled symbol spells it)
GATHER_WORDS = {1: ("unsigned char", "h"), 2: ("unsigned short", "t"), 4: ("unsigned int", "j"),
                8: ("uint2", "5uint2"), 16: ("uint4", "5uint4")}
FLOW_VEC = {"true": "Lb1E", "false": "Lb0E"}
KINDS = {"icfm": _ffi.FLOW_ICFM, "target": _ffi.FLOW_TARGET, "sb": _ffi.FLOW_SB, "vp": _ffi.FLOW_VP}
# matcher class and sigma whose row coefficients each kind is driven with; Target at sigma = 0 divides 0 by 0 at t = 1
KIND_MATCHER = {"icfm": ("ConditionalFlowMatcher", 0.5, "i_cfm"),
                "target": ("TargetConditionalFlowMatcher", 0, "t_cfm"),
                "sb": ("SchrodingerBridgeConditionalFlowMatcher", 0.7, "sb_cfm"),
                "vp": ("VariancePreservingConditionalFlowMatcher", 0.3, "vp_cfm")}
SENTINEL = -7.25e29  # outputs are pre-filled with it: an element the kernel skips shows up
DECOY_SIGMA = 3.0    # scalar sigma passed next to per-row sigma, which the kernel must ignore
_INT_OF = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}
_ELEM_DTYPE = {1: torch.uint8, 2: torch.float16, 4: torch.float32, 8: torch.float64}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pass_threads():
    """Threads in one pass of the capped grid."""
    return CTAS_PER_SM * _sms() * BLOCK


def _grid(work):
    return min((work + BLOCK - 1) // BLOCK, CTAS_PER_SM * _sms())


def _profiled(fn, tmp_path, launches):
    """(fn(), [(kernel, template argument, grid, block)] of every flow_pairs_kernel and gather_rows_kernel it ran, in
    launch order), read from a torch.profiler trace.

    A trace now and then lacks a kernel that ran, most likely a GPU timestamp placed outside the host-clock capture
    window (see the module docstring).  A trace with fewer than ``launches`` records of these kernels is taken again,
    running fn again with a wider idle margin on both sides, up to four times in all.  So fn must be repeatable."""
    from torch.profiler import ProfilerActivity, profile
    for margin in (0.0, 0.01, 0.1, 1.0):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            time.sleep(margin)
            out = fn()
            torch.cuda.synchronize()
            time.sleep(margin)
        path = tmp_path / "trace.json"
        prof.export_chrome_trace(str(path))
        ran = []
        for e in json.loads(path.read_text())["traceEvents"]:
            m = _KERNEL_RE.search(e.get("name", "")) if e.get("cat") == "kernel" else None
            if m:
                ran.append((e["ts"], m.group(1), m.group(2), e["args"]["grid"][0], e["args"]["block"][0]))
        path.unlink()
        if len(ran) >= launches:
            break
    return out, [r[1:] for r in sorted(ran)]


class _Recorder:
    """Stands in for the loaded library: records the arguments of every cfm_flow_pairs_f32 and cfm_gather_rows call
    and forwards all calls to the library."""

    def __init__(self, lib):
        self._lib, self.flow, self.gather = lib, [], []

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def cfm_flow_pairs_f32(self, *args):
        self.flow.append(args)
        return self._lib.cfm_flow_pairs_f32(*args)

    def cfm_gather_rows(self, *args):
        self.gather.append(args)
        return self._lib.cfm_gather_rows(*args)


@pytest.fixture
def calls(monkeypatch):
    rec = _Recorder(_ffi.lib())
    monkeypatch.setattr(_ffi, "_lib", rec)
    return rec


def _address(p):
    return p.value or 0 if isinstance(p, ctypes.c_void_p) else p or 0


def _flow_instantiation(args):
    """flow_pairs_kernel<VEC> a cfm_flow_pairs_f32 call launches: VEC when the row is a multiple of 4 floats and x0,
    x1, eps, xt and ut are 16-byte aligned."""
    row, ptrs = args[15], [_address(args[k]) for k in (1, 2, 5, 12, 13)]
    return "true" if row % 4 == 0 and not any(p % 16 for p in ptrs) else "false"


def _gather_width(args):
    """Word bytes of the gather_rows_kernel a cfm_gather_rows call launches: the largest of 16, 8, 4, 2, 1 dividing
    the row bytes and both addresses."""
    a = _address(args[0]) | _address(args[5])
    return math.gcd(math.gcd(args[1] * args[2], 16), a & -a if a else 16)


def _shortest_launch_us(call, reps=3):
    """Shortest time of ``reps`` launches of call(), from CUDA events around each."""
    best = math.inf
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b) * 1e3)
    return best


def _assert_each_thread_visits_its_work_once(us, moved):
    """A grid-stride loop with a stride shorter than the grid revisits work and writes the same values again, so only
    its time shows it: at three passes it takes about gridDim / 2 times as long.  Both kernels run near HBM speed;
    the bound, ``moved`` bytes at 50 GB/s (1/60 of the H100 SXM's 3.35 TB/s) and never under 200 us, leaves room for
    a shared GPU.  ``us`` is the shortest of several launches; returns it as a fraction of the bound."""
    bound = max(200.0, moved / 50e9 * 1e6)
    assert us <= bound, (us, moved)
    return us / bound


def _launches(fn):
    L = _ffi.lib()
    before = L.cfm_launch_count()
    out = fn()
    return out, L.cfm_launch_count() - before


def _bits(x):
    return x.view(_INT_OF[x.element_size()]) if x.dtype != torch.bool else x.view(torch.uint8)


def _assert_same(got, want, what):
    """Same dtype, shape and device, equal bits, and NaN exactly where ``want`` is NaN (any payload)."""
    assert (got.dtype, got.shape, got.device) == (want.dtype, want.shape, want.device), what
    nan = torch.isnan(want) if want.is_floating_point() else torch.zeros_like(want, dtype=torch.bool)
    bad = (_bits(got) != _bits(want)) & ~nan
    bad |= nan & ~torch.isnan(got)
    if bad.any():
        k = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ; first at {k}: "
                             f"{got[k].item()!r} != {want[k].item()!r}")


def _aligned(numel, offset, dtype=torch.float32):
    """Contiguous 1-D tensor of ``numel`` elements starting ``offset`` elements past a fresh (512-byte aligned)
    allocation."""
    return torch.empty(numel + offset, dtype=dtype, device=DEV)[offset:]


def _indices(n, hi, seed):
    """n row indices below hi: out of order, repeated, and holding hi - 1."""
    g = torch.Generator().manual_seed(seed)
    idx = torch.randint(0, hi, (n,), generator=g)
    idx[0] = hi - 1
    if n > 2:
        idx[n // 2] = idx[1]
    return idx.to(DEV)


# ================================================================================================ CPU
def test_compiled_flow_and_gather_instantiations_are_the_tested_ones(lib_built):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    found = set(re.findall(r"(flow_pairs|gather_rows)_kernelI(.+?)EEv", out))
    assert found == ({("flow_pairs", m) for m in FLOW_VEC.values()}
                     | {("gather_rows", m) for _, m in GATHER_WORDS.values()})


def test_randn_like_and_row_indexing_keep_transposed_and_channels_last_layouts():
    """The reference draws eps = randn_like(x0) (randn_like(x0[i]) when coupled); the fused path draws a contiguous
    eps, so it may take only batches on which the two are the same tensor."""
    xt = torch.randn(6, 5).t()
    assert torch.randn_like(xt).stride() == xt.stride() == (1, 5)
    cl = torch.randn(4, 3, 8, 8).to(memory_format=torch.channels_last)
    assert torch.randn_like(cl).stride() == cl.stride() and not cl.is_contiguous()
    rows = cl[torch.tensor([2, 0, 0, 3])]
    assert rows.is_contiguous(memory_format=torch.channels_last) and not rows.is_contiguous()
    x = torch.randn(6, 5)
    assert torch.randn_like(x).is_contiguous() and x[torch.tensor([5, 0, 0])].is_contiguous()


def test_flow_pairs_refusals_return_before_any_launch(lib_built):
    L = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)

    def call(kind=_ffi.FLOW_ICFM, rb=p, rc=p, n=4, row=8, x0=p):
        return L.cfm_flow_pairs_f32(kind, x0, p, None, None, p, p, rb, None, rc, 0.5, 1.0, p, p, n, row, None)

    refusals = [(dict(kind=-1), "unknown kind"), (dict(kind=4), "unknown kind"),
                (dict(n=-1), "negative size"), (dict(row=-1), "negative size"), (dict(x0=None), "null pointer")]
    refusals += [(dict(kind=_ffi.FLOW_ICFM, rb=None), "row_b required"),
                 (dict(kind=_ffi.FLOW_SB, rb=None), "row_b required"),
                 (dict(kind=_ffi.FLOW_VP, rb=None), "row_b required"),
                 (dict(kind=_ffi.FLOW_TARGET, rc=None), "row_c required"),
                 (dict(kind=_ffi.FLOW_SB, rc=None), "row_c required")]
    for kw, msg in refusals:
        before = L.cfm_launch_count()
        assert call(**kw) != 0, kw
        assert msg in L.cfm_last_error().decode() and L.cfm_launch_count() == before, kw
    # Target needs no row_b; nothing to do is success with no launch, whatever the pointers
    before = L.cfm_launch_count()
    assert call(kind=_ffi.FLOW_TARGET, rb=None, n=0) == 0 and call(row=0, x0=None, rb=None, rc=None) == 0
    assert L.cfm_launch_count() == before


def test_gather_rows_refusals_return_before_any_launch(lib_built):
    L = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf)
    for args, msg in [((p, 4, 4, p, -1, p), "negative size"), ((p, -1, 4, p, 3, p), "negative size"),
                      ((None, 4, 4, p, 3, p), "null pointer"), ((p, 4, 4, None, 3, p), "null pointer"),
                      ((p, 4, 4, p, 3, None), "null pointer"), ((p, 4, 3, p, 3, p), "elem_bytes"),
                      ((p, 4, 16, p, 3, p), "elem_bytes"), ((p, 4, 0, p, 3, p), "elem_bytes")]:
        before = L.cfm_launch_count()
        assert L.cfm_gather_rows(*args, None) != 0, args
        assert msg in L.cfm_last_error().decode() and L.cfm_launch_count() == before, args
    before = L.cfm_launch_count()
    assert L.cfm_gather_rows(None, 4, 4, None, 0, None, None) == 0
    assert L.cfm_gather_rows(None, 0, 4, None, 3, None, None) == 0
    assert L.cfm_launch_count() == before


def test_dispatch_rules_on_recorded_arguments():
    """The rules the GPU cases read the instantiation from, on argument tuples as the entry points receive them."""
    p = ctypes.c_void_p

    def flow(row, x0, x1, eps, xt, ut):
        return (0, p(x0), p(x1), None, None, p(eps), None, None, None, None, 0.0, 0.0, p(xt), p(ut), 1, row, None)

    assert _flow_instantiation(flow(8, 512, 1024, 2048, 4096, 8192)) == "true"
    assert _flow_instantiation(flow(6, 512, 1024, 2048, 4096, 8192)) == "false"
    for k in range(5):
        addrs = [512] * 5
        addrs[k] += 4
        assert _flow_instantiation(flow(8, *addrs)) == "false"
    widths = [_gather_width((p(x), row, elem, None, 1, p(out), None))
              for x, row, elem, out in [(512, 12, 4, 1024), (512, 3, 1, 1024), (520, 4, 4, 1024), (512, 8, 2, 1030)]]
    assert widths == [16, 1, 8, 2]


# ================================================================================ GPU (a): cfm_flow_pairs_f32
OPERANDS = ("x0", "x1", "eps", "xt", "ut")
MODES = [("identity", "scalar"), ("identity", "rows"), ("pairs", "scalar"), ("pairs", "rows")]


def _flow_shape(route, size):
    """(n, row) of a direct call: 'vec' runs flow_pairs_kernel<true>; 'odd_row' (row % 4 != 0) and 'offset:<operand>'
    (that operand one float past 16-byte alignment) run <false>.  Sizes are in threads of work: 1 (4 for an offset
    row), exactly one pass of the capped grid, one more, and at least three passes on a 3x32x32 or 7-float row."""
    sms, cap = _sms(), _pass_threads()
    table = {"vec": {"one": (1, 4), "pass": (cap // 8, 32), "pass+1": (cap + 1, 4),
                     "passes3": (CTAS_PER_SM * sms + 3, 3 * 32 * 32)},
             "odd_row": {"one": (1, 1), "pass": (cap // 2, 2), "pass+1": (cap + 1, 1),
                         "passes3": (3 * cap // 7 + 2, 7)},
             "offset": {"one": (1, 4), "pass": (cap // 4, 4), "passes3": (4 * sms + 1, 3 * 32 * 32)}}
    return table[route.split(":")[0]][size]


def _flow_cases():
    cases = []
    for kind in KINDS:
        for size, mode in itertools.product(("one", "pass", "pass+1", "passes3"), MODES):
            cases += [(kind, "vec", size, mode), (kind, "odd_row", size, mode)]
        for k, (operand, size) in enumerate(itertools.product(OPERANDS, ("one", "pass", "passes3"))):
            cases.append((kind, "offset:" + operand, size, MODES[k % len(MODES)]))
    return [pytest.param(*c, id="-".join(c[:3] + c[3])) for c in cases]


class _FlowCase:
    """Inputs, outputs (filled with SENTINEL) and the C call of one direct cfm_flow_pairs_f32 case."""

    def __init__(self, kind, route, size, mode):
        n, row = self.n, self.row = _flow_shape(route, size)
        self.kind, self.vec = kind, route == "vec"
        self.work = n * (row // 4 if self.vec else row)
        cap = _pass_threads()
        assert {"one": self.work <= 4, "pass": self.work == cap, "pass+1": self.work == cap + 1,
                "passes3": self.work >= 3 * cap}[size]
        off = {op: int(route == "offset:" + op) for op in OPERANDS}
        pairs, sig_mode = mode
        seed = 1000 * list(KINDS).index(kind) + n + row
        gd = torch.Generator(device=DEV).manual_seed(seed)

        def operand(name, scale=1.0, shift=0.0):
            x = _aligned(n * row, off[name]).view(n, row)
            x.copy_(torch.randn(n, row, generator=gd, device=DEV) * scale + shift)
            return x

        self.x0, self.x1, self.eps = operand("x0"), operand("x1", 1.7, 0.3), operand("eps")
        self.x0.view(-1)[::97] = -0.0
        self.x1.view(-1)[5::89] = 0.0
        self.i = _indices(n, n, seed) if pairs == "pairs" else None
        self.j = _indices(n, n, seed + 1) if pairs == "pairs" else None
        t = torch.rand(n, generator=torch.Generator().manual_seed(seed))
        t[0] = 1.0
        if n > 1:
            t[1], t[-1] = 0.0, 1.0
        self.t = t.to(DEV)
        cls, self.sigma, self.name = KIND_MATCHER[kind]
        ra, rb, rs, rc, s, k = getattr(cfm_b200, cls)(self.sigma)._row_coefficients(self.t)
        vec32 = lambda v: None if v is None else v.to(torch.float32).contiguous()  # noqa: E731
        self.ra, self.rb, rs, self.rc, self.k = vec32(ra), vec32(rb), vec32(rs), vec32(rc), k
        self.matcher_sigma = True  # the coefficients are the matcher's own: the float64 gate applies
        if sig_mode == "rows":
            rs, s = (torch.full((n,), s, device=DEV) if rs is None else rs), DECOY_SIGMA
        elif rs is not None:  # Target and SB with a scalar sigma_t: the kernel's form, but no matcher's
            rs, s, self.matcher_sigma = None, 0.37, False
        self.rs, self.s = rs, s
        self.xt = _aligned(n * row, off["xt"]).view(n, row).fill_(SENTINEL)
        self.ut = _aligned(n * row, off["ut"]).view(n, row).fill_(SENTINEL)

    def __call__(self):
        return _ffi.lib().cfm_flow_pairs_f32(
            KINDS[self.kind], *map(_ffi.ptr, (self.x0, self.x1, self.i, self.j, self.eps, self.ra, self.rb, self.rs,
                                              self.rc)),
            self.s, self.k, _ffi.ptr(self.xt), _ffi.ptr(self.ut), self.n, self.row, _ffi.stream_ptr(DEV))


def _f32(v):
    return torch.tensor(v, dtype=torch.float32, device=DEV)


def _flow_oracle(kind, g0, g1, e, ra, rb, rs, rc, s, k):
    """csrc/flow.cu's closed form as fp32 torch ops on the device: one op for each __f*_rn of the kernel, in its
    association order.  g0 = x0[i] and g1 = x1[j] are already gathered."""
    col = lambda v: v[:, None]  # noqa: E731
    sg = col(rs) if rs is not None else _f32(s)
    if kind == _ffi.FLOW_ICFM:
        mu = col(ra) * g1 + col(rb) * g0
        return mu + sg * e, g1 - g0
    if kind == _ffi.FLOW_TARGET:
        xt = col(ra) * g1 + sg * e
        return xt, (g1 - _f32(k) * xt) / col(rc)
    if kind == _ffi.FLOW_SB:
        mu = col(ra) * g1 + col(rb) * g0
        xt = mu + sg * e
        return xt, col(rc) * (xt - mu) + g1 - g0
    c, sn = col(ra), col(rb)
    return c * g0 + sn * g1 + sg * e, _f32(k) * (c * g1 - sn * g0)


def _float64_gate(name, g0, g1, e, t, sigma, xt, ut, record_property):
    """The kernel's xt and ut against oracle.coupling.matcher_xt_ut in float64, within 16 ulps (2^-24) of the sum of
    the magnitudes of the terms each output is built from, including the fp32 rounding of the row coefficients.
    NaN (Target's 0/0 at sigma = 0, t = 1) must be NaN on both sides."""
    g0, g1, e, t = g0.double(), g1.double(), e.double(), t.double()
    xt64, ut64 = oc.matcher_xt_ut(name, g0, g1, t, e, sigma)
    tp = t[:, None]
    if name == "i_cfm":
        txt, tut = (tp * g1).abs() + ((1 - tp) * g0).abs() + (sigma * e).abs(), g1.abs() + g0.abs()
    elif name == "t_cfm":
        den = (1 - (1 - sigma) * tp).abs()
        txt = (tp * g1).abs() + e.abs()
        tut = (g1.abs() + ((1 - sigma) * xt64).abs() + abs(1 - sigma) * txt + ut64.abs() * (1 + tp)) / den
    elif name == "sb_cfm":
        coef = ((1 - 2 * tp) / (2 * tp * (1 - tp) + 1e-8)).abs()
        txt = (tp * g1).abs() + ((1 - tp) * g0).abs() + (sigma * torch.sqrt(tp * (1 - tp)) * e).abs()
        tut = 3 * coef * txt + g1.abs() + g0.abs()
    else:
        txt, tut = g0.abs() + g1.abs() + (sigma * e).abs(), math.pi * (g0.abs() + g1.abs())
    worst = 0.0
    for got, want, terms, what in ((xt, xt64, txt, "xt"), (ut, ut64, tut, "ut")):
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan), what
        tol = 16 * 2.0**-24 * terms[~nan]
        err = (got.double()[~nan] - want[~nan]).abs()
        assert bool((err <= tol).all()), (what, float((err - tol).max()))
        if err.numel():
            worst = max(worst, float((err / tol.clamp_min(1e-300)).max()))
    record_property("err_over_gate", worst)


@gpu
@pytest.mark.parametrize("kind,route,size,mode", _flow_cases())
def test_flow_pairs_against_the_closed_form(kind, route, size, mode, calls, record_property):
    c = _FlowCase(kind, route, size, mode)
    rc, launches = _launches(c)
    assert rc == 0 and launches == 1, _ffi.last_error()
    assert [_flow_instantiation(a) for a in calls.flow] == ["true" if c.vec else "false"]
    g0 = c.x0[c.i] if c.i is not None else c.x0
    g1 = c.x1[c.j] if c.j is not None else c.x1
    want_xt, want_ut = _flow_oracle(KINDS[kind], g0, g1, c.eps, c.ra, c.rb, c.rs, c.rc, c.s, c.k)
    _assert_same(c.xt, want_xt, "xt")
    _assert_same(c.ut, want_ut, "ut")
    if c.matcher_sigma:
        _float64_gate(c.name, g0, g1, c.eps, c.t, c.sigma, c.xt, c.ut, record_property)
    if size == "passes3":
        record_property("time_over_bound", _assert_each_thread_visits_its_work_once(_shortest_launch_us(c),
                                                                                    5 * 4 * c.n * c.row))



# ============================================================================ GPU (b): the five matcher classes
MATCHERS = {"icfm": "ConditionalFlowMatcher", "otcfm": "ExactOptimalTransportConditionalFlowMatcher",
            "target": "TargetConditionalFlowMatcher", "sb": "SchrodingerBridgeConditionalFlowMatcher",
            "vp": "VariancePreservingConditionalFlowMatcher"}
SIGMA = {"icfm": 0.5, "otcfm": 0.25, "target": 0.5, "sb": 0.7, "vp": 0.3}


def _stock_and_unfused(name, sigma, x0, x1, fused, calls, t=None, labels=None, seed=11):
    """Run the stock class and its unfused subclass (a subclass is not stock: it takes the reference's torch-op chain)
    from the same seeds; assert every output equal, and that the stock class ran flow_pairs_kernel<fused> once (no
    flow kernel when ``fused`` is None) and the subclass none.  Returns the stock outputs and the word widths of the
    gathers it ran."""
    base = getattr(cfm_b200, MATCHERS[name])
    runs = []
    for klass in (base, type("Unfused" + base.__name__, (base,), {})):
        fm = klass(sigma)
        torch.manual_seed(seed)
        np.random.seed(seed)
        nf, ng = len(calls.flow), len(calls.gather)
        if labels is None:
            out = fm.sample_location_and_conditional_flow(x0, x1, t=t, return_noise=True)
        else:
            out = fm.guided_sample_location_and_conditional_flow(x0, x1, *labels, t=t, return_noise=True)
        runs.append((out, [_flow_instantiation(a) for a in calls.flow[nf:]],
                     [_gather_width(a) for a in calls.gather[ng:]]))
    (got, flows, gathers), (want, flows_ref, _) = runs
    names = ("t", "xt", "ut", "eps") if labels is None else ("t", "xt", "ut", "y0", "y1", "eps")
    for a, b, what in zip(got, want, names):
        if b is None:
            assert a is None, what
        else:
            _assert_same(a, b, f"{name} {what}")
    assert flows == ([fused] if fused else []) and flows_ref == [], (flows, flows_ref)
    return got, gathers


def _batch(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).to(DEV), (torch.randn(*shape, generator=g) * 1.7 + 0.3).to(DEV)


@gpu
@pytest.mark.parametrize("name,sigma", [("icfm", 0.5), ("icfm", 0), ("otcfm", 0), ("otcfm", 0.25), ("target", 0),
                                        ("target", 0.5), ("sb", 0.7), ("vp", 0.3), ("vp", 0)])
def test_matchers_at_t_zero_and_one(name, sigma, calls):
    """A caller's device t holding exact 0 and 1: SB's sigma_t = 0 with its +-1e8 coefficient, Target's 0/0 at
    sigma = 0; integer sigma = 0 as the reference allows it."""
    x0, x1 = _batch((256, 8), 20)
    t = torch.rand(256, generator=torch.Generator().manual_seed(21))
    t[:64:2], t[1:64:2] = 0.0, 1.0
    t = t.to(DEV)
    (tt, xt, ut, eps), _ = _stock_and_unfused(name, sigma, x0, x1, "true", calls, t=t)
    assert tt is t
    # the edge is reached: 0/0 only for Target at sigma = 0; SB's 1e8 coefficient multiplies an exact 0
    assert bool(torch.isnan(ut).any()) == (name == "target" and sigma == 0)
    assert name != "sb" or bool(torch.isfinite(ut).all())


def _layout(kind, name, seed):
    """(x0, x1, flow_pairs_kernel instantiation the stock class runs, or None) of one input layout.  A coupled
    matcher gathers a strided batch with torch indexing first: a transposed batch's rows x0[i] are contiguous and take
    the fused kernel with identity pairs, channels_last rows stay channels_last."""
    n = 64 if kind == "channels_last" else 256
    if kind == "odd_row":
        x0, x1 = _batch((n, 3, 7), seed)
        return x0, x1, "false"
    if kind == "offset":  # contiguous, one float past 16-byte alignment
        a, b = _batch((n, 8), seed)
        x0, x1 = _aligned(a.numel(), 1).view(n, 8), _aligned(b.numel(), 1).view(n, 8)
        x0.copy_(a)
        x1.copy_(b)
        return x0, x1, "false"
    coupled = name in ("otcfm", "sb")
    if kind == "x0_transposed":
        a, x1 = _batch((n, 12), seed)
        return a.t().contiguous().t(), x1, "true" if coupled else None
    if kind == "x1_transposed":
        x0, b = _batch((n, 12), seed)
        return x0, b.t().contiguous().t(), "true" if coupled else None
    a, b = _batch((n, 3, 32, 32), seed)
    return a.contiguous(memory_format=torch.channels_last), b, None


@gpu
@pytest.mark.parametrize("layout", ["odd_row", "offset", "x0_transposed", "x1_transposed", "channels_last"])
@pytest.mark.parametrize("name", list(MATCHERS))
def test_matchers_on_every_input_layout(name, layout, calls):
    """Contiguous batches take the fused kernel (the scalar instantiation for odd rows and misaligned batches); a
    transposed or channels_last batch, whose randn_like is not contiguous, takes the torch ops."""
    x0, x1, fused = _layout(layout, name, 30)
    (t, xt, ut, eps), _ = _stock_and_unfused(name, SIGMA[name], x0, x1, fused, calls)
    assert xt.shape == x0.shape


@gpu
@pytest.mark.parametrize("name", list(MATCHERS))
def test_matchers_with_a_float64_t_take_the_torch_ops(name, calls):
    x0, x1 = _batch((128, 8), 40)
    t = torch.rand(128, dtype=torch.float64, generator=torch.Generator().manual_seed(41)).to(DEV)
    (tt, xt, ut, eps), _ = _stock_and_unfused(name, SIGMA[name], x0, x1, None, calls, t=t)
    assert xt.dtype == torch.float64 and eps.dtype == torch.float32


def _labels(dtype, shape, seed):
    g = torch.Generator().manual_seed(seed)
    if dtype == torch.bool:
        return (torch.rand(shape, generator=g) < 0.5).to(DEV)
    if dtype == torch.float16:  # random bits: NaN payloads and -0 among them
        return torch.randint(-2**15, 2**15, shape, dtype=torch.int16, generator=g).view(torch.float16).to(DEV)
    return torch.randint(-2**31, 2**31, shape, dtype=torch.int64, generator=g).to(dtype).to(DEV)


@gpu
@pytest.mark.parametrize("shape", [(), (1,), (3,)])
@pytest.mark.parametrize("dtype", ["int64", "int32", "float16", "bool"])
@pytest.mark.parametrize("name", ["otcfm", "sb"])
def test_guided_labels_follow_the_pairs(name, dtype, shape, calls):
    """Labels are gathered by cfm_gather_rows at the word width their row bytes give; they equal y0[i], y1[j] of the
    same draw, read back from a second sampler with the same seed."""
    n, dtype = 128, getattr(torch, dtype)
    x0, x1 = _batch((n, 6), 50)
    y0, y1 = _labels(dtype, (n,) + shape, 51), _labels(dtype, (n,) + shape, 52)
    (t, xt, ut, l0, l1, eps), gathers = _stock_and_unfused(name, SIGMA[name], x0, x1, "false", calls,
                                                           labels=(y0, y1), seed=53)
    torch.manual_seed(53)
    np.random.seed(53)
    i, j = getattr(cfm_b200, MATCHERS[name])(SIGMA[name]).ot_sampler.sample_pairs(x0, x1)
    _assert_same(l0, y0[i], "y0[i]")
    _assert_same(l1, y1[j], "y1[j]")
    assert gathers == [math.gcd(y0.element_size() * (shape[0] if shape else 1), 16)] * 2


# ================================================================================= GPU (c): cfm_gather_rows
def _random_rows(n, row, elem, offset, seed):
    """(n, row) rows of element size ``elem`` holding random bits (NaN payloads and -0 among them), starting
    ``offset`` elements past an aligned allocation."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    bits = torch.randint(0, 256, ((n * row + offset) * elem,), dtype=torch.uint8, device=DEV, generator=g)
    return bits.view(_ELEM_DTYPE[elem])[offset:].view(n, row)


class _GatherCase:
    """Source, indices and a guarded output ``out_offset`` elements into a buffer of 0x5A bytes."""

    def __init__(self, x, idx, width, out_offset=0):
        self.x, self.idx, self.width, self.off = x, idx, width, out_offset
        n_idx, row, elem = idx.shape[0], x.shape[1], x.element_size()
        self.buf = torch.full(((out_offset + n_idx * row + 64) * elem,), 0x5A, dtype=torch.uint8, device=DEV)
        self.out = self.buf.view(_ELEM_DTYPE[elem])[out_offset:out_offset + n_idx * row].view(n_idx, row)
        self.words = n_idx * row * elem // width

    def __call__(self):
        return _ffi.lib().cfm_gather_rows(_ffi.ptr(self.x), self.x.shape[1], self.x.element_size(),
                                          _ffi.ptr(self.idx), self.idx.shape[0], _ffi.ptr(self.out),
                                          _ffi.stream_ptr(DEV))

    def check(self, calls):
        """One launch at the expected word width; bit equality with index_select; no write outside the output."""
        rc, launches = _launches(self)
        assert rc == 0 and launches == 1, _ffi.last_error()
        assert [_gather_width(a) for a in calls.gather[-1:]] == [self.width]
        _assert_same(_bits(self.out), _bits(torch.index_select(self.x, 0, self.idx)), "out")
        elem = self.x.element_size()
        inside = torch.zeros_like(self.buf, dtype=torch.bool)
        inside[self.off * elem:self.off * elem + self.out.numel() * elem] = True
        assert bool((self.buf[~inside] == 0x5A).all()), "write outside the output rows"


def _width_case(elem, width, how):
    """'row': 3 words of the width per row (48 bytes for uint4), aligned pointers.  'x_offset' / 'out_offset': 48-byte
    rows with the source or the output that width's bytes past 16-byte alignment (16 bytes keeps uint4).  'single':
    rows of one element."""
    if how == "single":
        return _GatherCase(_random_rows(500, 1, elem, 0, seed=elem), _indices(777, 500, elem), width)
    row_bytes = 48 if how != "row" or width == 16 else 3 * width
    shift = width // elem if how != "row" else 0
    x = _random_rows(300, row_bytes // elem, elem, shift if how == "x_offset" else 0, seed=elem * 100 + width)
    return _GatherCase(x, _indices(1000, 300, width), width, shift if how == "out_offset" else 0)


def _width_cases():
    return [(e, w, h) for e, w in itertools.product((1, 2, 4, 8), (1, 2, 4, 8, 16)) if w >= e
            for h in ("row", "x_offset", "out_offset")] + [(e, e, "single") for e in (1, 2, 4, 8)]


@gpu
@pytest.mark.parametrize("elem,width,how", _width_cases())
def test_gather_reaches_every_word_width(elem, width, how, calls):
    _width_case(elem, width, how).check(calls)



def _grid_case(width, size):
    """1 word, exactly one pass of the capped grid, one more, and at least three passes on 5-word rows."""
    cap = _pass_threads()
    n_idx, words = {"one": (1, 1), "pass": (cap, 1), "pass+1": (cap + 1, 1), "passes3": (3 * cap // 5 + 7, 5)}[size]
    elem = min(width, 8)
    x = _random_rows(1000, words * width // elem, elem, 0, seed=width)
    return _GatherCase(x, _indices(n_idx, 1000, width), width)


GRID_SIZES = ["one", "pass", "pass+1", "passes3"]


@gpu
@pytest.mark.parametrize("size", GRID_SIZES)
@pytest.mark.parametrize("width", [1, 2, 4, 8, 16])
def test_gather_grid_passes(width, size, calls, record_property):
    """At three passes the launch time must show that no word is visited twice."""
    c = _grid_case(width, size)
    c.check(calls)
    if size == "passes3":
        record_property("time_over_bound",
                        _assert_each_thread_visits_its_work_once(_shortest_launch_us(c), 2 * c.words * width))



@gpu
def test_gather_byte_rows_past_two_gigabytes(calls):
    """uint8 rows of 4097 bytes (the byte path) in a source just over 2^31 bytes, read at its last rows: word offsets
    past 2^31 need the kernel's 64-bit index arithmetic.  About 2.15 GB in all."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    row = 4097
    n_src = 2**31 // row + 3
    assert n_src * row > 2**31
    x = torch.randint(0, 256, (n_src, row), dtype=torch.uint8, device=DEV,
                      generator=torch.Generator(device=DEV).manual_seed(60))
    idx = torch.tensor([n_src - 1, 0, n_src - 2, n_src - 1, n_src // 2, n_src - 3, n_src - 1] * 9, device=DEV)
    _GatherCase(x, idx, 1).check(calls)
    assert torch.cuda.max_memory_allocated() < 3e9
    del x
    torch.cuda.empty_cache()


# ============================================================== GPU: dispatch read from the profiler
FLOW_CLASSES = [(r, s) for r in ("vec", "odd_row") for s in ("one", "pass", "pass+1", "passes3")] + [
    ("offset:x0", "one"), ("offset:x1", "pass"), ("offset:eps", "passes3"), ("offset:xt", "one"), ("offset:ut", "pass")]
FAMILIES = {"flow": lambda: [_FlowCase("icfm", r, s, MODES[0]) for r, s in FLOW_CLASSES],
            "grid": lambda: [_grid_case(w, s) for w in (1, 2, 4, 8, 16) for s in GRID_SIZES]}
FAMILIES.update({f"gather{elem}": (lambda elem=elem: [_width_case(*c) for c in _width_cases() if c[0] == elem])
                 for elem in (1, 2, 4, 8)})


def _dispatch_traces(tmp_dir):
    """Run in a child process: one trace per family of launches, one launch of every dispatch class; prints
    {family: {rcs, launches, expected, ran}} as JSON."""
    out = {}
    for family, make in FAMILIES.items():
        cases = make()
        (rcs, launches), ran = _profiled(lambda: _launches(lambda: [c() for c in cases]), pathlib.Path(tmp_dir),
                                         len(cases))
        expected = [("flow_pairs", "true" if c.vec else "false", _grid(c.work), BLOCK) if family == "flow" else
                    ("gather_rows", GATHER_WORDS[c.width][0], _grid(c.words), BLOCK) for c in cases]
        out[family] = {"rcs": rcs, "launches": launches, "expected": expected, "ran": ran}
        del cases
    print(json.dumps(out))


@pytest.fixture(scope="module")
def traces(tmp_path_factory):
    code = "import sys; sys.path[:0] = sys.argv[1:3]; import test_gpu_flow_gather as t; t._dispatch_traces(sys.argv[3])"
    r = subprocess.run([sys.executable, "-c", code, os.path.dirname(TESTS), TESTS,
                        str(tmp_path_factory.mktemp("traces"))], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@gpu
@pytest.mark.parametrize("family", list(FAMILIES))
def test_dispatch_read_from_the_profiler(family, traces):
    """Each launch ran flow_pairs_kernel<VEC> or gather_rows_kernel<W> as the dispatch rule says, on the grid capped
    at 16 CTAs per SM; every instantiation appears."""
    t = traces[family]
    assert t["rcs"] == [0] * len(t["expected"]) and t["launches"] == len(t["expected"])
    assert t["ran"] == t["expected"], t["ran"]


@gpu
def test_dispatch_traces_name_every_instantiation(traces):
    ran = {(r[0], r[1]) for t in traces.values() for r in t["ran"]}
    assert ran == {("flow_pairs", v) for v in FLOW_VEC} | {("gather_rows", w) for w, _ in GATHER_WORDS.values()}


# ====================================================================== GPU (d): OTPlanSampler._gather routing
def _fallback_input(kind):
    g = torch.Generator().manual_seed(70)
    x = torch.randn(200, 6, generator=g)
    if kind == "requires_grad":
        return x.to(DEV).requires_grad_()
    if kind == "cpu":
        return x
    if kind == "non_contiguous":
        return x.to(DEV)[:, ::2]
    return torch.complex(x, -x).to(torch.complex128).to(DEV)  # itemsize 16


@gpu
@pytest.mark.parametrize("kind", ["requires_grad", "cpu", "non_contiguous", "complex128"])
def test_gather_fallback_inputs_take_torch_indexing(kind, calls):
    x = _fallback_input(kind)
    idx = _indices(300, 200, 71)
    out, launches = _launches(lambda: OTPlanSampler._gather(x, idx))
    assert launches == 0 and calls.gather == []
    want = x[idx.to(x.device)]
    assert out.requires_grad == x.requires_grad and out.device == x.device
    out, want = out.detach(), want.detach()
    if out.is_complex():
        out, want = torch.view_as_real(out), torch.view_as_real(want)
    _assert_same(out, want, kind)


@gpu
def test_gather_contiguous_device_input_takes_the_kernel(calls):
    x = torch.randn(200, 6, device=DEV)
    idx = _indices(300, 200, 72)
    out, launches = _launches(lambda: OTPlanSampler._gather(x, idx))
    assert launches == 1 and [_gather_width(a) for a in calls.gather] == [8]
    _assert_same(out, x[idx], "x[idx]")


@gpu
@pytest.mark.parametrize("host", ["pinned_f32", "pageable_f32", "f64"])
def test_sample_plan_on_host_inputs_returns_host_rows(host):
    g = torch.Generator().manual_seed(80)
    x0, x1 = torch.randn(128, 2, 5, generator=g), torch.randn(128, 2, 5, generator=g) + 1
    if host == "f64":
        x0, x1 = x0.double(), x1.double()
    elif host == "pinned_f32":
        x0, x1 = x0.pin_memory(), x1.pin_memory()
    np.random.seed(81)
    i, j = OTPlanSampler("exact").sample_pairs(x0, x1)
    np.random.seed(81)
    a, b = OTPlanSampler("exact").sample_plan(x0, x1)
    _assert_same(a, x0[i.cpu()], "x0[i]")
    _assert_same(b, x1[j.cpu()], "x1[j]")
