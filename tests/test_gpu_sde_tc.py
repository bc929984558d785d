"""Schrodinger-bridge SDE sampling with WIDE drift and score nets (cfm_b200.sdeint's tensor-core class: the pair
forward mlp_pair_h3_kernel in csrc/mlp_h3.cu and the Euler-Maruyama step in csrc/sde_tc.cu) against the float64
restatement of torchsde's fixed-step Euler (oracle/sde.py).

CPU: argument checks before any CUDA call, the class predicate against the tensor-core shape rule, and the kernel
instantiations in the built library.
GPU: parity with supplied increments (per-layer path, the C3 model, a ragged K chunk, CTAs that switch from drift to
score slabs), by max-abs and per entry; the pair launch against two single launches, bit for bit, also across the slab
schedules of tests/tc_sampler_cases.py; bit identity with the wide Euler ODE path; one noise stream across both
classes; the device's own noise on a non-uniform step grid against float64, per entry (small_field_oracle.Bounded); rows independent of the batch;
graph against eager replay and the launch count; weights updated in place; dispatch and refusals."""
import ctypes
import functools
import math
import re
import subprocess

import numpy as np
import pytest
import torch

import cnf_tc_oracle as ho
import small_field_oracle as sfo
import tc_sampler_cases as tc
from oracle import sde as osde
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi
from cfm_b200 import sde as csde

DEV = "cuda:0"
gpu = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _many_slabs_batch():
    """A batch with SMs / 2 + 3 slabs of 128 rows per net: the pair launch has more slabs than CTAs, so CTAs run a
    drift slab and then a score slab."""
    return 128 * (_sms() // 2 + 3) - 5


def _nets(dim, w, seed, act="selu", zero_score=False, zero_drift=False):
    """(device nets, float64 device oracle nets) with the same weights."""
    torch.manual_seed(seed)
    out = []
    for zero in (zero_drift, zero_score):
        m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
        if zero:
            with torch.no_grad():
                m.net[6].weight.zero_()
                m.net[6].bias.zero_()
        mc = vf.make_mlp(dim, w=w, time_varying=True, dtype=torch.float64)
        mc.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
        if act == "silu":
            m.act = _ffi.ACT_SILU
            for k in (1, 3, 5):
                mc.net[k] = torch.nn.SiLU()
        out.append((m.to(DEV), mc.to(DEV)))
    return out


def _sde(dim, w, seed, sigma=1.0, **kw):
    (d, dc), (s, sc) = _nets(dim, w, seed, **kw)
    sde = cfm_b200.SDE(d, s, input_size=(dim,), sigma=sigma)

    def f64(t, y):
        tt = torch.tensor(t, dtype=torch.float64, device=y.device)
        return vf.wrapped_forward(dc, tt, y) + vf.wrapped_forward(sc, tt, y)
    return sde, f64


class DeviceBM:
    """Brownian increments N(0, tb - ta) drawn on the device from a seeded generator; keeps them for the oracle."""

    def __init__(self, B, D, seed, zero=False):
        self.g = torch.Generator(device=DEV).manual_seed(seed)
        self.B, self.D, self.zero, self.incs = B, D, zero, []

    def __call__(self, ta, tb):
        h = float(tb - ta)
        z = torch.zeros(self.B, self.D, device=DEV) if self.zero else \
            torch.randn(self.B, self.D, generator=self.g, device=DEV) * h ** 0.5
        self.incs.append(z)
        return z


def _launches(fn):
    L = _ffi.lib()
    before = L.cfm_launch_count()
    out = fn()
    return out, L.cfm_launch_count() - before


# the step-by-step trajectory bound and the Box-Muller radius uniform, shared with the small SDE kernel's tests
_radius_uniform = sfo.radius_uniform
_Bounded = functools.partial(sfo.Bounded, net_err=sfo.tc_net_err)


def _split(x):
    """The fp16x3 operand pair of x (finite, within fp16 range): hi = fp16(x), lo = fp16((x - hi) 2^11)."""
    hi = x.half()
    return hi, ((x - hi.float()) * 2048).half()


# ---- CPU: argument checks, the class predicate, the instantiations --------------------------------------------------
def test_tc_entry_points_check_their_arguments_before_any_cuda_call(lib_built):
    """Dummy host pointers that no call may dereference: each case fails its check before a launch."""
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(4096)
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    odd = p + 4
    f = ctypes.c_float

    def init(*, st=p, y0=p, y=p, n_steps=3, B=256, D=64):
        return lib.cfm_sde_tc_init(st, y0, y, p, p, p, None, 7, p, n_steps, B, D, None)

    def step(*, st=p, y=p, drift=p, B=256, D=64):
        return lib.cfm_sde_tc_euler_step(st, y, drift, p, p, p, p, p, p, p, f(0.5), B, D, None)

    def pair(*, a=p, b=p, B=256, D=64, w=256, ws_bytes=0):
        return lib.cfm_mlp_pair_forward_split_f32(a, b, p, p, B, D, w, D, 1, p, f(0.0), 0, p, p, p, ws_bytes, None)

    cases = [
        (lambda: init(st=None), "null pointer"), (lambda: init(y0=None), "null pointer"),
        (lambda: init(n_steps=0), "n_steps"), (lambda: init(n_steps=-2), "n_steps"),
        (lambda: init(B=127), "unsupported shape"), (lambda: init(D=36), "unsupported shape"),
        (lambda: init(D=24), "unsupported shape"), (lambda: init(y=odd), "16-byte aligned"),
        (lambda: init(y0=odd), "16-byte aligned"), (lambda: init(st=p + 4), "8-byte aligned"),
        (lambda: step(drift=None), "null pointer"), (lambda: step(B=64), "unsupported shape"),
        (lambda: step(D=100), "unsupported shape"), (lambda: step(y=odd), "16-byte aligned"),
        (lambda: step(drift=odd), "16-byte aligned"),
        (lambda: pair(b=None), "null pointer"), (lambda: pair(w=36), "shape not supported"),
        (lambda: pair(w=24), "shape not supported"), (lambda: pair(B=100), "shape not supported"),
        (lambda: pair(D=33), "shape not supported"), (lambda: pair(), "workspace too small"),
        (lambda: pair(w=128), "workspace too small"),
    ]
    for fn, msg in cases:
        assert fn() == -1
        assert msg.encode() in lib.cfm_last_error(), (msg, lib.cfm_last_error())


def test_supported_is_the_tensor_core_shape_rule(lib_built):
    lib = _ffi.load_library(lib_built)
    for B in (1, 64, 127, 128, 129, 1000, 1 << 20):
        for d in (2, 8, 24, 31, 32, 36, 40, 63, 64, 200, 784, 785):
            for w in (8, 24, 30, 32, 36, 64, 128, 256, 260):
                want = B >= 128 and d >= 32 and d % 8 == 0 and w % 8 == 0 and w >= 32
                assert lib.cfm_sde_tc_supported(B, d, w) == lib.cfm_mlp_tc_supported(B, d, w, d) == int(want), (B, d, w)


def test_compiled_sde_tc_instantiations_are_the_tested_ones(lib_built):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    pair = set(re.findall(r"\w*mlp_pair_h3_kernel\w*", out))
    assert {re.search(r"mlp_pair_h3_kernelILi(\d+)EEEv", s).group(1) for s in pair} == \
        {str(_ffi.ACT_SELU), str(_ffi.ACT_SILU)} and len(pair) == 2, pair
    assert len(set(re.findall(r"\w*sde_tc_step_kernel\w*", out))) == 1
    assert len(set(re.findall(r"\w*sde_tc_init_kernel\w*", out))) == 1


def test_sde_state_struct_layout_matches_header():
    assert ctypes.sizeof(_ffi.SdeState) == 40
    assert _ffi.SdeState.t.offset == 32 and _ffi.SdeState.ticket.offset == 36


# ---- GPU: parity with supplied increments --------------------------------------------------------------------------
_TS = {"offgrid": (torch.tensor([0.0, 0.0137, 0.05, 0.0501, 0.2, 0.31]), 7e-3),
       "sf2m": (torch.linspace(0, 1, 100), 1e-3)}
# (B, dim, w, act): the per-layer path; the C3 model with a ragged last slab; a ragged K chunk (200 = 3 x 64 + 8);
# CTAs switching nets (B from the device's SM count)
_SHAPES = [(200, 32, 128, "selu"), (1000, 784, 256, "selu"), (300, 200, 256, "silu"), (None, 64, 256, "selu")]


@gpu
@pytest.mark.parametrize("kind", ["offgrid", "sf2m"])
@pytest.mark.parametrize("B,dim,w,act", _SHAPES)
def test_parity_with_supplied_increments(B, dim, w, act, kind, record_property):
    """Two gates: the trajectory's max-abs, and per entry the bound _Bounded carries step by step."""
    B = B or _many_slabs_batch()
    (d, dc), (s, sc) = _nets(dim, w, seed=dim + w, act=act)
    sde = cfm_b200.SDE(d, s, input_size=(dim,), sigma=0.8)
    ts, dt = _TS[kind]
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(dim)).to(DEV)
    bm = DeviceBM(B, dim, seed=w + dim)
    ys = cfm_b200.sdeint(sde, y0, ts, bm=bm, method="euler", dt=dt)
    assert ys.shape == (len(ts), B, dim) and ys.dtype == torch.float32 and ys.device.type == "cuda"
    assert torch.equal(ys[0], y0)
    incs = torch.stack(bm.incs).double()
    del bm
    field = _Bounded((dc, sc), act, ts, dt, 0.8, incs)
    ref = osde.euler_sdeint(field, 0.8, y0.double(), ts, dt, incs)
    err = (ys.double() - ref).abs()
    gate = 1e-4 * max(1.0, ref.abs().max().item())
    record_property("err_over_gate", err.max().item() / gate)
    assert err.max().item() <= gate, (err.max().item(), gate)
    lip = ho.lipschitz(dc, act) + ho.lipschitz(sc, act)
    bound = field.bound(math.exp(float(ts[-1] - ts[0]) * lip))
    print(f"margins sde parity {B}x{dim}x{w} {kind}: max-abs {err.max().item() / gate:.3f}, per entry "
          f"{float((err / bound)[1:].max()):.2e} of the gate (Lip {lip:.1f})")
    assert bool((err <= bound).all()), float((err / bound)[1:].max())


# ---- GPU: the pair launch is two single launches -------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("B,dim,w", [(s[0], s[1], s[2]) for s in _SHAPES] + tc.PAIR_SHAPES)
def test_pair_launch_equals_two_single_launches_bit_for_bit(B, dim, w, act):
    """Also at the slab schedules of tests/tc_sampler_cases.py: one slab per net, one slab per CTA, 2 S = grid + 2,
    S >= SMs (two drift slabs before a score slab) and a ragged drift slab followed by a score slab on one CTA."""
    B = _many_slabs_batch() if B is None else tc.batch(B, _sms())
    (d, _), (s, _) = _nets(dim, w, seed=3 * dim + w, act=act)
    L = _ffi.lib()
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(5)).to(DEV)
    hi, lo = _split(x)
    t = torch.tensor([0.37], device=DEV)
    blobs = [m._prepared(True, torch.device(DEV)) for m in (d, s)]
    one = L.cfm_mlp_workspace_bytes(B, dim, w, dim, 2)
    ws = _ffi.workspace(2 * one, DEV)
    sp = _ffi.stream_ptr(DEV)
    ya, yb = torch.full((B, dim), float("nan"), device=DEV), torch.full((B, dim), float("nan"), device=DEV)
    _, n = _launches(lambda: _ffi.check(L.cfm_mlp_pair_forward_split_f32(
        _ffi.ptr(blobs[0]), _ffi.ptr(blobs[1]), _ffi.ptr(hi), _ffi.ptr(lo), B, dim, w, dim, 1, _ffi.ptr(t), 0.0, d.act,
        _ffi.ptr(ya), _ffi.ptr(yb), _ffi.ptr(ws), ws.numel(), sp), "pair"))
    assert n == (1 if w == 256 and dim >= 64 else 8)
    for blob, got in zip(blobs, (ya, yb)):
        want = torch.full((B, dim), float("nan"), device=DEV)
        _ffi.check(L.cfm_mlp_forward_split_gated_f32(
            _ffi.ptr(blob), _ffi.ptr(hi), _ffi.ptr(lo), B, dim, w, dim, 1, _ffi.ptr(t), 0.0, d.act, _ffi.ptr(want),
            None, _ffi.ptr(ws), one, sp), "single")
        assert torch.isfinite(got).all() and torch.equal(got, want)


# ---- GPU: bit identity with the wide Euler ODE path; sigma = 0 -----------------------------------------------------
@gpu
@pytest.mark.parametrize("B,dim,w,act", [(500, 64, 256, "selu"), (200, 32, 128, "silu")])
def test_zero_score_and_zero_noise_equal_the_wide_ode_euler_bit_for_bit(B, dim, w, act):
    sde, _ = _sde(dim, w, seed=70 + w, act=act, zero_score=True)
    grid, *_ = csde.step_schedule(torch.linspace(0, 1, 11), 1e-2)
    ts = torch.from_numpy(grid)
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(71)).to(DEV)
    ys = cfm_b200.sdeint(sde, y0, ts, bm=DeviceBM(B, dim, 0, zero=True), method="euler", dt=1e-2)
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(sde.drift), solver="euler")
    node.use_fused_small = False  # the wide path: one tensor-core forward and one axpy per step
    assert sde.drift.tc_path(B)
    ode = node.trajectory(y0, ts)
    assert ys.shape == ode.shape and torch.equal(ys, ode)
    sde.sigma = 0.0
    assert torch.equal(cfm_b200.sdeint(sde, y0, ts, method="euler", dt=1e-2), ys)


# ---- GPU: one noise stream across the two classes -----------------------------------------------------------------
@gpu
def test_one_noise_stream_across_the_small_and_tensor_core_classes():
    B = 1000
    ts = torch.arange(0, 5, dtype=torch.float32)
    tc, _ = _sde(64, 256, seed=110, zero_score=True, zero_drift=True)
    small, _ = _sde(8, 32, seed=111, zero_score=True, zero_drift=True)
    L = _ffi.lib()
    assert L.cfm_sde_tc_supported(B, 64, 256) and not L.cfm_sde_small_supported(B, 64, 256)
    assert L.cfm_sde_small_supported(B, 8, 32)
    torch.manual_seed(11)
    a = cfm_b200.sdeint(tc, torch.zeros(B, 64, device=DEV), ts, method="euler", dt=1.0)
    torch.manual_seed(11)
    b, n = _launches(lambda: cfm_b200.sdeint(small, torch.zeros(B, 8, device=DEV), ts, method="euler", dt=1.0))
    assert n == 1  # the small class ran sde_small_kernel
    assert torch.equal(a[:, :, :8], b)
    torch.manual_seed(11)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    dz = (a[1:] - a[:-1]).cpu().double().numpy()
    for n in range(4):
        z = osde.device_normals(seed, n, np.arange(B), 64)
        # the device rounds a radius uniform u >= 1/2 to fp32 (2^-25 apart from the float64 one), which moves
        # sqrt(-2 log u) by up to 2^-25 / sqrt(-2 log u): more than the gate only for u within ~2^-12 of 1
        near_one = _radius_uniform(seed, n, np.arange(B), 64) > 1 - 2.0**-12
        assert near_one.mean() < 1e-3
        ok = np.abs(dz[n] - z) <= 1e-5 * np.maximum(1.0, np.abs(z))
        assert (ok | near_one).all(), n


# ---- GPU: the device's own noise against float64 -------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B,dim,w,act", tc.NOISE_SHAPES)
def test_own_noise_against_float64_entry_by_entry(B, dim, w, act):
    """bm=None on a step grid whose h changes (an off-grid ts, a dt that does not divide the span): the step kernel
    draws dW_n = sqrt(h_n) z_n itself.  On the rows of tc.noise_rows (the first, both sides of every 128-row slab
    boundary, the last) the trajectory stays within _Bounded's per-entry bound of the float64 Euler loop driven by
    osde.device_normals(seed, n) sqrt(h_n).  The device increment errs by at most sqrt(h_n) (2^-23 / rad + 2^-20 rad +
    2^-23 |z|) per entry, rad = sqrt(-2 log u) the Box-Muller radius: the fp32 rounding of a radius uniform u >= 1/2
    moves rad by up to 2^-24 / rad, logf, sqrtf, sincospif and the angle's rounding by a few units of 2^-24 of rad,
    the products by 2^-24 each."""
    (d, dc), (s, sc) = _nets(dim, w, seed=150 + dim, act=act)
    with torch.no_grad():
        for m in (d, dc, s, sc):
            for li in (2, 4, 6):
                m.net[li].weight.mul_(0.4)
    lip = ho.lipschitz(dc, act) + ho.lipschitz(sc, act)
    assert lip < 2, lip
    sigma, dt = tc.NOISE_SIGMA, tc.NOISE_DT
    sde = cfm_b200.SDE(d, s, input_size=(dim,), sigma=sigma)
    ts = torch.tensor(tc.NOISE_TS, dtype=torch.float32)
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(151)).to(DEV)
    torch.manual_seed(152)
    ys = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=dt)
    torch.manual_seed(152)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    rows = tc.noise_rows(B)
    grid, _ = osde.step_grid(ts, dt)
    incs, errs = [], []
    for n in range(len(grid) - 1):
        root = float(grid[n + 1] - grid[n]) ** 0.5
        z = osde.device_normals(seed, n, rows, dim)
        rad = np.sqrt(-2.0 * np.log(_radius_uniform(seed, n, rows, dim)))
        incs.append(torch.from_numpy(z * root))
        errs.append(torch.from_numpy(root * (2.0**-23 / rad + 2.0**-20 * rad + 2.0**-23 * np.abs(z))))
    incs, errs = torch.stack(incs).to(DEV), torch.stack(errs).to(DEV)
    field = _Bounded((dc, sc), act, ts, dt, sigma, incs, errs)
    ref = osde.euler_sdeint(field, sigma, y0[rows].double(), ts, dt, incs)
    bound = field.bound(math.exp(float(ts[-1] - ts[0]) * lip))
    err = (ys[:, rows].double() - ref).abs()
    print(f"margins sde own noise {B}x{dim}x{w} {act}: {float((err / bound)[1:].max()):.3f} of the gate")
    assert bool((err <= bound).all()), float((err / bound)[1:].max())


# ---- GPU: rows independent of the batch; seeding --------------------------------------------------------------------
@gpu
def test_rows_are_independent_of_the_batch_and_the_seed_reproduces():
    sde, _ = _sde(64, 256, seed=90, sigma=0.5)
    y0 = torch.randn(3000, 64, generator=torch.Generator().manual_seed(91)).to(DEV)
    ts = torch.linspace(0, 1, 5)
    runs = []
    for s, rows in ((5, 3000), (5, 1000), (5, 3000), (6, 3000)):
        torch.manual_seed(s)
        runs.append(cfm_b200.sdeint(sde, y0[:rows], ts, method="euler", dt=0.02))
    assert torch.equal(runs[1], runs[0][:, :1000])
    assert torch.equal(runs[0], runs[2])
    assert not torch.equal(runs[0][1:], runs[3][1:]) and torch.equal(runs[0][0], runs[3][0])


# ---- GPU: graph and eager -------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B,dim,w,per_step", [(1000, 64, 256, 2), (200, 32, 128, 9)])
def test_graph_and_eager_give_the_same_bits_and_two_launches_per_step(B, dim, w, per_step, monkeypatch):
    sde, _ = _sde(dim, w, seed=120, sigma=0.7)
    ts = torch.linspace(0, 1, 5)
    n_steps = len(csde.step_schedule(ts, 0.05)[0]) - 1
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(121)).to(DEV)
    raw = torch.empty(B * dim + 1, device=DEV)[1:].view(B, dim)  # a 4-byte-misaligned y0 is copied, not refused
    raw.copy_(y0)
    runs = []
    for eager in (False, False, True, False):
        monkeypatch.setattr(csde, "_EAGER", eager)
        torch.manual_seed(3)
        ys, n = _launches(lambda: cfm_b200.sdeint(sde, raw if eager else y0, ts, method="euler", dt=0.05))
        runs.append((ys, n))
    for ys, _ in runs[1:]:
        assert torch.equal(ys, runs[0][0])
    assert runs[2][1] == 1 + per_step * n_steps  # eager: the init, then (pair forward + step) per step
    assert runs[1][1] == 1 and runs[3][1] == 1   # replays: the init only


# ---- GPU: weights updated in place ----------------------------------------------------------------------------------
@gpu
def test_weights_updated_in_place_give_the_trajectory_of_fresh_nets():
    dim, w, B = 64, 256, 512
    sde, _ = _sde(dim, w, seed=130, sigma=0.3)
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(131)).to(DEV)
    ts = torch.linspace(0, 1, 3)
    torch.manual_seed(1)
    before = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=0.1)
    params = list(sde.drift.parameters()) + list(sde.score.parameters())
    opt = torch.optim.Adam(params, lr=1e-3)
    g = torch.Generator(device=DEV).manual_seed(132)
    for _ in range(3):  # SF2M: flow loss on the drift, the score loss through row_scale = lambda_t
        xt = torch.randn(256, dim, generator=g, device=DEV)
        t = torch.rand(256, generator=g, device=DEV)
        ut, eps = torch.randn(256, dim, generator=g, device=DEV), torch.randn(256, dim, generator=g, device=DEV)
        lam = torch.rand(256, generator=g, device=DEV) + 0.5
        opt.zero_grad()
        loss = cfm_b200.flow_matching_loss(sde.drift, xt, t, ut) + \
            cfm_b200.flow_matching_loss(sde.score, xt, t, -eps, row_scale=lam)
        loss.backward()
        opt.step()
    torch.manual_seed(1)
    after = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=0.1)
    fresh = []
    for m in (sde.drift, sde.score):
        c = cfm_b200.MLP(dim, w=w, time_varying=True).to(DEV)
        c.load_state_dict(m.state_dict())
        fresh.append(c)
    torch.manual_seed(1)
    want = cfm_b200.sdeint(cfm_b200.SDE(*fresh, input_size=(dim,), sigma=0.3), y0, ts, method="euler", dt=0.1)
    assert not torch.equal(after, before)
    assert torch.equal(after, want)


# ---- GPU: dispatch and refusals -------------------------------------------------------------------------------------
@gpu
def test_a_shape_both_classes_take_runs_the_small_kernel():
    L = _ffi.lib()
    assert L.cfm_sde_small_supported(1024, 32, 32) and L.cfm_sde_tc_supported(1024, 32, 32)
    sde, _ = _sde(32, 32, seed=140)
    y0 = torch.randn(1024, 32, generator=torch.Generator().manual_seed(141)).to(DEV)
    ys, n = _launches(lambda: cfm_b200.sdeint(sde, y0, torch.linspace(0, 1, 4), method="euler", dt=0.05))
    assert n == 1 and ys.shape == (4, 1024, 32)


@gpu
def test_refusals_name_both_classes_and_launch_nothing():
    L = _ffi.lib()
    cases = [(64, 2, 128), (8, 400, 64), (127, 64, 256), (256, 36, 256), (256, 64, 36)]
    for B, dim, w in cases:
        assert not L.cfm_sde_small_supported(B, dim, w) and not L.cfm_sde_tc_supported(B, dim, w)
        sde = cfm_b200.SDE(cfm_b200.MLP(dim, w=w, time_varying=True).to(DEV),
                           cfm_b200.MLP(dim, w=w, time_varying=True).to(DEV), input_size=(dim,))
        before = L.cfm_launch_count()
        with pytest.raises(NotImplementedError, match=r"w in \{32, 64\}.*tensor-core class"):
            cfm_b200.sdeint(sde, torch.zeros(B, dim, device=DEV), torch.linspace(0, 1, 5), method="euler")
        assert L.cfm_launch_count() == before
