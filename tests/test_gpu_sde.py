"""Schrodinger-bridge SDE sampling (cfm_b200.SDE, cfm_b200.sdeint; csrc/ode_small.cu sde_small_kernel) against the
float64 restatement of torchsde's fixed-step Euler (oracle/sde.py).

CPU: the SDE class's f and g, every refusal that needs no device, the oracle's step grid and interpolation, the
package's host tables against the oracle, the NumPy Philox4x32-10 against Random123's known answers, and the kernel
instantiations in the built library.
GPU: parity with supplied increments over widths, dimensions, activations and both kinds of ts; bit identity with the
ODE kernel's Euler; sigma = 0; seeding; row independence across launch shapes (one test per instantiation); the
device generator's mapping; the increments' statistics; no launch on refusal."""
import re
import subprocess

import numpy as np
import pytest
import torch

from oracle import sde as osde
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi
from cfm_b200 import sde as csde

DEV = "cuda:0"
gpu = pytest.mark.gpu

# sde_small_kernel<U, MAXT> instantiations (U = w / 32, MAXT = threads per CTA); the planner gives at most 16 warps
SDE_KERNELS = [(1, 256), (2, 256), (1, 512), (2, 512)]
_KERNEL_RE = re.compile(r"sde_small_kernel<(\d), (\d+)>")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _nets(dim, w, seed, act="selu", zero_score=False, zero_drift=False):
    """(device SDE nets, float64 CPU oracle nets) with the same weights."""
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
        out.append((m, mc))
    return out


def _sde(dim, w, seed, sigma=1.0, **kw):
    (d, dc), (s, sc) = _nets(dim, w, seed, **kw)
    sde = cfm_b200.SDE(d.to(DEV), s.to(DEV), input_size=(dim,), sigma=sigma)

    def f64(t, y):
        return vf.wrapped_forward(dc, torch.tensor(t, dtype=torch.float64), y) + \
            vf.wrapped_forward(sc, torch.tensor(t, dtype=torch.float64), y)
    return sde, f64


class FixedBM:
    """Brownian increments N(0, tb - ta) from a seeded CPU generator; keeps them for the oracle."""

    def __init__(self, B, D, seed, zero=False):
        self.g = torch.Generator().manual_seed(seed)
        self.B, self.D, self.zero, self.incs = B, D, zero, []

    def __call__(self, ta, tb):
        h = float(tb - ta)
        z = torch.zeros(self.B, self.D) if self.zero else torch.randn(self.B, self.D, generator=self.g) * h ** 0.5
        self.incs.append(z)
        return z.to(DEV)


def _launches(fn):
    L = _ffi.lib()
    before = L.cfm_launch_count()
    out = fn()
    return out, L.cfm_launch_count() - before


# ---- CPU: the SDE class ----------------------------------------------------------------------------------------
def test_sde_f_and_g_are_the_notebook_expressions():
    torch.manual_seed(0)
    d, s = cfm_b200.MLP(2, w=32, time_varying=True), cfm_b200.MLP(2, w=32, time_varying=True)
    sde = cfm_b200.SDE(d, s, input_size=(2,), sigma=0.7)
    assert (sde.noise_type, sde.sde_type) == ("diagonal", "ito")
    y, t = torch.randn(9, 2), torch.tensor(0.3)
    x = torch.cat([y, t.repeat(9)[:, None]], 1)
    assert torch.equal(sde.f(t, y), d(x) + s(x))
    tcol = torch.full((9, 1), 0.3)  # t with y's number of dimensions: concatenated as it is
    assert torch.equal(sde.f(tcol, y), d(torch.cat([y, tcol], 1)) + s(torch.cat([y, tcol], 1)))
    assert torch.equal(sde.g(t, y), torch.full_like(y, 0.7))
    sde.f(t, y).sum().backward()  # plain PyTorch: autograd reaches the nets
    assert d.net[0].weight.grad is not None and s.net[0].weight.grad is not None
    assert cfm_b200.SDE(d, s).input_size == (3, 32, 32) and cfm_b200.SDE(d, s).sigma == 1.0


# ---- CPU: refusals that need no device -------------------------------------------------------------------------
def _cpu_sde(dim=2, w=32):
    d, s = cfm_b200.MLP(dim, w=w, time_varying=True), cfm_b200.MLP(dim, w=w, time_varying=True)
    return cfm_b200.SDE(d, s, input_size=(dim,))


@pytest.mark.parametrize("kw,match", [
    ({}, "SRK"), ({"method": "srk"}, "euler"), ({"method": "milstein"}, "euler"),
    ({"method": "euler", "adaptive": True}, "fixed steps"), ({"method": "euler", "logqp": True}, "logqp"),
    ({"solver": "euler"}, "no `solver` argument"), ({"method": "euler", "rtol": 1e-3}, "unsupported"),
])
def test_unsupported_options_raise_not_implemented(kw, match):
    with pytest.raises(NotImplementedError, match=match):
        cfm_b200.sdeint(_cpu_sde(), torch.zeros(4, 2), torch.linspace(0, 1, 3), **kw)


def test_wrong_objects_raise_type_error():
    y, ts = torch.zeros(4, 2), torch.linspace(0, 1, 3)
    with pytest.raises(TypeError, match="cfm_b200.SDE"):
        cfm_b200.sdeint(cfm_b200.MLP(2, w=32, time_varying=True), y, ts, method="euler")
    m = cfm_b200.MLP(2, w=32, time_varying=True)
    bad = [
        cfm_b200.SDE(torch.nn.Linear(3, 2), m, input_size=(2,)),
        cfm_b200.SDE(m, cfm_b200.MLP(2, w=32, time_varying=False), input_size=(2,)),
        cfm_b200.SDE(m, cfm_b200.MLP(2, w=64, time_varying=True), input_size=(2,)),
        cfm_b200.SDE(m, cfm_b200.MLP(3, w=32, time_varying=True), input_size=(2,)),
        cfm_b200.SDE(m, cfm_b200.MLP(2, out_dim=3, w=32, time_varying=True), input_size=(2,)),
        cfm_b200.SDE(m, m, input_size=(3,)),
    ]
    silu = cfm_b200.MLP(2, w=32, time_varying=True)
    silu.act = _ffi.ACT_SILU
    bad.append(cfm_b200.SDE(m, silu, input_size=(2,)))
    for sde in bad:
        with pytest.raises(TypeError):
            cfm_b200.sdeint(sde, y, ts, method="euler")


def test_cpu_y0_raises_library_error():
    with pytest.raises(_ffi.CfmLibraryError, match="CUDA"):
        cfm_b200.sdeint(_cpu_sde(), torch.zeros(4, 2), torch.linspace(0, 1, 3), method="euler")


# ---- CPU: the oracle's grid and interpolation; the package's host tables -----------------------------------------
def test_oracle_grid_accumulates_in_fp32():
    ts = torch.tensor([0.0, 0.0025])
    grid, bracket = osde.step_grid(ts, 1e-3)
    f = np.float32
    want = [f(0), f(0) + f(1e-3), f(0) + f(1e-3) + f(1e-3), f(0.0025)]
    assert [g.item() for g in grid] == [float(v) for v in want]
    assert all(g.dtype == torch.float32 for g in grid) and bracket == [2]
    assert float(want[2]) != 0.002  # fp32 arithmetic, not the decimal value


def test_oracle_interpolation_is_exact_at_grid_points():
    g = torch.Generator().manual_seed(0)
    y0, y1 = torch.randn(5, 3, generator=g, dtype=torch.float64), torch.randn(5, 3, generator=g, dtype=torch.float64)
    t0, t1 = torch.tensor(0.1), torch.tensor(0.1) + 1e-3
    assert torch.equal(osde.linear_interp(t0, y0, t1, y1, t1), y1)
    mid = osde.linear_interp(0.0, y0, 1.0, y1, 0.25)
    assert torch.allclose(mid, 0.75 * y0 + 0.25 * y1, rtol=0, atol=1e-15)


@pytest.mark.parametrize("ts,dt", [
    (torch.tensor([0.0, 0.0025]), 1e-3),
    (torch.linspace(0, 1, 100), 1e-3),
    (torch.tensor([0.0, 0.0137, 0.05, 0.0501, 0.2]), 7e-3),
    (torch.linspace(0, 3, 4), 1.0),
    (torch.linspace(1, 4, 300, dtype=torch.float64), 1e-2),
    (torch.tensor([-1.0, -0.5, 2.0]), 0.3),
])
def test_host_tables_follow_the_oracle_grid(ts, dt):
    grid, out_begin, a, b = csde.step_schedule(ts, dt)
    ogrid, bracket = osde.step_grid(ts, dt)
    assert grid.dtype == ts.numpy().dtype
    assert np.array_equal(grid, np.array([g.item() for g in ogrid], dtype=grid.dtype))
    n_steps = len(grid) - 1
    assert out_begin.shape == (n_steps + 1,) and out_begin[-1] == len(ts) and out_begin[0] >= 1
    owner = np.repeat(np.arange(n_steps), np.diff(out_begin))
    assert np.array_equal(owner, np.array(bracket))
    for k in range(1, len(ts)):
        t0, t1, t = (float(ogrid[bracket[k - 1]]), float(ogrid[bracket[k - 1] + 1]), float(ts[k]))
        assert a[k] == np.float32((t1 - t) / (t1 - t0)) and b[k] == np.float32((t - t0) / (t1 - t0))
        if t == t1:
            assert (a[k], b[k]) == (0.0, 1.0)


# ---- CPU: the generator --------------------------------------------------------------------------------------------
def test_numpy_philox_matches_random123_known_answers():
    kat = [
        ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
        ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
        ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
         [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
    ]
    for ctr, key, want in kat:
        assert osde.philox4x32_10(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32)).tolist() == want


def test_device_normals_restatement_is_standard_normal():
    z = osde.device_normals(12345, 3, np.arange(20000), 8)
    assert z.shape == (20000, 8) and np.isfinite(z).all()
    assert abs(z.mean()) < 5 / np.sqrt(z.size) and abs(z.var() - 1) < 5 * np.sqrt(2 / z.size)


def test_compiled_sde_small_instantiations_are_the_tested_ones(lib_built):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    found = {(int(u), int(t)) for u, t in re.findall(r"sde_small_kernelILi(\d)ELi(\d+)EE", out)}
    assert found == set(SDE_KERNELS)


def test_sde_entry_point_checks_its_arguments_before_any_cuda_call(lib_built):
    import ctypes
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    arr = ctypes.c_void_p * 8
    rc = lib.cfm_sde_small_euler_f32(arr(*([p] * 7 + [None])), arr(*([p] * 8)), 2, 64, 0, 1.0, p, 4, p, 3, p, p, p,
                                     3, 7, None, p, None)
    assert rc == -1 and b"null weight pointer" in lib.cfm_last_error()


# ---- GPU: parity with supplied increments ------------------------------------------------------------------------
_TS = {"offgrid": (torch.tensor([0.0, 0.0137, 0.05, 0.0501, 0.2, 0.31]), 7e-3),
       "sf2m": (torch.linspace(0, 1, 100), 1e-3)}


@gpu
@pytest.mark.parametrize("kind", ["offgrid", "sf2m"])
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", [1, 2, 5, 40])
@pytest.mark.parametrize("w", [32, 64])
def test_parity_with_supplied_increments(w, dim, act, kind, record_property):
    sde, f64 = _sde(dim, w, seed=10 * dim + w, act=act, sigma=0.8)
    ts, dt = _TS[kind]
    B = 1024 if kind == "sf2m" else 333
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(dim))
    bm = FixedBM(B, dim, seed=w + dim)
    tsd = ts.to(DEV) if kind == "offgrid" else ts  # the single-cell notebook passes a device ts
    ys = cfm_b200.sdeint(sde, y0.to(DEV), tsd, bm=bm, method="euler", dt=dt)
    assert ys.shape == (len(ts), B, dim) and ys.dtype == torch.float32 and ys.device.type == "cuda"
    ref = osde.euler_sdeint(f64, 0.8, y0, ts, dt, torch.stack(bm.incs))
    err = (ys.cpu().double() - ref).abs().max().item()
    gate = 1e-4 * max(1.0, ref.abs().max().item())
    record_property("err_over_gate", err / gate)
    assert err <= gate, (err, gate)
    assert torch.equal(ys[0].cpu(), y0)


# ---- GPU: bit identity with the ODE kernel; sigma = 0 ------------------------------------------------------------
@gpu
@pytest.mark.parametrize("w,dim,act", [(32, 2, "selu"), (64, 5, "silu")])
def test_zero_score_and_zero_noise_equal_the_ode_euler_kernel_bit_for_bit(w, dim, act):
    sde, _ = _sde(dim, w, seed=70 + w, act=act, zero_score=True)
    grid, *_ = csde.step_schedule(torch.linspace(0, 1, 11), 1e-2)
    ts = torch.from_numpy(grid)
    B = 777
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(71)).to(DEV)
    ys = cfm_b200.sdeint(sde, y0, ts, bm=FixedBM(B, dim, 0, zero=True), method="euler", dt=1e-2)
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(sde.drift), solver="euler")
    ode = node.trajectory(y0, ts)
    assert node.stats["fused"] and ys.shape == ode.shape
    assert torch.equal(ys, ode)
    sde.sigma = 0.0
    assert torch.equal(cfm_b200.sdeint(sde, y0, ts, method="euler", dt=1e-2), ys)


@gpu
def test_sigma_zero_device_noise_equals_the_zero_increment_run():
    sde, _ = _sde(3, 64, seed=80, sigma=0.0)
    y0 = torch.randn(500, 3, generator=torch.Generator().manual_seed(81)).to(DEV)
    ts = torch.tensor([0.0, 0.033, 0.5, 1.0])
    a = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=0.01)
    b = cfm_b200.sdeint(sde, y0, ts, bm=FixedBM(500, 3, 0, zero=True), method="euler", dt=0.01)
    assert torch.equal(a, b)


# ---- GPU: seeding and row independence ---------------------------------------------------------------------------
@gpu
def test_manual_seed_reproduces_and_another_seed_differs():
    sde, _ = _sde(2, 64, seed=90)
    y0 = torch.randn(1024, 2, generator=torch.Generator().manual_seed(91)).to(DEV)
    ts = torch.linspace(0, 1, 100)
    runs = []
    for s in (5, 5, 6):
        torch.manual_seed(s)
        runs.append(cfm_b200.sdeint(sde, y0, ts, method="euler"))
    assert torch.equal(runs[0], runs[1])
    assert not torch.equal(runs[0][1:], runs[2][1:]) and torch.equal(runs[0][0], runs[2][0])


def _profiled(fn, tmp_path):
    """(fn(), [(U, MAXT, grid, block)] of every sde_small_kernel it ran), from a torch.profiler trace."""
    import json

    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    path = tmp_path / f"trace{len(list(tmp_path.iterdir()))}.json"
    prof.export_chrome_trace(str(path))
    ran = []
    for e in json.loads(path.read_text())["traceEvents"]:
        m = _KERNEL_RE.search(e.get("name", "")) if e.get("cat") == "kernel" else None
        if m:
            ran.append((int(m.group(1)), int(m.group(2)), e["args"]["grid"][0], e["args"]["block"][0]))
    return out, ran


@gpu
@pytest.mark.parametrize("u,maxt", SDE_KERNELS)
def test_rows_are_independent_of_the_launch_shape(u, maxt, tmp_path):
    """Each instantiation runs once (the profiler names it); the first rows of that batch equal a small run with the
    same seed, which the planner launches with 4 warps per CTA, and the float64 oracle on the device's own noise."""
    w, dim, sms = 32 * u, 3, _sms()
    # 256 threads: 8 warps per CTA, one row group each; 512 threads: 16 warps with three row groups each
    B = 12 * sms + 1 if maxt == 256 else 80 * sms + 3
    sde, f64 = _sde(dim, w, seed=100 + u, act="silu" if u == 2 else "selu")
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(101)).to(DEV)
    ts = torch.tensor([0.0, 0.1, 0.25])
    torch.manual_seed(7)
    big, ran = _profiled(lambda: cfm_b200.sdeint(sde, y0, ts, method="euler", dt=0.02), tmp_path)
    assert len(ran) == 1 and ran[0][:2] == (u, maxt), ran
    for k in (1, 7, 333):
        torch.manual_seed(7)
        small, n = _launches(lambda: cfm_b200.sdeint(sde, y0[:k], ts, method="euler", dt=0.02))
        assert n == 1 and torch.equal(small, big[:, :k])
    torch.manual_seed(7)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    rows = np.concatenate([np.arange(5), np.arange(B - 5, B)])
    grid, _ = osde.step_grid(ts, 0.02)
    incs = torch.stack([torch.from_numpy(osde.device_normals(seed, n, rows, dim)) * float(grid[n + 1] - grid[n]) ** 0.5
                        for n in range(len(grid) - 1)])
    ref = osde.euler_sdeint(f64, 1.0, y0[rows].cpu(), ts, 0.02, incs)
    assert (big[:, rows].cpu().double() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())


# ---- GPU: the generator's mapping and statistics -----------------------------------------------------------------
@gpu
def test_device_increments_follow_the_philox_box_muller_mapping():
    dim, B = 6, 333
    sde, _ = _sde(dim, 32, seed=110, zero_score=True, zero_drift=True)
    ts = torch.arange(0, 5, dtype=torch.float32)
    torch.manual_seed(11)
    ys = cfm_b200.sdeint(sde, torch.zeros(B, dim, device=DEV), ts, method="euler", dt=1.0)
    torch.manual_seed(11)
    seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
    dz = (ys[1:] - ys[:-1]).cpu().double().numpy()
    for n in range(4):
        z = osde.device_normals(seed, n, np.arange(B), dim)
        assert (np.abs(dz[n] - z) <= 1e-5 * np.maximum(1.0, np.abs(z))).all(), n


@gpu
def test_device_increments_have_brownian_statistics():
    from scipy import stats
    sigma, B = 0.7, 1 << 16
    sde, _ = _sde(2, 64, seed=120, sigma=sigma, zero_score=True, zero_drift=True)
    ts = torch.linspace(0, 1, 11)
    y0 = torch.randn(B, 2, generator=torch.Generator().manual_seed(121)).to(DEV)
    torch.manual_seed(12)
    ys = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=1e-2).cpu().double()
    d = ys - ys[0]
    N = d[0].numel()
    for k in range(1, 11):
        t = float(ts[k])
        x = d[k].flatten()
        assert abs(x.mean().item()) <= 5 * sigma * t ** 0.5 / N ** 0.5, k
        var = sigma ** 2 * t
        assert abs(x.var().item() - var) <= 5 * var * (2 / N) ** 0.5, k
    assert stats.kstest(d[10].flatten().numpy() / sigma, "norm").pvalue > 1e-3  # against N(0, sigma^2)
    a, b = (ys[5] - ys[0])[:, 0], (ys[10] - ys[5])[:, 0]
    assert abs(np.corrcoef(a.numpy(), b.numpy())[0, 1]) <= 5 / B ** 0.5
    assert abs(np.corrcoef(d[10][:, 0].numpy(), d[10][:, 1].numpy())[0, 1]) <= 5 / B ** 0.5


# ---- GPU: refusals launch nothing ----------------------------------------------------------------------------------
@gpu
def test_refusals_launch_nothing():
    sde, _ = _sde(2, 64, seed=130)
    y0, ts = torch.zeros(64, 2, device=DEV), torch.linspace(0, 1, 5)
    w128 = cfm_b200.SDE(cfm_b200.MLP(2, w=128, time_varying=True).to(DEV),
                        cfm_b200.MLP(2, w=128, time_varying=True).to(DEV), input_size=(2,))
    wide = cfm_b200.SDE(cfm_b200.MLP(400, w=64, time_varying=True).to(DEV),
                        cfm_b200.MLP(400, w=64, time_varying=True).to(DEV), input_size=(400,))
    cases = [
        (NotImplementedError, lambda: cfm_b200.sdeint(sde, y0, ts)),
        (NotImplementedError, lambda: cfm_b200.sdeint(sde, y0, ts, method="euler", adaptive=True)),
        (TypeError, lambda: cfm_b200.sdeint(sde.drift, y0, ts, method="euler")),
        (ValueError, lambda: cfm_b200.sdeint(sde, y0[None], ts, method="euler")),
        (ValueError, lambda: cfm_b200.sdeint(sde, y0, ts[None], method="euler")),
        (ValueError, lambda: cfm_b200.sdeint(sde, y0, ts.flip(0), method="euler")),
        (ValueError, lambda: cfm_b200.sdeint(sde, y0, torch.tensor([0.0, 0.5, 0.5]), method="euler")),
        (ValueError, lambda: cfm_b200.sdeint(sde, y0, ts, method="euler", dt=0.0)),
        (ValueError, lambda: cfm_b200.sdeint(sde, torch.zeros(64, 3, device=DEV), ts, method="euler")),
        (NotImplementedError, lambda: cfm_b200.sdeint(w128, y0, ts, method="euler")),
        (NotImplementedError, lambda: cfm_b200.sdeint(wide, torch.zeros(8, 400, device=DEV), ts, method="euler")),
    ]
    L = _ffi.lib()
    assert not L.cfm_sde_small_supported(64, 2, 128) and not L.cfm_sde_small_supported(8, 400, 64)
    assert L.cfm_sde_small_supported(1024, 2, 64) and L.cfm_sde_small_supported(1024, 2, 32)
    for exc, fn in cases:
        before = L.cfm_launch_count()
        with pytest.raises(exc):
            fn()
        assert L.cfm_launch_count() == before
    with pytest.raises(NotImplementedError, match=r"w in \{32, 64\}"):
        cfm_b200.sdeint(w128, y0, ts, method="euler")
