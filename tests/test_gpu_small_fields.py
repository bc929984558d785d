"""Every shape class of the small-field ODE kernel (csrc/ode_small.cu) and of the per-layer tensor-core MLP
(csrc/mlp_h3.cu part (2)) against float64 references.

* Exact-likelihood (CNF) variant: one Euler evaluation at every w in {32, 64, 128} x dim in 1..8 against the
  float64 jacrev trace (tests/cnf_oracle.py); dopri5 step for step; the largest batch the planner accepts for every
  (w, dim), where it runs one warp per CTA with many row groups each; the planner's fewer-warps fallback.
* Plain variant: one test per compiled ode_small_kernel<U, MAXT, false>, with the profiler naming the kernel that
  ran.  A CPU test reads the instantiations out of the built library, so a new one without a test fails there.
* MLP: the per-layer fp16x3 tensor-core path (and the SIMT path) at hidden widths that are not multiples of 32, one
  partial K-chunk, and w = 512; the multi-kernel dopri5 driver on it.

Batch sizes follow from the device's SM count or from the library's own plan queries, so the cases keep their meaning
on a part with a different SM count."""
import itertools
import json
import re
import subprocess

import pytest
import torch

import cnf_oracle as co
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

DEV = "cuda:0"
gpu = pytest.mark.gpu

# ode_small_kernel<U, MAXT, false> instantiations (U = w / 32, MAXT = threads per CTA).  w = 128 has no 1024-thread
# kernel: 32 warps of hidden buffers next to W1 and W2 never fit the planner's shared-memory budget.
PLAIN_KERNELS = [(1, 256), (2, 256), (4, 256), (1, 512), (2, 512), (4, 512), (1, 1024), (2, 1024)]
CNF_KERNELS = [(1, 256), (2, 256), (4, 256)]
_KERNEL_RE = re.compile(r"ode_small_kernel<(\d), (\d+), (true|false)>")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pair(dim, w, seed, act="selu", out_dim=None):
    """(device MLP, float64 CPU oracle MLP) with the same weights."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    mc = vf.make_mlp(dim, out_dim=out_dim, w=w, time_varying=True, dtype=torch.float64)
    mc.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            mc.net[k] = torch.nn.SiLU()
    return m.to(DEV), mc


def _state(x):
    return torch.cat([x, torch.zeros(x.shape[0], 1, dtype=x.dtype)], 1)


def _profiled(fn, tmp_path):
    """(fn(), [(U, MAXT, cnf, grid, block)] of every ode_small_kernel it ran), read from a torch.profiler trace."""
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
            ran.append((int(m.group(1)), int(m.group(2)), m.group(3) == "true", e["args"]["grid"][0],
                        e["args"]["block"][0]))
    return out, ran


def _launches(fn):
    L = _ffi.lib()
    before = L.cfm_launch_count()
    out = fn()
    return out, L.cfm_launch_count() - before


# SELU's derivative jumps from 1.76 to 1.05 at 0, so the exact trace is discontinuous wherever a hidden pre-activation
# is 0.  An fp32 pre-activation sum_i W_ui h_i + b_u of n <= 129 terms carries a rounding error of up to
# n * 2^-24 * (sum_i |W_ui h_i| + |b_u|), below 7.7e-6 of that magnitude sum, so closer than 1e-5 of it to 0 the sign,
# and with it act', is not fixed by the arithmetic.  The trace column is gated on the rows that stay further away.
_KINK_REL = 1e-5


def smooth_rows(mc, seen, act):
    """Rows whose float64 evaluation points ``seen`` ((t, [x, ll]) pairs, as cnf_oracle.recording keeps them) all keep
    every hidden pre-activation further than _KINK_REL of its magnitude sum from SELU's kink; every row for SiLU."""
    B = seen[0][1].shape[0]
    keep = torch.ones(B, dtype=torch.bool)
    if act != "selu":
        return keep
    with torch.no_grad():
        for t, z in seen:
            h = torch.cat([z[:, :-1], t.reshape(()).repeat(B)[:, None]], 1).double()
            for li in (0, 2, 4):
                W, b = mc.net[li].weight.double(), mc.net[li].bias.double()
                p = h @ W.T + b
                keep &= (p.abs() > _KINK_REL * (h.abs() @ W.abs().T + b.abs())).all(1)
                h = torch.nn.functional.selu(p)
    return keep


def assert_cnf_close(got, ref, keep, rel):
    """x columns of every row, the log-density column of the ``keep`` rows: within rel * max(1, |ref|)."""
    assert int(keep.sum()) >= keep.numel() // 2, int(keep.sum())
    gate = rel * max(1.0, ref.abs().max().item())
    ex = (got[..., :-1] - ref[..., :-1]).abs().max().item()
    el = (got[:, keep, -1] - ref[:, keep, -1]).abs().max().item()
    assert ex <= gate and el <= gate, (ex, el, gate)


def _cnf_bmax(dim, w):
    """Largest batch cfm_ode_small_cnf_supported accepts (bisection keeps lo accepted, hi refused)."""
    L = _ffi.lib()
    lo, hi = 1, 1 << 24
    assert L.cfm_ode_small_cnf_supported(lo, dim, w) and not L.cfm_ode_small_cnf_supported(hi, dim, w)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        if L.cfm_ode_small_cnf_supported(mid, dim, w):
            lo = mid
        else:
            hi = mid
    return lo


# ---- exact-likelihood variant: one evaluation at every width, dimension and activation -------------------------
@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", range(1, 9))
@pytest.mark.parametrize("w", [32, 64, 128])
def test_cnf_one_euler_step_gives_the_field_and_the_float64_trace(w, dim, act, record_property):
    m, mc = _pair(dim, w, seed=10 * dim + w // 32, act=act)
    # odd, so the last row pair is partial; at 8 warps per CTA every warp holds four row groups
    B = 48 * _sms() + 1
    span = torch.tensor([0.5, 1.5])  # h = 1 exactly: traj[1] = x + f(0.5, x) and, from ll = 0, traj[1, :, dim] = div
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="euler")
    plain = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="euler")
    field = co.cnf_field(mc)
    g = torch.Generator().manual_seed(1000 * w + dim)
    worst = 0.0
    # randn * 30 drives SELU deep into its exponential branch and SiLU into saturation, where act_deriv_fast's ex2f
    # over- or underflows
    for scale in (1.0, 30.0):
        x = scale * torch.randn(B, dim, generator=g)
        traj = node.trajectory(_state(x).to(DEV), span)
        assert node.stats["fused"] and traj.shape == (2, B, dim + 1)
        assert torch.equal(node.trajectory(_state(x[:1]).to(DEV), span), traj[:, :1])  # B = 1: padding partner
        t64, z64 = torch.tensor(0.5, dtype=torch.float64), _state(x).double()
        ref = field(t64, z64)
        keep = smooth_rows(mc, [(t64, z64)], act)
        assert int(keep.sum()) >= B // 2
        div, div64 = traj[1, :, dim].cpu().double()[keep], ref[keep, dim]
        gate = 1e-5 * max(1.0, div64.abs().max().item())
        err = (div - div64).abs().max().item()
        worst = max(worst, err / gate)
        assert err <= gate, (scale, err, gate)
        xf, xf64 = traj[1, :, :dim].cpu().double(), x.double() + ref[:, :dim]
        assert (xf - xf64).abs().max() <= 1e-5 * max(1.0, xf64.abs().max().item())
        # the x columns run the plain variant's instructions: bit-identical to it on the same rows (Euler rows are
        # independent, so where the plain kernel does not plan the whole batch a prefix stands for it)
        n = B if _ffi.lib().cfm_ode_small_supported(B, dim, w, dim) else 333
        px = plain.trajectory(x[:n].to(DEV), span)
        assert plain.stats["fused"]
        assert torch.equal(traj[:, :n, :dim], px)
    record_property("worst_div_error_over_gate", worst)


@gpu
def test_cnf_w128_plans_dims_7_and_8():
    L = _ffi.lib()
    for dim in (7, 8):
        assert L.cfm_ode_small_cnf_supported(1, dim, 128) == 1
        assert L.cfm_ode_small_cnf_supported(48 * _sms() + 1, dim, 128) == 1


# ---- exact-likelihood variant: dopri5 step for step ------------------------------------------------------------
_DOPRI5_CASES = [(w, dim, span, "silu" if (i + i // 2) % 2 else "selu")
                 for i, (w, dim, span) in enumerate(itertools.product((32, 128), (1, 5, 8), ((0.0, 1.0), (1.0, 0.0))))]


@gpu
@pytest.mark.parametrize("w,dim,span,act", _DOPRI5_CASES)
def test_cnf_dopri5_matches_the_float64_oracle_step_for_step(w, dim, span, act):
    m, mc = _pair(dim, w, seed=200 + 10 * dim + w // 32, act=act)
    z = _state(torch.randn(333, dim, generator=torch.Generator().manual_seed(300 + dim)))
    ts = torch.tensor(span)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    traj = node.trajectory(z.to(DEV), ts)
    seen = []
    ref, st = co.dopri5_any_direction(co.recording(co.cnf_field(mc), seen), z.double(), ts.double(), 1e-4, 1e-4)
    assert node.stats["fused"]
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert node.stats["t"] == pytest.approx(span[-1], abs=1e-6)
    assert traj.shape == ref.shape
    assert_cnf_close(traj.cpu().double(), ref, smooth_rows(mc, seen, act), 1e-4)


# ---- exact-likelihood variant: the planner's edges -------------------------------------------------------------
def _check_cnf_euler_batch(w, dim, B, act, seed, tmp_path=None):
    """Euler over 3 points at batch B: one launch, sampled rows and the last 7 against the float64 oracle, the first
    333 rows alone bit-identical.  With ``tmp_path``, returns the threads per CTA the profiler saw."""
    m, mc = _pair(dim, w, seed=seed, act=act)
    g = torch.Generator().manual_seed(seed)
    z = _state(torch.randn(B, dim, generator=g))
    span = torch.linspace(1, 0, 3)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="euler")
    zd = z.to(DEV)
    block = None
    if tmp_path is None:
        traj, n = _launches(lambda: node.trajectory(zd, span))
        assert n == 1
    else:
        traj, ran = _profiled(lambda: node.trajectory(zd, span), tmp_path)
        assert len(ran) == 1 and ran[0][:3] == (w // 32, 256, True), ran
        grid, block = ran[0][3:]
        assert grid <= _sms() and block % 32 == 0 and block <= 256, ran
    assert node.stats["fused"] and traj.shape == (3, B, dim + 1)
    rows = torch.cat([torch.randperm(B, generator=g)[:512], torch.arange(max(0, B - 7), B)])
    seen = []
    ref = co.euler_any_direction(co.recording(co.cnf_field(mc), seen), z[rows].double(), span.double())
    assert_cnf_close(traj[:, rows.to(DEV)].cpu().double(), ref, smooth_rows(mc, seen, act), 2e-5)
    assert torch.equal(node.trajectory(zd[:333], span), traj[:, :333])
    return block


@gpu
@pytest.mark.parametrize("dim", range(1, 9))
@pytest.mark.parametrize("w", [32, 64, 128])
def test_cnf_largest_planned_batch_and_the_first_refused_one(w, dim, record_property):
    B = _cnf_bmax(dim, w)
    _check_cnf_euler_batch(w, dim, B, "silu" if dim % 2 else "selu", 400 + 10 * dim + w // 32)
    record_property("bmax", B)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True).to(DEV)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="euler")
    z = torch.zeros(B + 1, dim + 1, device=DEV)
    L = _ffi.lib()
    before = L.cfm_launch_count()
    with pytest.raises(NotImplementedError, match="no exact-likelihood kernel"):
        node.trajectory(z, torch.linspace(1, 0, 3))
    assert L.cfm_launch_count() == before


@gpu
@pytest.mark.parametrize("which", ["above_4_warps", "half_of_bmax"])
def test_cnf_fewer_warps_fallback(which, tmp_path, record_property):
    """w = 128, dim = 3: 8 warps of tangent buffers do not fit next to the weights, so the planner runs fewer warps
    per CTA with more row groups each."""
    B = 24 * _sms() + 1 if which == "above_4_warps" else _cnf_bmax(3, 128) // 2 | 1
    block = _check_cnf_euler_batch(128, 3, B, "selu" if which == "above_4_warps" else "silu", 500, tmp_path)
    record_property("threads_per_cta", block)
    assert block < 256


# ---- plain variant: one test per compiled instantiation --------------------------------------------------------
def _plain_batch(maxt, sms):
    return {256: 8 * sms - 3, 512: 24 * sms + 1, 1024: 48 * sms + 1}[maxt]


def _plain_warps(B, sms):
    """Warps per CTA the plain planner picks when one row group per warp fits: the fewest of 4, 8, 16, 32."""
    groups = (B + 1) // 2
    return next(n for n in (4, 8, 16, 32) if groups <= n * sms)


@gpu
@pytest.mark.parametrize("u,maxt", PLAIN_KERNELS)
def test_plain_instantiation_vs_float64_oracle(u, maxt, tmp_path):
    w, dim, sms = 32 * u, {1: 5, 2: 3, 4: 8}[u], _sms()
    B = _plain_batch(maxt, sms)
    m, mc = _pair(dim, w, seed=600 + maxt + u, act="silu" if PLAIN_KERNELS.index((u, maxt)) % 2 else "selu")
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(700 + u))
    xd = x.to(DEV)
    span = torch.linspace(0, 1, 4)
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    traj, ran = _profiled(lambda: node.trajectory(xd, span), tmp_path)
    assert ran == [(u, maxt, False, ran[0][3], 32 * _plain_warps(B, sms))], ran
    f = lambda t, z: vf.wrapped_forward(mc, t, z)  # noqa: E731
    ref, st = vf.dopri5_trajectory(f, x.double(), span.double(), 1e-4, 1e-4)
    assert node.stats["fused"] and traj.shape == ref.shape
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert (traj.cpu().double() - ref).abs().max() <= 5e-5 * max(1.0, ref.abs().max().item())
    assert torch.equal(node.trajectory(xd, span), traj)
    ne = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="euler")
    te = ne.trajectory(xd, torch.linspace(0, 1, 9))
    re_ = vf.euler_trajectory(f, x.double(), torch.linspace(0, 1, 9, dtype=torch.float64))
    assert ne.stats["fused"] and (te.cpu().double() - re_).abs().max() <= 2e-5 * max(1.0, re_.abs().max().item())
    assert torch.equal(ne.trajectory(xd, torch.linspace(0, 1, 9)), te)


def test_compiled_ode_small_instantiations_are_the_tested_ones(lib_built):
    """Reads the kernels out of the library's cubin; no device needed."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    found = {(int(u), int(t), c == "1") for u, t, c in re.findall(r"ode_small_kernelILi(\d)ELi(\d+)ELb([01])E", out)}
    assert found == {(u, t, False) for u, t in PLAIN_KERNELS} | {(u, t, True) for u, t in CNF_KERNELS}


# ---- per-layer tensor-core MLP and the SIMT path ---------------------------------------------------------------
# (B, dim, w, out_dim): K = 32 (one partial K-chunk), hidden widths that are not multiples of 32 (the scalar epilogue
# applies layer 0's time column), w = 256 with dim < 64 (per-layer, not the fused kernel), and w = 512
_TC_SHAPES = [(128, 32, 32, 32), (129, 40, 40, 8), (1000, 56, 72, 12), (777, 64, 128, 68), (4097, 32, 200, 36),
              (300, 48, 256, 48), (2000, 784, 512, 784)]
_SIMT_ONLY_SHAPES = [(7, 3, 50, 3), (300, 7, 36, 5)]  # w % 4 != 0: the tensor-core path does not take these
_MLP_CASES = [s + (algo,) for s in _TC_SHAPES for algo in (0, 1)] + [s + (1,) for s in _SIMT_ONLY_SHAPES]


def _mlp64(mc, state, x, t, act):
    inp = torch.cat([x.double(), torch.full((x.shape[0], 1), t, dtype=torch.float64)], 1)
    if act == "selu":
        return vf.mlp_forward_from_state(state, inp)
    with torch.no_grad():
        return mc(inp)


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("B,dim,w,out_dim,algo", _MLP_CASES)
def test_mlp_vector_field_per_layer_vs_float64(B, dim, w, out_dim, algo, act):
    m, mc = _pair(dim, w, seed=800 + w, act=act, out_dim=out_dim)
    state = {k: v.double().cpu() for k, v in m.state_dict().items()}
    m.mlp_algo = algo
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(900 + dim))
    xd, t = x.to(DEV), 0.37
    with torch.no_grad():
        m.vector_field(t, xd)  # builds the prepared weights
        y, n = _launches(lambda: m.vector_field(t, xd))
        y_dev = m.vector_field(torch.tensor(t, device=DEV), xd)
    if algo == 0:
        assert m.tc_path(B) and n == 5  # the input split and one GEMM per layer: not the fused kernel
    else:
        assert not m.tc_path(B) and n == 4
    assert torch.equal(y_dev, y)
    ref = _mlp64(mc, state, x, t, act)
    assert y.shape == (B, out_dim)
    assert (y.cpu().double() - ref).abs().max() <= 1e-5 * ref.abs().max().item()


@gpu
def test_multi_kernel_dopri5_on_the_per_layer_tensor_core_mlp():
    m, mc = _pair(64, 128, seed=31)
    B = 1500
    assert not _ffi.lib().cfm_ode_small_supported(B, 64, 128, 64) and m.tc_path(B)
    x = torch.randn(B, 64, generator=torch.Generator().manual_seed(32))
    span = torch.linspace(0, 1, 4)
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    traj = node.trajectory(x.to(DEV), span)
    assert not node.stats.get("fused") and node.stats["graph"]
    ref, st = vf.dopri5_trajectory(lambda t, z: vf.wrapped_forward(mc, t, z), x.double(), span.double(), 1e-4, 1e-4)
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert (traj.cpu().double() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())
    eager = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    eager.use_cuda_graph = False
    assert torch.equal(eager.trajectory(x.to(DEV), span), traj) and not eager.stats["graph"]
