"""The one-launch SDE kernel (sde_small_kernel<U, MAXT>) and gradient-field kernel (ode_grad_kernel<U, 256>) of
csrc/ode_small.cu entry by entry and at every planner edge, against float64 under the per-entry gates of
tests/small_field_oracle.py, on the cases of tests/small_field_cases.py.

* One-step fields: the gradient field's Euler step over (t, t + 1) at every w, dim 1..8, SELU and SiLU, plain and x30
  inputs; each SDE net alone (the other's output layer zeroed, sigma = 0, one step of dt = 1) at dims on both layer-3
  branches and the largest planned dim.
* Gradient-field dopri5 step for step at a tolerance where steps are rejected, both span directions; one plan from the
  planner's fewer-warps fallback, the profiler naming its block size.
* Planner edges: the restated planners against cfm_*_supported; the largest planned batch and dim, their edge rows
  under the per-entry gate; the next batch refused with no launch, or run by the tensor-core class on the same noise.
* The SDE's own noise on a non-uniform step grid, entry by entry (small_field_oracle.Bounded).
* Buffers: nothing written past [n_out][B][dim]; the gradient field's dopri5 gives the same bits from a NaN-filled
  workspace and on a second call."""
import ctypes as C
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cnf_oracle as co
import cnf_tc_oracle as ho
import small_field_cases as sc
import small_field_oracle as so
import tc_sampler_cases as tc
from oracle import sde as osde
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi
from cfm_b200 import sde as csde

DEV = "cuda:0"
TESTS = os.path.dirname(os.path.abspath(__file__))
gpu = pytest.mark.gpu
_KINK_REL = 1e-5  # tests/test_gpu_action.py's SELU kink filter


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launches(fn):
    L = _ffi.lib()
    before = L.cfm_launch_count()
    out = fn()
    return out, L.cfm_launch_count() - before


def _mlp(dim, w, seed, act, out_dim=None, shrink=None):
    """A device MLP with torch's default initialisation (hidden weights times ``shrink``) and its CPU state."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    with torch.no_grad():
        for li in ((2, 4, 6) if shrink else ()):
            m.net[li].weight.mul_(shrink)
    if act == "silu":
        m.act = _ffi.ACT_SILU
    return m.to(DEV), {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}


def _f64(state, dim, w, act, out_dim=None):
    mc = vf.make_mlp(dim, out_dim=out_dim, w=w, time_varying=True, dtype=torch.float64)
    mc.load_state_dict({k: v.double() for k, v in state.items()})
    if act == "silu":
        for k in (1, 3, 5):
            mc.net[k] = torch.nn.SiLU()
    return mc


def _kink_free(state, points, act):
    """Rows whose float64 evaluation points ((t, x) pairs) keep every hidden pre-activation further than _KINK_REL of
    its magnitude sum from SELU's kink; every row for SiLU."""
    keep = torch.ones(points[0][1].shape[0], dtype=torch.bool)
    if act != "selu":
        return keep
    for t, x in points:
        h = torch.cat([x.double().cpu(), torch.full((x.shape[0], 1), float(t), dtype=torch.float64)], 1)
        for li in (0, 2, 4):
            W, b = state[f"net.{li}.weight"].double(), state[f"net.{li}.bias"].double()
            p = h @ W.T + b
            keep &= (p.abs() > _KINK_REL * (h.abs() @ W.abs().T + b.abs())).all(1)
            h = torch.nn.functional.selu(p)
    return keep


def _grad_node(m, **kw):
    return cfm_b200.NeuralODE(cfm_b200.torch_wrapper(cfm_b200.GradModel(m)), **kw)


def _check_grad_step(state, act, x, traj, t0, rows=None):
    """traj[1] - traj[0] against the float64 field at (t0, x) on ``rows`` (all when None), within the per-entry gate
    plus half an ulp of traj[1]; returns the worst ratio to the gate."""
    rows = torch.arange(x.shape[0]) if rows is None else torch.as_tensor(rows)
    xr = x[rows].cpu()
    t1 = traj[1][rows.to(traj.device)].cpu()
    f, G, gate, kink = so.grad_bounds(state, t0, xr, act)
    assert (f.abs() <= G).all()
    keep = _kink_free(state, [(t0, xr)], act) & ~kink
    assert int(keep.sum()) >= (len(rows) + 1) // 2, (int(keep.sum()), len(rows))
    err = (t1.double() - xr.double() - f).abs()
    bound = gate + so.half_ulp(t1)
    ratio = float((err / bound)[keep].max())
    assert bool((err <= bound)[keep].all()), ratio
    return ratio


# ---- one-step fields -------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", range(1, 9))
@pytest.mark.parametrize("w", [32, 64])
def test_grad_field_one_euler_step_entry_by_entry(w, dim, act, record_property):
    """Euler over (0.25, 1.25): h = 1, so traj[1] - traj[0] is the field to within half an ulp of traj[1].  x30 inputs
    drive SELU deep into its exponential branch and SiLU into saturation."""
    m, state = _mlp(dim, w, seed=1000 + 10 * dim + w, act=act, out_dim=1)
    B = 2 * w + 2 * dim + 1  # odd: the last row's group partner is padding
    g = torch.Generator().manual_seed(dim + w)
    node = _grad_node(m, solver="euler")
    worst = 0.0
    for scale in (1.0, 30.0):
        x = scale * torch.randn(B, dim, generator=g)
        traj, n = _launches(lambda: node.trajectory(x.to(DEV), torch.tensor([0.25, 1.25])))
        assert n == 1 and node.stats["fused"]
        worst = max(worst, _check_grad_step(state, act, x, traj, 0.25))
    print(f"margins grad field w={w} dim={dim} {act}: {worst:.2e} of the gate")
    record_property("err_over_gate", worst)


def _sde_case(dim, w, act, seed, which=None, shrink=None):
    """(SDE, drift state, score state): ``which`` = "drift" / "score" zeroes the other net's output layer."""
    d, ds = _mlp(dim, w, seed, act, shrink=shrink)
    s, ss = _mlp(dim, w, seed + 1, act, shrink=shrink)
    zero = {"drift": s, "score": d}.get(which)
    if zero is not None:
        with torch.no_grad():
            zero.net[6].weight.zero_()
            zero.net[6].bias.zero_()
    return cfm_b200.SDE(d, s, input_size=(dim,), sigma=0.0), ds, ss


@gpu
@pytest.mark.parametrize("d", sc.SDE_FIELD_DIMS)
@pytest.mark.parametrize("w", [32, 64])
def test_sde_nets_one_step_entry_by_entry(w, d, record_property):
    """Each net alone: the other's output layer zeroed (its output is exactly 0), sigma = 0 and one step of h = 1 over
    (0.25, 1.25), so ys[1] - ys[0] is the net's output to within half an ulp of ys[1], against its own scale."""
    dim = sc.resolve_dim(w, d, _sms())
    act = "silu" if sc.SDE_FIELD_DIMS.index(d) % 2 else "selu"
    B = 333
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(dim)).to(DEV)
    ts = torch.tensor([0.25, 1.25])
    worst = 0.0
    for which in ("drift", "score"):
        sde, ds, ss = _sde_case(dim, w, act, seed=2000 + dim + w, which=which)
        ys, n = _launches(lambda: cfm_b200.sdeint(sde, y0, ts, method="euler", dt=1.0))
        assert n == 1 and _ffi.lib().cfm_sde_small_supported(B, dim, w)
        f, F, gate = so.mlp_bounds(ds if which == "drift" else ss, 0.25, y0, act)
        assert (f.abs() <= F).all()
        err = (ys[1].cpu().double() - y0.cpu().double() - f).abs()
        bound = gate + so.half_ulp(ys[1])
        worst = max(worst, float((err / bound).max()))
        assert bool((err <= bound).all()), (which, float((err / bound).max()))
    print(f"margins sde nets w={w} dim={dim} {act}: {worst:.2e} of the gate")
    record_property("err_over_gate", worst)


# ---- gradient-field dopri5 step for step ----------------------------------------------------------------------------
_DOPRI5_TOL = 1e-6  # the SELU fields below reject steps at this tolerance


def _grad_field64(mc):
    def f(t, x):
        with torch.enable_grad():
            y = x.detach().clone().requires_grad_(True)
            s = mc(torch.cat([y, t.reshape(()).repeat(y.shape[0])[:, None].to(y.dtype)], 1))
            return torch.autograd.grad(s.sum(), y)[0]
    return f


def _check_dopri5(m, state, dim, w, x, span, tol, node):
    traj = node.trajectory(x.to(DEV), torch.tensor(span))
    seen, record = [], []
    ref, st = co.dopri5_any_direction(co.recording(_grad_field64(_f64(state, dim, w, "selu", 1)), seen), x.double(),
                                      torch.tensor(span).double(), tol, tol, record=record)
    assert node.stats["fused"]
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert st["rejected"] > 0 and any(not r["accepted"] for r in record)
    # every accept / reject decision is clear of the fp32 arithmetic's reach
    assert min(abs(r["ratio"] - 1) for r in record) > 1e-3
    # hundreds of evaluations bring most rows close to a SELU kink at some point: the rows that never come close
    keep = _kink_free(state, [(t, z) for t, z in seen], "selu")
    assert int(keep.sum()) >= 32, int(keep.sum())
    got = traj.cpu().double()
    assert torch.isfinite(got).all()
    gate = 1e-4 * max(1.0, ref.abs().max().item())
    assert (got[:, keep] - ref[:, keep]).abs().max().item() <= gate
    return traj


@gpu
@pytest.mark.parametrize("w,dim,span", sc.GRAD_DOPRI5)
def test_grad_dopri5_with_rejected_steps_step_for_step(w, dim, span):
    m, state = _mlp(dim, w, seed=50 + 10 * dim + w // 32, act="selu", out_dim=1)
    x = torch.randn(333, dim, generator=torch.Generator().manual_seed(60 + dim)) * 2.0
    node = _grad_node(m, solver="dopri5", atol=_DOPRI5_TOL, rtol=_DOPRI5_TOL)
    _check_dopri5(m, state, dim, w, x, span, _DOPRI5_TOL, node)


_FALLBACK = (64, 5, "fallback:4")  # (w, dim, batch): 8 warps of hidden buffers do not fit, the plan runs 4


def _fallback_case():
    w, dim, name = _FALLBACK
    B = sc.resolve("grad", name, dim, w, _sms())
    m, state = _mlp(dim, w, seed=77, act="selu", out_dim=1)
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(78)) * 2.0
    return m, state, x, _grad_node(m, solver="dopri5", atol=1e-4, rtol=1e-4)


def _trace_fallback(tmp_dir):
    """Run in a child process: one traced dopri5 trajectory of _fallback_case; prints its grad kernels as JSON."""
    import pathlib

    from torch.profiler import ProfilerActivity, profile
    m, _, x, node = _fallback_case()
    xd = x.to(DEV)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        traj = node.trajectory(xd, torch.tensor((0.0, 1.0)))
        torch.cuda.synchronize()
    path = pathlib.Path(tmp_dir) / "trace.json"
    prof.export_chrome_trace(str(path))
    ran = [(e["name"], e["args"]["grid"][0], e["args"]["block"][0]) for e in json.loads(path.read_text())["traceEvents"]
           if e.get("cat") == "kernel" and "ode_grad_kernel" in e.get("name", "")]
    torch.save(traj.cpu(), pathlib.Path(tmp_dir) / "traj.pt")
    print(json.dumps(ran))


@pytest.fixture(scope="module")
def fallback_trace(tmp_path_factory):
    """(kernels, trajectory) of the fallback plan, traced in a child process as tests/test_gpu_sde.py does: once a
    process has taken a trace, kernels go missing from its later traces."""
    tmp = tmp_path_factory.mktemp("grad_trace")
    code = ("import sys; sys.path[:0] = sys.argv[1:3]; import test_gpu_small_field_edges as t; "
            "t._trace_fallback(sys.argv[3])")
    r = subprocess.run([sys.executable, "-c", code, os.path.dirname(TESTS), TESTS, str(tmp)], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1]), torch.load(tmp / "traj.pt")


@gpu
def test_grad_dopri5_on_the_fewer_warps_fallback(fallback_trace):
    """The planner's fallback plan (4 warps per CTA where 8 would not fit), confirmed by the profiler's block size; the
    whole batch step for step against float64 (the controller's error norm spans every row)."""
    w, dim, name = _FALLBACK
    m, state, x, node = _fallback_case()
    plan = sc.plan_grad(x.shape[0], dim, w, _sms())
    assert plan[1] == 4 and plan[2] > sc.RB
    ran, traced = fallback_trace
    assert len(ran) == 1 and "ode_grad_kernel<2, 256>" in ran[0][0] and ran[0][1:] == [plan[0], 32 * plan[1]], ran
    traj = node.trajectory(x.to(DEV), torch.tensor((0.0, 1.0)))
    assert torch.equal(traj.cpu(), traced)
    seen = []
    ref, st = co.dopri5_any_direction(co.recording(_grad_field64(_f64(state, dim, w, "selu", 1)), seen), x.double(),
                                      torch.tensor((0.0, 1.0)).double(), 1e-4, 1e-4)
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    keep = _kink_free(state, seen, "selu")
    gate = 1e-4 * max(1.0, ref.abs().max().item())
    assert (traj.cpu().double()[:, keep] - ref[:, keep]).abs().max().item() <= gate


# ---- planner edges --------------------------------------------------------------------------------------------------
@gpu
def test_restated_planners_are_the_library_predicates():
    L, sms = _ffi.lib(), _sms()
    dims = [1, 2, 5, 8, 9, 33, 64, 100, 113, 114, 115, 284, 285, 286, 1024, 1025]
    batches = {1, 2, 3, 127, 128, 129, 8 * sms - 1, 8 * sms + 1, 16 * sms + 1, 32 * sms + 1, 80 * sms + 3, 1 << 20}
    for w in (32, 64):
        for dim in range(1, 9):
            bmax = sc.grad_bmax(dim, w, sms)
            for B in batches | {bmax, bmax + 1} | {sc.grad_fallback_batch(dim, w, n, sms) or 1 for n in (4, 2, 1)}:
                assert L.cfm_ode_small_grad_supported(B, dim, w) == int(sc.plan_grad(B, dim, w, sms) is not None), \
                    (B, dim, w)
        for dim in dims:
            bmax = sc.sde_bmax(dim, w, sms) if dim <= sc.MAX_DIM and sc.plan_sde(1, dim, w, sms) else 1
            for B in batches | {bmax, bmax + 1}:
                assert L.cfm_sde_small_supported(B, dim, w) == int(sc.plan_sde(B, dim, w, sms) is not None), \
                    (B, dim, w)
    for dim, w in ((2, 128), (2, 96), (9, 64)):
        assert not L.cfm_ode_small_grad_supported(1024, dim, w) and sc.plan_grad(1024, dim, w, sms) is None
    assert not L.cfm_sde_small_supported(1024, 2, 128) and sc.plan_sde(1024, 2, 128, sms) is None


_GRAD_EDGES = [("bmax", w, dim) for w, dim in sc.GRAD_BMAX] + [(B, w, dim) for w, dim, B in sc.GRAD_WARP_SHAPES]


@gpu
@pytest.mark.parametrize("name,w,dim", _GRAD_EDGES)
def test_grad_field_planner_edges(name, w, dim, record_property):
    """One Euler step of h = 1 at the named batch: the plan's edge rows (sc.edge_rows) and 64 sampled rows under the
    per-entry gate; past the largest batch, the next one raises with no launch."""
    sms = _sms()
    B = sc.resolve("grad", name, dim, w, sms)
    plan = sc.plan_grad(B, dim, w, sms)
    act = "silu" if (dim + w // 32) % 2 else "selu"
    m, state = _mlp(dim, w, seed=3000 + 10 * dim + w, act=act, out_dim=1)
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, dim, generator=g)
    node = _grad_node(m, solver="euler")
    traj, n = _launches(lambda: node.trajectory(x.to(DEV), torch.tensor([0.25, 1.25])))
    assert n == 1
    edges = sc.edge_rows(B, plan)
    rows = sorted(set(edges.values()) | set(torch.randint(0, B, (64,), generator=g).tolist()))
    worst = _check_grad_step(state, act, x, traj, 0.25, rows)
    record_property("B", B)
    record_property("plan", plan[:3])
    print(f"margins grad edges {name} B={B} plan={plan[:3]}: {worst:.2e} of the gate")
    if name == "bmax":
        L = _ffi.lib()
        assert sc.plan_grad(B + 1, dim, w, sms) is None
        before = L.cfm_launch_count()
        with pytest.raises(NotImplementedError, match="no gradient-field kernel"):
            node.trajectory(torch.zeros(B + 1, dim, device=DEV), torch.tensor([0.25, 1.25]))
        assert L.cfm_launch_count() == before


# the SDE trajectory cases: a non-uniform step grid, own noise; hidden weights shrunk so that the growth factor
# exp(T Lip) of the trajectory bound stays small
_SDE_TS, _SDE_DT, _SDE_SIGMA = tc.NOISE_TS, tc.NOISE_DT, tc.NOISE_SIGMA


def _own_noise_run(sde, y0, seed_draw):
    torch.manual_seed(seed_draw)
    ys, n = _launches(lambda: cfm_b200.sdeint(sde, y0, torch.tensor(_SDE_TS, dtype=torch.float32), method="euler",
                                                dt=_SDE_DT))
    torch.manual_seed(seed_draw)
    return ys, n, int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))


def _sde_bound(ds, ss, dim, w, act, y0_rows, seed, rows, net_err):
    """(float64 trajectory, per-entry bound) on ``rows`` of the device's own noise."""
    dc, scn = _f64(ds, dim, w, act), _f64(ss, dim, w, act)
    lip = ho.lipschitz(dc, act) + ho.lipschitz(scn, act)
    assert lip < 3, lip
    ts = torch.tensor(_SDE_TS, dtype=torch.float32)
    incs, errs = so.device_increments(seed, ts, _SDE_DT, rows, dim)
    field = so.Bounded((dc, scn), act, ts, _SDE_DT, _SDE_SIGMA, incs, errs, net_err=net_err)
    ref = osde.euler_sdeint(field, _SDE_SIGMA, y0_rows.double().cpu(), ts, _SDE_DT, incs)
    return ref, field.bound(math.exp(float(ts[-1] - ts[0]) * lip))


def _sde_edge_check(sde, ds, ss, dim, w, act, B, plan, seed_draw):
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(B + dim)).to(DEV)
    ys, n, seed = _own_noise_run(sde, y0, seed_draw)
    assert n == 1
    rows = np.array(sorted(set(sc.edge_rows(B, plan).values()) | {B // 3}))
    ref, bound = _sde_bound(ds, ss, dim, w, act, y0[rows], seed, rows, so.small_net_err)
    err = (ys[:, rows].cpu().double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound)[1:].max())
    return y0, ys, rows, ref, bound, float((err / bound)[1:].max())


@gpu
@pytest.mark.parametrize("w,d", sc.SDE_BMAX)
def test_sde_planner_edges(w, d, record_property):
    """The largest planned batch of (w, dim): edge rows under the per-entry trajectory bound.  The next batch either
    raises with no launch or, where the tensor-core class takes it, runs there on the same noise stream: the rows the
    two runs share agree within the sum of the two classes' bounds."""
    sms = _sms()
    dim = sc.resolve_dim(w, d, sms)
    B = sc.resolve("sde", "bmax", dim, w, sms)
    plan = sc.plan_sde(B, dim, w, sms)
    act = "silu" if dim % 2 else "selu"
    sde, ds, ss = _sde_case(dim, w, act, seed=4000 + dim + w, shrink=0.4)
    sde.sigma = _SDE_SIGMA
    y0, ys, rows, ref, bound, worst = _sde_edge_check(sde, ds, ss, dim, w, act, B, plan, 5)
    record_property("B", B)
    print(f"margins sde edges w={w} dim={dim} B={B} plan={plan[:3]}: {worst:.2e} of the gate")
    L = _ffi.lib()
    assert not L.cfm_sde_small_supported(B + 1, dim, w)
    y1 = torch.cat([y0, torch.randn(1, dim, device=DEV)])
    if sc.tc_supported(B + 1, dim, w):
        big, n, _ = _own_noise_run(sde, y1, 5)
        assert n > 1  # the tensor-core class: an init launch, then the captured steps
        torch.manual_seed(5)
        seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
        ref_tc, bound_tc = _sde_bound(ds, ss, dim, w, act, y0[rows], seed, rows, so.tc_net_err)
        got = big[:, rows].cpu().double()
        assert bool(((got - ref_tc).abs() <= bound_tc).all()), float(((got - ref_tc).abs() / bound_tc)[1:].max())
        assert bool(((got - ys[:, rows].cpu().double()).abs() <= bound + bound_tc).all())
    else:
        before = L.cfm_launch_count()
        with pytest.raises(NotImplementedError, match="no SDE kernel"):
            cfm_b200.sdeint(sde, y1, torch.tensor(_SDE_TS), method="euler", dt=_SDE_DT)
        assert L.cfm_launch_count() == before
    if d == "dmax":
        big = cfm_b200.SDE(cfm_b200.MLP(dim + 1, w=w, time_varying=True).to(DEV),
                           cfm_b200.MLP(dim + 1, w=w, time_varying=True).to(DEV), input_size=(dim + 1,))
        before = L.cfm_launch_count()
        with pytest.raises(NotImplementedError, match="no SDE kernel"):
            cfm_b200.sdeint(big, torch.zeros(1, dim + 1, device=DEV), torch.tensor(_SDE_TS), method="euler")
        assert L.cfm_launch_count() == before


_SDE_EDGES = [(w, dim, B) for w, dim, B in sc.SDE_WARP_SHAPES]


@gpu
@pytest.mark.parametrize("w,dim,name", _SDE_EDGES)
def test_sde_warp_count_plans(w, dim, name):
    """4, 8 and 16 warps per CTA with one row group each, and 16 with three: edge rows under the per-entry bound."""
    sms = _sms()
    B = sc.resolve("sde", name, dim, w, sms)
    plan = sc.plan_sde(B, dim, w, sms)
    sde, ds, ss = _sde_case(dim, w, "selu", seed=5000 + w, shrink=0.4)
    sde.sigma = _SDE_SIGMA
    *_, worst = _sde_edge_check(sde, ds, ss, dim, w, "selu", B, plan, 6)
    print(f"margins sde warps {name} B={B} plan={plan[:3]}: {worst:.2e} of the gate")


# ---- the SDE's own noise entry by entry -----------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B,dim,w,act", sc.NOISE_SHAPES)
def test_sde_own_noise_against_float64_entry_by_entry(B, dim, w, act):
    """bm=None on a step grid whose h changes (an off-grid ts, a dt that does not divide the span): the kernel draws
    dW_n = sqrt(h_n) z_n itself; every checked row stays within small_field_oracle.Bounded's per-entry bound."""
    sms = _sms()
    B = sc.resolve("sde", B, dim, w, sms)
    plan = sc.plan_sde(B, dim, w, sms)
    sde, ds, ss = _sde_case(dim, w, act, seed=6000 + dim + w, shrink=0.4)
    sde.sigma = _SDE_SIGMA
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(151)).to(DEV)
    ys, n, seed = _own_noise_run(sde, y0, 152)
    assert n == 1
    rows = np.array(sorted(set(sc.edge_rows(B, plan).values()) | set(range(0, B, max(1, B // 40)))))
    ref, bound = _sde_bound(ds, ss, dim, w, act, y0[rows], seed, rows, so.small_net_err)
    err = (ys[:, rows].cpu().double() - ref).abs()
    print(f"margins sde own noise B={B} dim={dim} w={w} {act}: {float((err / bound)[1:].max()):.3e} of the gate")
    assert bool((err <= bound).all()), float((err / bound)[1:].max())


# ---- buffers --------------------------------------------------------------------------------------------------------
_PAD = 67  # sentinel floats past the trajectory


def _padded(n):
    buf = torch.full((n + _PAD,), float("nan"), device=DEV)
    return buf, buf[:n]


def _untouched(buf, n):
    return bool(torch.isnan(buf[n:]).all()) and bool(torch.isfinite(buf[:n]).all())


@gpu
@pytest.mark.parametrize("w,dim,B", [(32, 3, 333), (64, 33, 1001), (64, 9, "80*SMs+3")])
def test_sde_writes_nothing_past_the_trajectory(w, dim, B):
    B = sc.resolve("sde", B, dim, w, _sms())
    sde, _, _ = _sde_case(dim, w, "selu", seed=7000 + w)
    d, s = sde.drift, sde.score
    ts = torch.tensor(_SDE_TS, dtype=torch.float32)
    grid, out_begin, out_a, out_b, _ = csde._tables_for(ts, _SDE_DT, torch.device(DEV))
    y0 = torch.randn(B, dim, generator=torch.Generator().manual_seed(7)).to(DEV)
    n = len(ts) * B * dim
    buf, traj = _padded(n)
    arr = C.c_void_p * 8
    L = _ffi.lib()
    _ffi.check(L.cfm_sde_small_euler_f32(
        arr(*[p.data_ptr() for p in d._device_params(y0.device)]),
        arr(*[p.data_ptr() for p in s._device_params(y0.device)]), dim, w, d.act, 0.5, _ffi.ptr(y0), B,
        _ffi.ptr(grid), grid.numel() - 1, _ffi.ptr(out_begin), _ffi.ptr(out_a), _ffi.ptr(out_b), len(ts), 123, None,
        _ffi.ptr(traj), _ffi.stream_ptr(DEV)), "sde")
    torch.cuda.synchronize()
    assert _untouched(buf, n)


def _grad_call(m, x, span, solver, traj, ws):
    L = _ffi.lib()
    B, dim = x.shape
    st = torch.zeros(C.sizeof(_ffi.RkState), dtype=torch.uint8, device=DEV)
    _ffi.check(L.cfm_ode_small_grad_trajectory_f32(
        *[_ffi.ptr(p) for p in m._device_params(x.device)], dim, m.w, 1, m.act, _ffi.ptr(x), B, _ffi.ptr(span),
        span.numel(), 1e-5, 1e-5, solver, _ffi.ptr(traj), _ffi.ptr(st), _ffi.ptr(ws), ws.numel(),
        _ffi.stream_ptr(DEV)), "grad")
    return st


@gpu
@pytest.mark.parametrize("w,dim,B", [(32, 1, 333), (64, 8, 1001), (64, 5, "fallback:2")])
def test_grad_field_buffers(w, dim, B):
    """Euler and dopri5 write nothing past [n_span][B][dim]; dopri5's grid partials are written before they are read:
    a NaN-filled workspace and a second call give the same bits."""
    B = sc.resolve("grad", B, dim, w, _sms())
    m, _ = _mlp(dim, w, seed=8000 + w, act="selu", out_dim=1)
    x = (2 * torch.randn(B, dim, generator=torch.Generator().manual_seed(8))).to(DEV)
    span = torch.linspace(0, 1, 4, device=DEV)
    nbytes = _ffi.lib().cfm_ode_small_workspace_bytes(B, dim, w)
    n = 4 * B * dim
    runs = []
    for solver, fill in ((1, 0), (0, 0), (0, 0xFF), (0, 0xFF)):
        ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV)  # 0xFF bytes: NaN doubles
        buf, traj = _padded(n)
        _grad_call(m, x, span, solver, traj, ws)
        torch.cuda.synchronize()
        assert _untouched(buf, n), solver
        runs.append(traj.clone())
    assert torch.equal(runs[1], runs[2]) and torch.equal(runs[2], runs[3])
