"""GPU checks of the exact-likelihood (CNF) path: NeuralODE(cnf_wrapper(MLP(time_varying=True), "exact")) in the
CNF variant of the one-launch kernel (csrc/ode_small.cu) against the float64 CNF oracle (tests/cnf_oracle.py),
and plain dopri5 over decreasing spans (the time-reversed field) in both ODE drivers."""
import math

import pytest
import torch

import cnf_oracle as co
from oracle import vector_field as vf
from test_gpu_small_fields import assert_cnf_close, smooth_rows

import cfm_b200
from cfm_b200 import _ffi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _pair(dim=2, w=64, seed=0, silu=False):
    """(device MLP, float64 CPU oracle MLP) with the same weights."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
    mc = vf.make_mlp(dim, w=w, time_varying=True, dtype=torch.float64)
    mc.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    if silu:
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            mc.net[k] = torch.nn.SiLU()
    return m.to(DEV), mc


def _state(x):
    return torch.cat([x, torch.zeros(x.shape[0], 1, dtype=x.dtype)], 1)


def test_euler_tutorial_shape_bit_identical_x_and_float64_trace():
    m, mc = _pair(seed=1)
    x1 = torch.randn(256, 2, generator=torch.Generator().manual_seed(2))
    span = torch.linspace(1, 0, 101)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator="exact"), solver="euler")
    traj = node.trajectory(_state(x1).to(DEV), span)
    assert traj.shape == (101, 256, 3) and node.stats["fused"] and node.stats["nfe"] == 100
    plain = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="euler").trajectory(x1.to(DEV), span)
    assert torch.equal(traj[..., :2], plain)
    ref = co.euler_any_direction(co.cnf_field(mc), _state(x1).double(), span.double())
    ll, ll_ref = traj[..., 2].cpu().double(), ref[..., 2]
    assert (ll - ll_ref).abs().max() <= 1e-4 * max(1.0, ll_ref.abs().max().item())
    assert (traj[..., :2].cpu().double() - ref[..., :2]).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("B,span", [(256, [1.0, 0.0]), (1001, [1.0, 0.75, 0.5, 0.0])])
def test_dopri5_reversed_span_matches_the_float64_oracle_step_for_step(B, span):
    m, mc = _pair(seed=3)
    z = _state(torch.randn(B, 2, generator=torch.Generator().manual_seed(4)))
    ts = torch.tensor(span)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    traj = node.trajectory(z.to(DEV), ts)
    ref, st = co.dopri5_any_direction(co.cnf_field(mc), z.double(), ts.double(), 1e-4, 1e-4)
    assert node.stats["fused"]
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert node.stats["t"] == pytest.approx(span[-1], abs=1e-6)
    assert traj.shape == ref.shape
    assert (traj.cpu().double() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("solver", ["euler", "dopri5"])
def test_analytic_affine_field_log_density_is_minus_trace(solver):
    """Positive hidden pre-activations: SELU is linear, tr(df/dx) = tr(A) everywhere, ll over [1, 0] = -tr(A)."""
    mc = co.positive_selu_mlp(dim=2, w=64, seed=5, dtype=torch.float32)
    m = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    m.load_state_dict(mc.state_dict())
    m = m.to(DEV)
    tr = co.affine_trace(mc, 2)
    z = _state(2 * torch.randn(128, 2, generator=torch.Generator().manual_seed(6)))
    span = torch.linspace(1, 0, 101) if solver == "euler" else torch.tensor([1.0, 0.0])
    seen = []  # positivity along the (float64) path through the same points
    mc64 = co.positive_selu_mlp(dim=2, w=64, seed=5, dtype=torch.float32).double()
    f = co.recording(lambda t, zz: vf.wrapped_forward(mc64, t, zz[:, :-1]), seen)
    co.euler_any_direction(lambda t, zz: torch.cat([f(t, zz), torch.zeros_like(zz[:, :1])], 1), z.double(),
                           torch.linspace(1, 0, 101, dtype=torch.float64))
    assert co.min_preactivation(mc64, seen) > 1.0
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver=solver, atol=1e-5, rtol=1e-5)
    ll = node.trajectory(z.to(DEV), span)[-1, :, 2].cpu().double()
    assert (ll + tr).abs().max() <= 2e-5 * max(1.0, abs(tr)), (ll[:4], tr)


@pytest.mark.parametrize("fused", [True, False])
def test_plain_dopri5_decreasing_span_matches_the_reversed_oracle(fused):
    m, mc = _pair(seed=7)
    x = torch.randn(512, 2, generator=torch.Generator().manual_seed(8))
    span = torch.linspace(1, 0, 4)
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    node.use_fused_small = fused
    traj = node.trajectory(x.to(DEV), span)
    ref, st = co.dopri5_any_direction(lambda t, z: vf.wrapped_forward(mc, t, z), x.double(), span.double())
    assert bool(node.stats.get("fused")) == fused
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert node.stats["t"] == pytest.approx(0.0, abs=1e-6)
    assert torch.isfinite(traj).all()
    assert (traj.cpu().double() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())
    # an increasing span afterwards still takes the forward field
    fwd = node.trajectory(x.to(DEV), torch.linspace(0, 1, 4))
    ref_f, _ = vf.dopri5_trajectory(lambda t, z: vf.wrapped_forward(mc, t, z), x.double(),
                                    torch.linspace(0, 1, 4, dtype=torch.float64))
    assert (fwd.cpu().double() - ref_f).abs().max() <= 1e-4 * max(1.0, ref_f.abs().max().item())


def _moons(n, gen):
    """Two interleaved half circles with noise (the tutorial's target density), scaled as sample_moons does."""
    k = n // 2
    a = math.pi * torch.rand(k, generator=gen)
    b = math.pi * torch.rand(n - k, generator=gen)
    upper = torch.stack([torch.cos(a), torch.sin(a)], 1)
    lower = torch.stack([1 - torch.cos(b), 0.5 - torch.sin(b)], 1)
    x = torch.cat([upper, lower]) + 0.2 * torch.randn(n, 2, generator=gen)
    return 3 * (x - 0.5)


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_tutorial_log_likelihood_matches_stock_pytorch(act):
    """log p(x1) = prior.log_prob(x0) + ll, integrated [x1, 0] over linspace(1, 0, 101) with Euler: the kernel
    against the tutorial's cnf_wrapper on a plain torch MLP (eager PyTorch, same GPU)."""
    m, mc = _pair(seed=9, silu=act == "silu")
    stock = mc.float().to(DEV)
    x1 = _moons(256, torch.Generator().manual_seed(10)).to(DEV)
    z1 = torch.cat([x1, torch.zeros(256, 1, device=DEV)], 1)
    span = torch.linspace(1, 0, 101, device=DEV)
    prior = torch.distributions.MultivariateNormal(torch.zeros(2, device=DEV), torch.eye(2, device=DEV))
    z0 = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator="exact"), solver="euler").trajectory(
        z1, span)[-1]
    z0_ref = vf.euler_trajectory(cfm_b200.cnf_wrapper(stock, likelihood_estimator="exact"), z1, span)[-1]
    logp = prior.log_prob(z0[..., :-1]) + z0[..., -1]
    logp_ref = prior.log_prob(z0_ref[..., :-1]) + z0_ref[..., -1]
    assert (logp - logp_ref).abs().max().item() <= 1e-4 * max(1.0, logp_ref.abs().max().item())


def test_density_grid_40000_points_in_one_launch():
    m, mc = _pair(seed=11)
    g = torch.linspace(-3, 3, 200)
    xx, yy = torch.meshgrid(g, g, indexing="ij")
    zc = _state(torch.stack([xx.reshape(-1), yy.reshape(-1)], 1))
    z = zc.to(DEV)
    assert _ffi.lib().cfm_ode_small_cnf_supported(40000, 2, 64)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="euler")
    before = _ffi.lib().cfm_launch_count()
    span = torch.linspace(1, 0, 201)
    traj = node.trajectory(z, span)
    assert _ffi.lib().cfm_launch_count() - before == 1
    assert node.stats["fused"] and traj.shape == (201, 40000, 3) and torch.isfinite(traj).all()
    # Euler rows are independent: a sub-batch integrates to the same bits, and sampled rows match the float64 oracle
    sub = node.trajectory(z[:333], span)
    assert torch.equal(sub, traj[:, :333])
    rows = torch.randperm(40000, generator=torch.Generator().manual_seed(13))[:1000]
    ref = co.euler_any_direction(co.cnf_field(mc), zc[rows].double(), span.double())
    assert (traj[:, rows.to(DEV)].cpu().double() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())
    # dopri5: the log-density column is gated away from SELU's kink, where fp32 need not take float64's branch of act'
    node5 = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    out = node5.trajectory(z, torch.linspace(1, 0, 2))
    assert node5.stats["fused"] and torch.isfinite(out).all()
    seen = []
    ref5, st = co.dopri5_any_direction(co.recording(co.cnf_field(mc), seen), zc.double(),
                                       torch.linspace(1, 0, 2, dtype=torch.float64), 1e-4, 1e-4)
    assert (node5.stats["nfe"], node5.stats["accepted"], node5.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert_cnf_close(out.cpu().double(), ref5, smooth_rows(mc, seen, "selu"), 1e-4)


def test_refusals():
    m, _ = _pair(seed=12)
    z = torch.zeros(64, 3, device=DEV)
    span = torch.linspace(1, 0, 3)
    for est in ("hutch_gaussian", "hutch_rademacher"):
        with pytest.raises(NotImplementedError, match="Hutchinson"):
            cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator=est), solver="euler").trajectory(z, span)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="dopri5")
    node.lockstep = True
    with pytest.raises(NotImplementedError, match="lock-step"):
        node.trajectory(z, span)
    wide = cfm_b200.MLP(dim=2, w=256, time_varying=True).to(DEV)
    with pytest.raises(NotImplementedError, match="no exact-likelihood kernel"):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(wide), solver="euler").trajectory(z, span)
    big_dim = cfm_b200.MLP(dim=9, w=64, time_varying=True).to(DEV)
    with pytest.raises(NotImplementedError, match="no exact-likelihood kernel"):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(big_dim), solver="euler").trajectory(torch.zeros(8, 10, device=DEV),
                                                                                      span)
    assert not _ffi.lib().cfm_ode_small_cnf_supported(64, 9, 64)
    assert not _ffi.lib().cfm_ode_small_cnf_supported(64, 2, 256)
    with pytest.raises(ValueError):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver="euler").trajectory(torch.zeros(8, 2, device=DEV), span)
    with pytest.raises(TypeError):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(torch.nn.Linear(3, 2)), solver="euler").trajectory(z, span)
