"""GPU checks of gradients through the exact-likelihood Euler trajectory (csrc/cnf_train.cu, DESIGN.md section 3.14):
the backward kernel against the float64 discrete adjoint at the device's own fp32 states, the tutorial's cell end to
end against float64 autograd, launch counts and bit-repeatability, autograd semantics, training, and the node that
refuses gradients outside the kernel's class.  The achieved errors and the reasons for each gate are in DESIGN.md
section 3.14."""
import math
import re

import pytest
import torch

import cnf_oracle as co
import cnf_train_oracle as cto
import train_scale_oracle as so
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KERNEL_GATE = 2e-5  # of each gradient tensor's max-abs, kernel at the device states against float64
ENTRY_GATE = 2e-6   # and of each entry's own absolute scale (tests/train_scale_oracle.py)
E2E_GATE = 5e-6     # the tutorial's cell against float64 autograd through the float64 trajectory
SGD_GATE = 5e-6     # parameters after 20 SGD steps against float64 training
BATCHES = [1, 2, 3, 15, 16, 17, 255, 256, 257, 4096]
SPANS = [(101, "reverse"), (2, "forward"), (3, "reverse"), (101, "forward"), (3, "forward"), (2, "reverse")]


def _mlp(dim, w, act, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
    return m.to(DEV)


def _span(n, direction):
    s = torch.linspace(0, 1, n)
    return s.flip(0) if direction == "reverse" else s


def _launches():
    return _ffi.lib().cfm_launch_count()


def _largest_batch(dim, w):
    lib = _ffi.lib()
    lo, hi = 4096, 1 << 31
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if lib.cfm_ode_small_cnf_backward_supported(mid, dim, w) else (lo, mid)
    return lo


def _entry_errors(got, ref, scales):
    return [((g.double().cpu() - r.cpu()).abs() / s.cpu().clamp_min(1e-300)).max().item()
            for g, r, s in zip(got, ref, scales)]


def _rel_errors(got, ref):
    return [(g.double() - r).abs().max().item() / max(r.abs().max().item(), 1e-30) for g, r in zip(got, ref)]


def _kernel_case(m, act, B, n, direction, seed):
    dim = m.dim
    g = torch.Generator(device=DEV).manual_seed(seed)
    z = torch.randn(B, dim + 1, device=DEV, generator=g).requires_grad_(True)
    span = _span(n, direction)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver="euler")
    traj = node.trajectory(z, span)
    G = torch.randn(traj.shape, device=DEV, generator=g)
    G[1:-1:2] = 0.0  # cotangents on every other inner checkpoint only
    state = {k: v.detach() for k, v in m.state_dict().items()}
    if act == "selu":
        G[:, cto.kink_rows(state, traj.detach(), span)] = 0.0
    params = list(m.parameters())
    got = torch.autograd.grad(traj, params + [z], G)
    ref_p, ref_z = cto.restated_backward(state, traj.detach(), span, G, act, h32=True)
    sc_p, sc_z = so.cnf_grad_scales(state, traj.detach(), span, G, act)
    ref = list(ref_p) + [ref_z]
    return _entry_errors(got, ref, list(sc_p) + [sc_z]), _rel_errors(got, ref)


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", range(1, 9))
@pytest.mark.parametrize("w", [32, 64])
def test_backward_kernel_against_the_float64_adjoint_at_the_device_states(w, dim, act):
    m = _mlp(dim, w, act, seed=10 * dim + w)
    worst = [0.0, 0.0]
    for i, B in enumerate(BATCHES + [_largest_batch(dim, w)]):
        n, direction = SPANS[i % len(SPANS)]
        if B > 4096:
            n = 2 + i % 2
        errs, rel = _kernel_case(m, act, B, n, direction, seed=i)
        worst = [max(worst[0], max(errs)), max(worst[1], max(rel))]
        assert max(errs) <= ENTRY_GATE and max(rel) <= KERNEL_GATE, (B, n, direction, errs, rel)
    print(f"ERR kernel w={w} dim={dim} act={act} worst grad/abs-scale {worst[0]:.3e} grad/max-abs {worst[1]:.3e}")


def _moons(n, g, noise=0.1):
    """sklearn's make_moons, restated: two interleaved half circles plus Gaussian noise."""
    half = n // 2
    t_out = torch.rand(n - half, generator=g, dtype=torch.float64) * math.pi
    t_in = torch.rand(half, generator=g, dtype=torch.float64) * math.pi
    x = torch.cat([torch.stack([torch.cos(t_out), torch.sin(t_out)], 1),
                   torch.stack([1 - torch.cos(t_in), 0.5 - torch.sin(t_in)], 1)])
    return (x + noise * torch.randn(x.shape, generator=g, dtype=torch.float64)).float()


def _tutorial_loss(traj, prior, weight=None):
    x0 = traj[-1]
    logprob = prior.log_prob(x0[..., :-1]) + x0[..., -1]
    if weight is not None:
        logprob = logprob * weight
    return -torch.mean(logprob)


def test_tutorial_cell_end_to_end_against_float64_autograd():
    m = _mlp(2, 64, "selu", seed=1)
    mc = vf.make_mlp(2, w=64, time_varying=True, dtype=torch.float64)
    mc.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    g = torch.Generator().manual_seed(2)
    x1 = _moons(256, g)
    span = torch.linspace(1, 0, 101)
    z = torch.cat([x1, torch.zeros(256, 1)], 1)
    ref_traj = cto.euler_loop(co.cnf_field(mc), z.double(), span.double())
    keep = (~cto.kink_rows(mc.state_dict(), ref_traj.detach(), span.double())).double()
    prior64 = torch.distributions.MultivariateNormal(torch.zeros(2, dtype=torch.float64),
                                                     torch.eye(2, dtype=torch.float64))
    _tutorial_loss(ref_traj, prior64, keep).backward()
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator="exact"), solver="euler",
                              sensitivity="adjoint")
    prior = torch.distributions.MultivariateNormal(torch.zeros(2, device=DEV), torch.eye(2, device=DEV))
    traj = node.trajectory(z.to(DEV), t_span=torch.linspace(1, 0, 101, device=DEV))
    _tutorial_loss(traj, prior, keep.float().to(DEV)).backward()
    errs = _rel_errors([p.grad.cpu() for p in m.parameters()], [p.grad for p in mc.parameters()])
    print(f"ERR end-to-end {max(errs):.3e} kink rows {int((keep == 0).sum())}")
    assert max(errs) <= E2E_GATE, errs


def test_forward_is_unchanged_and_backward_is_one_launch_with_the_same_bits():
    m = _mlp(2, 64, "selu", seed=3)
    z = torch.randn(256, 3, device=DEV)
    span = torch.linspace(1, 0, 101)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver="euler")
    with torch.no_grad():
        plain = node.trajectory(z, span)
    grads = []
    for _ in range(2):
        before = _launches()
        traj = node.trajectory(z, span)
        assert _launches() - before == 1
        assert traj.requires_grad and torch.equal(traj, plain)
        loss = traj[-1].square().sum()
        before = _launches()
        grads.append(torch.autograd.grad(loss, list(m.parameters())))
        assert _launches() - before == 1
    assert all(torch.equal(a, b) for a, b in zip(*grads))
    t, traj = node(z, span)  # NeuralODE.forward: (t_span, traj) like torchdyn's
    assert traj.requires_grad and torch.equal(t.cpu(), span) and torch.equal(traj, plain)


def test_autograd_semantics():
    m = _mlp(2, 32, "silu", seed=4)
    span = torch.linspace(1, 0, 11)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver="euler")
    z = torch.randn(64, 3, device=DEV)
    node.trajectory(z, span)[-1].sum().backward()
    assert z.grad is None  # only the parameters require grad
    first = [p.grad.clone() for p in m.parameters()]
    node.trajectory(z, span)[-1].sum().backward()
    assert all(torch.equal(p.grad, 2 * f) for p, f in zip(m.parameters(), first))  # accumulates
    m.zero_grad()
    (0.5 * node.trajectory(z, span)[-1].sum()).backward()
    assert all(torch.allclose(p.grad, 0.5 * f, rtol=1e-6, atol=0) for p, f in zip(m.parameters(), first))
    zr = z.clone().requires_grad_(True)
    node.trajectory(zr, span)[-1].sum().backward()
    assert zr.grad is not None and zr.grad.shape == (64, 3) and torch.all(zr.grad[:, 2] == 1.0)
    traj = node.trajectory(z, span)
    with torch.no_grad():
        m.net[2].weight.add_(0.01)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        traj.sum().backward()


def test_twenty_sgd_steps_track_float64_training_and_adam_runs_the_cell_verbatim():
    m = _mlp(2, 64, "selu", seed=5)
    mc = vf.make_mlp(2, w=64, time_varying=True, dtype=torch.float64)
    mc.load_state_dict({k: v.double().cpu() for k, v in m.state_dict().items()})
    opt, opt64 = torch.optim.SGD(m.parameters(), lr=1e-2), torch.optim.SGD(mc.parameters(), lr=1e-2)
    prior = torch.distributions.MultivariateNormal(torch.zeros(2, device=DEV), torch.eye(2, device=DEV))
    prior64 = torch.distributions.MultivariateNormal(torch.zeros(2, dtype=torch.float64),
                                                     torch.eye(2, dtype=torch.float64))
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver="euler", sensitivity="adjoint")
    span = torch.linspace(1, 0, 101)
    g = torch.Generator().manual_seed(6)
    for _ in range(20):
        x1 = _moons(256, g)
        z = torch.cat([x1, torch.zeros(256, 1)], 1)
        opt.zero_grad()
        _tutorial_loss(node.trajectory(z.to(DEV), span), prior).backward()
        opt.step()
        opt64.zero_grad()
        _tutorial_loss(cto.euler_loop(co.cnf_field(mc), z.double(), span.double()), prior64).backward()
        opt64.step()
    errs = _rel_errors([p.detach().cpu() for p in m.parameters()], [p.detach() for p in mc.parameters()])
    print(f"ERR sgd-20 {max(errs):.3e}")
    assert max(errs) <= SGD_GATE, errs

    # the tutorial's cell 4, verbatim but for the classes
    device = DEV
    model = m
    optimizer = torch.optim.Adam(model.parameters())
    cnf = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(model, likelihood_estimator="exact"), solver="euler",
                             sensitivity="adjoint")
    steps = 100
    for k in range(3):
        before = _launches()
        optimizer.zero_grad()
        x1 = _moons(256, g).to(device)
        x1_with_ll = torch.cat([x1, torch.zeros(x1.shape[0], 1, device=device)], dim=-1)
        x0_with_ll = cnf.trajectory(x1_with_ll, t_span=torch.linspace(1, 0, steps + 1, device=device))[-1]
        logprob = prior.log_prob(x0_with_ll[..., :-1]) + x0_with_ll[..., -1]
        loss = -torch.mean(logprob)
        loss.backward()
        optimizer.step()
        assert _launches() - before == 2
    assert all(torch.isfinite(p).all() for p in model.parameters())


@pytest.mark.parametrize("solver,w,text", [
    ("dopri5", 64, "gradients through the adaptive dopri5 solve are not implemented; use solver='euler'"),
    ("euler", 128, "w=128"),
])
def test_outside_the_class_the_forward_is_unchanged_and_backward_raises(solver, w, text):
    m = _mlp(2, w, "selu", seed=7)
    z = torch.randn(256, 3, device=DEV)
    span = torch.linspace(1, 0, 11)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver=solver)
    with torch.no_grad():
        before = _launches()
        plain = node.trajectory(z, span)
        n_plain = _launches() - before
    before = _launches()
    traj = node.trajectory(z, span)
    assert _launches() - before == n_plain
    assert torch.equal(traj, plain) and traj.requires_grad
    with pytest.raises(NotImplementedError, match=re.escape(text)):
        traj[-1].sum().backward()
