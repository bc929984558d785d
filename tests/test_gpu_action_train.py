"""cfm_b200.action_matching_loss on the device (mlp_action_train_kernel in csrc/action_train.cu: the action-matching
loss of a scalar-action MLP, its input gradient and all eight parameter gradients in one launch) against
tests/action_oracle.py, the notebook's lines in float64 on the CPU with torch's double backward.

The loss is a difference of terms of size mean(|s0| + |s1| + 1/2 |g_x|^2 + |g_t|), so its error is gated relative to
that; each parameter gradient both relative to its tensor's max-abs and entry by entry relative to its own absolute
scale (tests/train_scale_oracle.py).  SELU' and SELU'' jump at 0, so with SELU only rows
whose float64 pre-activations at all three evaluation points stay further than _KINK_REL of their magnitude sum from
the kink are compared (as test_gpu_train.py and test_gpu_action.py gate theirs)."""
import math

import action_oracle as ao
import train_scale_oracle as so
import pytest
import torch

import cfm_b200
from cfm_b200 import _ffi

DEV = "cuda:0"
gpu = pytest.mark.gpu

BATCHES = [1, 2, 3, 15, 16, 17, 255, 256, 257, 1000, 4096]
LOSS_REL, GRAD_REL = 2e-6, 2e-5  # GRAD_REL: every gradient tensor's error, of its max-abs
GRAD_ABS = 1.5e-6  # and every entry, of its own absolute scale (tests/train_scale_oracle.py); DESIGN.md 3.13
_KINK_REL = 1e-5


def _model(dim, w, act, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m.to(DEV)


def _away_from_kink(mc, z):
    """Rows of z whose float64 hidden pre-activations all stay further than _KINK_REL of their magnitude sum from 0."""
    with torch.no_grad():
        h = z.double()
        keep = torch.ones(h.shape[0], dtype=torch.bool)
        for li in (0, 2, 4):
            W, b = mc.net[li].weight, mc.net[li].bias
            p = h @ W.T + b
            keep &= (p.abs() > _KINK_REL * (h.abs() @ W.abs().T + b.abs())).all(1)
            h = mc.net[li + 1](p)
    return keep


def _keep(m, act, xt, t, x0, x1):
    if act != "selu":
        return torch.ones(xt.shape[0], dtype=torch.bool)
    mc = ao.make_action(m.state_dict(), m.dim, m.w, act)
    n = xt.shape[0]
    return (_away_from_kink(mc, torch.cat([xt, t.reshape(n, 1)], 1))
            & _away_from_kink(mc, torch.cat([x0, torch.zeros(n, 1)], 1))
            & _away_from_kink(mc, torch.cat([x1, torch.ones(n, 1)], 1)))


def _batch(m, B, seed, act="selu"):
    """Seeded (xt, t (B, 1), x0, x1) on the CPU, the notebook's way (xt on the segment from x0 to x1), every row away
    from SELU's kink at all three points."""
    g = torch.Generator().manual_seed(seed)
    n = B + max(64, B // 20)
    x0, x1 = torch.randn(n, m.dim, generator=g) * 1.5, torch.randn(n, m.dim, generator=g) * 1.5 + 1.0
    t = torch.rand(n, 1, generator=g)
    xt = t * x1 + (1 - t) * x0
    keep = _keep(m, act, xt, t, x0, x1)
    assert int(keep.sum()) >= B
    return tuple(v[keep][:B].clone() for v in (xt, t, x0, x1))


def _device_loss_and_grads(m, xt, t, x0, x1):
    m.zero_grad(set_to_none=True)
    loss = cfm_b200.action_matching_loss(m, *(v.to(DEV) for v in (xt, t, x0, x1)))
    loss.backward()
    return loss.detach(), [p.grad.detach().clone() for p in m.parameters()]


def _gaps(m, act, xt, t, x0, x1):
    """(loss error over its scale, worst gradient error over its entry's absolute scale, worst gradient error over
    the tensor's max-abs) against the float64 oracle, with b3's gradient checked to be exactly 0."""
    loss, grads = _device_loss_and_grads(m, xt, t, x0, x1)
    assert loss.shape == () and loss.dtype == torch.float32 and loss.is_cuda
    rl, rg = ao.action_matching_loss_and_grads(m.state_dict(), m.dim, m.w, xt, t, x0, x1, act)
    scale = ao.loss_scale(ao.make_action(m.state_dict(), m.dim, m.w, act), xt, t, x0, x1)
    lgap = abs(loss.item() - rl.item()) / scale
    scales = so.action_grad_scales(m.state_dict(), xt, t, x0, x1, act)
    ggap = rgap = 0.0
    for p, g, r, sc in zip(list(m.parameters())[:7], grads[:7], rg[:7], scales[:7]):
        assert g.shape == p.shape and torch.isfinite(g).all()
        err = (g.cpu().double() - r).abs()
        ggap = max(ggap, (err / sc.clamp_min(1e-300)).max().item())
        rgap = max(rgap, err.max().item() / r.abs().max().item())
    assert grads[7].shape == (1,) and grads[7].item() == 0.0
    return lgap, ggap, rgap


# ---- every instantiation, every batch-size class -------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dim", [1, 2, 5, 8])
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("w", [32, 64])
def test_loss_and_gradients_match_the_float64_oracle(w, act, dim):
    m = _model(dim, w, act, seed=200 + w + dim)
    worst = [0.0, 0.0, 0.0]
    for B in BATCHES:
        gaps = _gaps(m, act, *_batch(m, B, seed=B, act=act))
        assert gaps[0] <= LOSS_REL and gaps[1] <= GRAD_ABS and gaps[2] <= GRAD_REL, (B, gaps)
        worst = [max(a, b) for a, b in zip(worst, gaps)]
    print(f"margins w={w} {act} dim={dim}: loss {worst[0]:.2e} grad/abs-scale {worst[1]:.2e} "
          f"grad/max-abs {worst[2]:.2e}")


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_edge_times_where_the_middle_point_is_an_endpoint(act):
    m = _model(2, 64, act, seed=11)
    xt, t, x0, x1 = _batch(m, 300, seed=5, act=act)
    t[::2], t[1::2] = 0.0, 1.0
    xt = t * x1 + (1 - t) * x0
    keep = _keep(m, act, xt, t, x0, x1)
    lgap, ggap, rgap = _gaps(m, act, xt[keep], t[keep], x0[keep], x1[keep])
    assert lgap <= LOSS_REL and ggap <= GRAD_ABS and rgap <= GRAD_REL, (lgap, ggap, rgap)


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_zero_output_layer_gives_exact_zeros(act):
    """W3 = 0: s is the constant b3, so the loss and every gradient but dW3 are exactly 0; dW3 is the mean of
    h_2(x0) - h_2(x1) + the tangent h'_2 along c = [0, 1], and matches the oracle."""
    m = _model(3, 32, act, seed=12)
    with torch.no_grad():
        m.net[6].weight.zero_()
    xt, t, x0, x1 = _batch(m, 257, seed=6, act=act)
    loss, grads = _device_loss_and_grads(m, xt, t, x0, x1)
    assert loss.item() == 0.0
    assert all(not g.any() for k, g in enumerate(grads) if k != 6)
    _, rg = ao.action_matching_loss_and_grads(m.state_dict(), 3, 32, xt, t, x0, x1, act)
    assert (grads[6].cpu().double() - rg[6]).abs().max().item() <= GRAD_REL * rg[6].abs().max().item()


# ---- determinism and launches ------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B", [256, 5000])
def test_repeated_calls_give_the_same_bits_and_no_grad_gives_the_same_loss(B):
    m = _model(2, 64, "selu", seed=5)
    args = [v.to(DEV) for v in _batch(m, B, seed=9)]
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        loss = cfm_b200.action_matching_loss(m, *args)
        loss.backward()
        runs.append((loss.detach().clone(), [p.grad.clone() for p in m.parameters()]))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
    with torch.no_grad():
        only = cfm_b200.action_matching_loss(m, *args)
    assert not only.requires_grad and torch.equal(only, runs[0][0])


@gpu
def test_one_launch_per_call_and_none_in_backward():
    m = _model(2, 64, "selu", seed=5)
    args = [v.to(DEV) for v in _batch(m, 256, seed=9)]
    cfm_b200.action_matching_loss(m, *args).backward()  # loads the kernel
    L = _ffi.lib()
    before = L.cfm_launch_count()
    loss = cfm_b200.action_matching_loss(m, *args)
    assert L.cfm_launch_count() - before == 1
    loss.backward()
    with torch.no_grad():
        cfm_b200.action_matching_loss(m, *args)
    assert L.cfm_launch_count() - before == 2


# ---- the autograd contract --------------------------------------------------------------------------------------------
@gpu
def test_gradients_accumulate_scale_and_follow_in_place_updates():
    m = _model(2, 64, "selu", seed=6)
    args = [v.to(DEV) for v in _batch(m, 256, seed=4)]
    _, g1 = _device_loss_and_grads(m, *args)
    m.zero_grad(set_to_none=True)
    cfm_b200.action_matching_loss(m, *args).backward()
    cfm_b200.action_matching_loss(m, *args).backward()
    for p, g in zip(m.parameters(), g1):
        assert torch.equal(p.grad, g + g)
    m.zero_grad(set_to_none=True)
    (0.5 * cfm_b200.action_matching_loss(m, *args)).backward()
    for p, g in zip(m.parameters(), g1):
        assert torch.equal(p.grad, 0.5 * g)
    opt = torch.optim.SGD(m.parameters(), lr=1e-3)
    before = cfm_b200.action_matching_loss(m, *args)
    opt.zero_grad()
    before.backward()
    opt.step()
    after, ga = _device_loss_and_grads(m, *args)
    assert after.item() < before.item()
    cpu = [v.cpu() for v in args]
    rl, rg = ao.action_matching_loss_and_grads(m.state_dict(), 2, 64, *cpu)
    scale = ao.loss_scale(ao.make_action(m.state_dict(), 2, 64), *cpu)
    assert abs(after.item() - rl.item()) <= LOSS_REL * scale
    for g, r in zip(ga[:7], rg[:7]):
        assert (g.cpu().double() - r).abs().max().item() <= GRAD_REL * r.abs().max().item()


def _eight_gaussians(n, g):
    centers = torch.tensor([(1, 0), (-1, 0), (0, 1), (0, -1), (1 / math.sqrt(2), 1 / math.sqrt(2)),
                            (1 / math.sqrt(2), -1 / math.sqrt(2)), (-1 / math.sqrt(2), 1 / math.sqrt(2)),
                            (-1 / math.sqrt(2), -1 / math.sqrt(2))], dtype=torch.float32) * 5.0
    return centers[torch.randint(0, 8, (n,), generator=g)] + 0.5 * torch.randn(n, 2, generator=g)


def _moons(n, g):
    a = torch.rand(n, generator=g) * math.pi
    upper = torch.rand(n, generator=g) < 0.5
    x = torch.where(upper, torch.cos(a), 1 - torch.cos(a))
    y = torch.where(upper, torch.sin(a), 0.5 - torch.sin(a))
    return (torch.stack([x, y], 1) + 0.2 * torch.randn(n, 2, generator=g)) * 3 - 1


@gpu
def test_twenty_sgd_steps_track_float64_training():
    """The notebook's action-matching loop (8 gaussians -> moons, batch 256, t ~ U(0, 1), xt on the segment) for 20 SGD
    steps through action_matching_loss, against the same 20 steps in float64 on the same batches."""
    g = torch.Generator().manual_seed(0)
    m = _model(2, 64, "selu", seed=1)
    mc = ao.make_action(m.state_dict(), 2, 64)
    opt, optc = torch.optim.SGD(m.parameters(), lr=1e-3), torch.optim.SGD(mc.parameters(), lr=1e-3)
    for _ in range(20):
        x0, x1 = _eight_gaussians(256, g), _moons(256, g)
        t = torch.rand(256, 1, generator=g)
        xt = t * x1 + (1 - t) * x0
        opt.zero_grad()
        cfm_b200.action_matching_loss(m, xt.to(DEV), t.to(DEV), x0.to(DEV), x1.to(DEV)).backward()
        opt.step()
        optc.zero_grad()
        ao.loss_of(mc, xt, t, x0, x1).backward()
        optc.step()
    for p, r in zip(m.parameters(), mc.parameters()):
        assert (p.detach().cpu().double() - r.detach()).abs().max().item() <= 1e-4 * r.detach().abs().max().item()


# ---- scale and layout --------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_large_batch_keeps_every_cta_busy(act):
    m = _model(2, 64, act, seed=8)
    lgap, ggap, rgap = _gaps(m, act, *_batch(m, 65536, seed=10, act=act))
    print(f"margins B=65536 {act}: loss {lgap:.2e} grad/abs-scale {ggap:.2e} grad/max-abs {rgap:.2e}")
    assert lgap <= LOSS_REL and ggap <= GRAD_ABS and rgap <= GRAD_REL, (lgap, ggap, rgap)


@gpu
def test_strided_inputs_are_made_contiguous():
    m = _model(2, 32, "silu", seed=9)
    xt, t, x0, x1 = _batch(m, 64, seed=3, act="silu")
    wide = torch.randn(64, 9)
    wide[:, 0:6:3], wide[:, 1:7:3], wide[:, 2:8:3], wide[:, 8] = xt, x0, x1, t[:, 0]
    wd = wide.to(DEV)
    with torch.no_grad():
        a = cfm_b200.action_matching_loss(m, wd[:, 0:6:3], wd[:, 8], wd[:, 1:7:3], wd[:, 2:8:3])
        b = cfm_b200.action_matching_loss(m, *(v.to(DEV) for v in (xt, t, x0, x1)))
    assert torch.equal(a, b) and math.isfinite(a.item())


# ---- refusals on the device ----------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("kw", [dict(dim=2, out_dim=1, w=128), dict(dim=9, out_dim=1, w=64),
                                dict(dim=2, out_dim=2, w=64), dict(dim=2, out_dim=1, w=64, time_varying=False)],
                         ids=["w128", "dim9", "out_dim2", "not_time_varying"])
def test_actions_outside_the_class_raise_on_the_device(kw):
    m = cfm_b200.MLP(**{"time_varying": True, **kw}).to(DEV)
    d = kw["dim"]
    args = [torch.randn(8, d, device=DEV), torch.rand(8, device=DEV), torch.randn(8, d, device=DEV),
            torch.randn(8, d, device=DEV)]
    with pytest.raises(NotImplementedError, match="action_matching_loss"):
        cfm_b200.action_matching_loss(m, *args)


@gpu
def test_a_non_mlp_action_raises_on_the_device():
    net = torch.nn.Sequential(torch.nn.Linear(3, 64), torch.nn.SELU(), torch.nn.Linear(64, 1)).to(DEV)
    args = [torch.randn(8, 2, device=DEV), torch.rand(8, 1, device=DEV), torch.randn(8, 2, device=DEV),
            torch.randn(8, 2, device=DEV)]
    with pytest.raises(NotImplementedError, match="Sequential"):
        cfm_b200.action_matching_loss(net, *args)
