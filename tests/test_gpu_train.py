"""cfm_b200.flow_matching_loss on the device (mlp_train_kernel in csrc/train_small.cu: the regression loss of a small
MLP and all eight parameter gradients in one launch) against oracle/train.py, the notebook's lines in float64 on the
CPU with torch autograd.

SELU' jumps at 0, so a parameter gradient is discontinuous in the weights wherever a hidden pre-activation of some
row is 0.  Batches are drawn so that every row keeps every float64 pre-activation further than _KINK_REL of its
magnitude sum from the kink (as test_gpu_small_fields.py and test_gpu_action.py gate the rows they compare tightly);
at the 65 536 rows of the largest test about one row in the batch would otherwise sit within fp32 rounding of it."""
import math

import numpy as np
import pytest
import torch

import cfm_b200
from cfm_b200 import _ffi
import wide_train_oracle as wo
from oracle import train as ot

DEV = "cuda:0"
gpu = pytest.mark.gpu

SHAPES = [(1, 1), (2, 2), (5, 5), (8, 8), (2, 1), (8, 3)]  # (dim, out_dim)
BATCHES = [1, 2, 3, 255, 256, 257, 1000, 4096]
LOSS_REL, GRAD_REL = 2e-6, 2e-5  # GRAD_REL: every gradient tensor's error, of its max-abs
GRAD_ABS = 5e-7  # and every entry, of its own absolute scale (tests/wide_train_oracle.py); DESIGN.md 3.12
_KINK_REL = 1e-5


def _model(dim, out_dim, w, act, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m.to(DEV)


def _away_from_kink(mc, xt, t):
    """Rows whose float64 hidden pre-activations all stay further than _KINK_REL of their magnitude sum from 0."""
    with torch.no_grad():
        h = torch.cat([xt, t[:, None]], 1).double()
        keep = torch.ones(h.shape[0], dtype=torch.bool)
        for li in (0, 2, 4):
            W, b = mc.net[li].weight, mc.net[li].bias
            p = h @ W.T + b
            keep &= (p.abs() > _KINK_REL * (h.abs() @ W.abs().T + b.abs())).all(1)
            h = mc.net[li + 1](p)
    return keep


def _batch(m, B, seed, act="selu", row_scale=False):
    """Seeded (xt, t, ut, row_scale or None) on the CPU, B rows, every row away from SELU's kink for m's weights."""
    g = torch.Generator().manual_seed(seed)
    n = B + max(64, B // 50)  # about 0.4 % of the rows fall within _KINK_REL of the kink
    xt, t = torch.randn(n, m.dim, generator=g) * 1.5, torch.rand(n, generator=g)
    ut, s = torch.randn(n, m.out_dim, generator=g), torch.rand(n, generator=g) * 2.0
    if act == "selu":
        keep = _away_from_kink(ot.make_model(m.state_dict(), m.dim, m.out_dim, m.w, act), xt, t)
        assert int(keep.sum()) >= B
        xt, t, ut, s = xt[keep], t[keep], ut[keep], s[keep]
    return xt[:B].clone(), t[:B].clone(), ut[:B].clone(), (s[:B].clone() if row_scale else None)


def _device_loss_and_grads(m, xt, t, ut, s=None):
    m.zero_grad(set_to_none=True)
    loss = cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), ut.to(DEV), None if s is None else s.to(DEV))
    loss.backward()
    return loss.detach(), [p.grad.detach().clone() for p in m.parameters()]


def _gaps(m, act, xt, t, ut, s=None):
    """(loss error over its scale, worst gradient error over its entry's absolute scale, worst gradient error over
    the tensor's max-abs) against the float64 oracle.  The loss scale is the oracle loss plus mean(ut^2): the residual
    s*vt - ut is a difference, so its rounding error is relative to its terms, not to itself."""
    loss, grads = _device_loss_and_grads(m, xt, t, ut, s)
    assert loss.shape == () and loss.dtype == torch.float32 and loss.is_cuda
    rl, rg = ot.loss_and_grads(m.state_dict(), m.dim, m.out_dim, m.w, xt, t, ut, row_scale=s, act=act)
    scales = wo.grad_scales(m.state_dict(), m.dim, m.out_dim, m.w, xt, t, ut, row_scale=s, act=act)
    lgap = abs(loss.item() - rl.item()) / (rl.item() + ut.double().pow(2).mean().item())
    ggap = rgap = 0.0
    for p, g, r, sc in zip(m.parameters(), grads, rg, scales):
        assert g.shape == p.shape and torch.isfinite(g).all()
        err = (g.cpu().double() - r).abs()
        ggap = max(ggap, (err / sc.clamp_min(1e-300)).max().item())
        rgap = max(rgap, err.max().item() / r.abs().max().item())
    return lgap, ggap, rgap


# ---- every instantiation, every batch-size class -------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("dim,out_dim", SHAPES)
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("w", [32, 64])
def test_loss_and_gradients_match_the_float64_oracle(w, act, dim, out_dim):
    m = _model(dim, out_dim, w, act, seed=100 + w + dim)
    worst = [0.0, 0.0, 0.0]
    for B in BATCHES:
        gaps = _gaps(m, act, *_batch(m, B, seed=B, act=act))
        assert gaps[0] <= LOSS_REL and gaps[1] <= GRAD_ABS and gaps[2] <= GRAD_REL, (B, gaps)
        worst = [max(a, b) for a, b in zip(worst, gaps)]
    print(f"margins w={w} {act} dim={dim} out_dim={out_dim}: loss {worst[0]:.2e} grad/abs-scale {worst[1]:.2e} "
          f"grad/max-abs {worst[2]:.2e}")


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("w", [32, 64])
def test_row_scale_matches_the_oracle_including_zero_rows(w, act):
    m = _model(2, 2, w, act, seed=7)
    for B in (5, 300):
        xt, t, ut, s = _batch(m, B, seed=B, act=act, row_scale=True)
        s[::3] = 0.0  # a zero row adds ut^2 to the loss and nothing to any gradient
        lgap, ggap, rgap = _gaps(m, act, xt, t, ut, s)
        assert lgap <= LOSS_REL and ggap <= GRAD_ABS and rgap <= GRAD_REL, (B, lgap, ggap, rgap)
    # the SF2M score loss mean((lambda_t * st + eps)^2), written the notebook's way in float64
    eps = -ut
    mc = ot.make_model(m.state_dict(), 2, 2, w, act)
    st = mc(torch.cat([xt, t[:, None]], -1).double())
    ref = torch.mean((s.double()[:, None] * st + eps.double()) ** 2)
    with torch.no_grad():
        got = cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), (-eps).to(DEV), row_scale=s.to(DEV))
    assert abs(got.item() - ref.item()) <= LOSS_REL * (ref.item() + eps.pow(2).mean().item())


@gpu
def test_every_row_uses_its_own_time():
    """The time column of net.0.weight.grad is sum_r delta_0[r] * t_r: with per-row times it differs from what any
    shared scalar gives, and it must match the oracle on its own."""
    m = _model(2, 2, 64, "selu", seed=3)
    xt, t, ut, _ = _batch(m, 257, seed=1)
    t = torch.linspace(0.0, 1.0, 257)[torch.randperm(257, generator=torch.Generator().manual_seed(2))]
    keep = _away_from_kink(ot.make_model(m.state_dict(), 2, 2, 64), xt, t)
    xt, t, ut = xt[keep], t[keep], ut[keep]
    _, grads = _device_loss_and_grads(m, xt, t, ut)
    _, rg = ot.loss_and_grads(m.state_dict(), 2, 2, 64, xt, t, ut)
    col, ref = grads[0][:, -1].cpu().double(), rg[0][:, -1]
    assert (col - ref).abs().max().item() <= GRAD_REL * ref.abs().max().item()
    _, shared = ot.loss_and_grads(m.state_dict(), 2, 2, 64, xt, torch.full_like(t, t.mean().item()), ut)
    assert (col - shared[0][:, -1]).abs().max().item() > 1e-2 * ref.abs().max().item()


# ---- determinism ------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B", [256, 5000])
def test_repeated_calls_give_the_same_bits_and_no_grad_gives_the_same_loss(B):
    m = _model(2, 2, 64, "selu", seed=5)
    xt, t, ut, s = (v.to(DEV) for v in _batch(m, B, seed=9, row_scale=True))
    runs = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        loss = cfm_b200.flow_matching_loss(m, xt, t, ut, row_scale=s)
        loss.backward()
        runs.append((loss.detach().clone(), [p.grad.clone() for p in m.parameters()]))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
    with torch.no_grad():
        only = cfm_b200.flow_matching_loss(m, xt, t, ut, row_scale=s)
    assert not only.requires_grad and torch.equal(only, runs[0][0])


@gpu
def test_one_launch_per_call_and_none_in_backward():
    m = _model(2, 2, 64, "selu", seed=5)
    xt, t, ut, _ = (None if v is None else v.to(DEV) for v in _batch(m, 256, seed=9))
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()  # loads the kernel
    L = _ffi.lib()
    before = L.cfm_launch_count()
    loss = cfm_b200.flow_matching_loss(m, xt, t, ut)
    assert L.cfm_launch_count() - before == 1
    loss.backward()
    with torch.no_grad():
        cfm_b200.flow_matching_loss(m, xt, t, ut)
    assert L.cfm_launch_count() - before == 2


# ---- the autograd contract --------------------------------------------------------------------------------------------
@gpu
def test_gradients_accumulate_scale_and_follow_in_place_updates():
    m = _model(2, 2, 64, "selu", seed=6)
    xt, t, ut, _ = (None if v is None else v.to(DEV) for v in _batch(m, 256, seed=4))
    _, g1 = _device_loss_and_grads(m, xt, t, ut)
    # two backward() calls accumulate into .grad
    m.zero_grad(set_to_none=True)
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
    for p, g in zip(m.parameters(), g1):
        assert torch.equal(p.grad, g + g)
    # an upstream factor scales every gradient
    m.zero_grad(set_to_none=True)
    (0.5 * cfm_b200.flow_matching_loss(m, xt, t, ut)).backward()
    for p, g in zip(m.parameters(), g1):
        assert torch.equal(p.grad, 0.5 * g)
    # clipping and an optimizer work on the gradients, and the next call reads the updated weights
    opt = torch.optim.SGD(m.parameters(), lr=0.1)
    before = cfm_b200.flow_matching_loss(m, xt, t, ut)
    opt.zero_grad()
    before.backward()
    torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
    opt.step()
    after, ga = _device_loss_and_grads(m, xt, t, ut)
    assert after.item() < before.item()
    rl, rg = ot.loss_and_grads(m.state_dict(), 2, 2, 64, xt, t, ut)
    assert abs(after.item() - rl.item()) <= 1e-5 * rl.item()
    for g, r in zip(ga, rg):
        assert (g.cpu().double() - r).abs().max().item() <= 1e-4 * r.abs().max().item()
    # a parameter that does not require grad gets none; the others still do
    m.zero_grad(set_to_none=True)
    m.net[0].bias.requires_grad_(False)
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
    assert m.net[0].bias.grad is None and torch.equal(m.net[0].weight.grad, ga[0])


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
    """The tutorial's loop (8 gaussians -> moons, ConditionalFlowMatcher(sigma=0.1), batch 256) for 20 SGD steps
    through flow_matching_loss, against the same 20 steps in float64 on the same batches."""
    g = torch.Generator().manual_seed(0)
    m = _model(2, 2, 64, "selu", seed=1)
    mc = ot.make_model(m.state_dict(), 2, 2, 64)
    fm = cfm_b200.ConditionalFlowMatcher(sigma=0.1)
    opt, optc = torch.optim.SGD(m.parameters(), lr=1e-2), torch.optim.SGD(mc.parameters(), lr=1e-2)
    torch.manual_seed(2)
    for _ in range(20):
        x0, x1 = _eight_gaussians(256, g), _moons(256, g)
        t, xt, ut = fm.sample_location_and_conditional_flow(x0, x1)
        opt.zero_grad()
        cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), ut.to(DEV)).backward()
        opt.step()
        optc.zero_grad()
        ot.loss_of(mc, xt, t, ut).backward()
        optc.step()
    for p, r in zip(m.parameters(), mc.parameters()):
        assert (p.detach().cpu().double() - r.detach()).abs().max().item() <= 1e-4 * r.detach().abs().max().item()


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_large_batch_keeps_every_cta_busy(act):
    """65 536 rows: every CTA takes many tiles, and the fold adds as many partial vectors as the launch has CTAs."""
    m = _model(2, 2, 64, act, seed=8)
    lgap, ggap, rgap = _gaps(m, act, *_batch(m, 65536, seed=10, act=act, row_scale=True))
    print(f"margins B=65536 {act}: loss {lgap:.2e} grad/abs-scale {ggap:.2e} grad/max-abs {rgap:.2e}")
    assert lgap <= LOSS_REL and ggap <= GRAD_ABS and rgap <= GRAD_REL, (lgap, ggap, rgap)


@gpu
def test_strided_inputs_are_made_contiguous():
    m = _model(2, 1, 32, "silu", seed=9)
    xt, t, ut, _ = _batch(m, 64, seed=3, act="silu")
    wide = torch.randn(64, 6)
    wide[:, ::3], wide[:, 1], wide[:, 2] = xt, t, ut[:, 0]
    wd = wide.to(DEV)
    with torch.no_grad():
        a = cfm_b200.flow_matching_loss(m, wd[:, ::3], wd[:, 1], wd[:, 2:3])
        b = cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), ut.to(DEV))
    assert torch.equal(a, b)
    assert np.isfinite(a.item())
