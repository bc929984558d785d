"""Hutchinson log-likelihood of wide MLP flows on the tensor cores (``cnf_wrapper(mlp, "hutch_gaussian" |
"hutch_rademacher")`` through ``NeuralODE``; csrc/cnf_tc.cu) against the float64 restatement driven by the same probes
(tests/cnf_tc_oracle.py).

Error bounds.  DESIGN 3.0-3.1: an fp16x3 GEMM output errs by at most EPS_GEMM = 1e-6 of its magnitude sum |a| |b| (the
H100 measures <= 5e-7 at K <= 1024; the operand split adds 2^-22 relative, or 2^-36 absolute for entries below fp16's
normal range).  Per evaluation and row (cnf_tc_oracle.magnitudes):
  * div: 4 tangent GEMMs, each within EPS_GEMM of its stage of the magnitude chain S, the act' perturbation carried in
    S itself, the device probe's fp32 transcendental (<= 2^-21 relative per entry, entering twice) and the fp32
    products: at most (4 + 1 + 1) EPS_GEMM S; gated at DIV_K = 10 EPS_GEMM S.
  * f: 4 primal GEMMs whose relative errors reach the output through the |W| |act'| chain: gated at
    F_K = 16 EPS_GEMM F, F = |W3| |a_3| + |b3|.
Trajectories add the per-evaluation bounds over the steps (|h| each; dopri5: the largest stage-coefficient sum, 25,
times the largest bound seen), times the growth exp(T Lip) with Lip = prod ||W_l||_2 max|act'|^3 of the net, plus
fp32 rounding of the state (2^-24 of it per step).  The test nets are scaled to Lip < 2."""
import math

import numpy as np
import pytest
import torch

import cnf_oracle as co
import cnf_tc_oracle as ho
import tc_sampler_cases as tc
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
EPS_GEMM, DIV_K, F_K = ho.EPS_GEMM, ho.DIV_K, ho.F_K
ESTS = ("hutch_gaussian", "hutch_rademacher")
EST_CODE = {"hutch_gaussian": _ffi.HUTCH_GAUSSIAN, "hutch_rademacher": _ffi.HUTCH_RADEMACHER}


def _pair(dim, w, seed, act="selu", scale=1.0):
    """(device MLP, float64 device oracle MLP) with the same weights; ``scale`` multiplies W1..W3."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
    with torch.no_grad():
        for li in (2, 4, 6):
            m.net[li].weight.mul_(scale)
    mc = vf.make_mlp(dim, w=w, time_varying=True, dtype=torch.float64)
    mc.load_state_dict({k: v.double() for k, v in m.state_dict().items()})
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            mc.net[k] = torch.nn.SiLU()
    return m.to(DEV), mc.to(DEV)


def _state(mc):
    return {k: v.detach() for k, v in mc.state_dict().items()}


def _field(m, x, t, est, seed, n, pair=None, f=None, div=None, ws=None):
    """One device evaluation through the C entry (fp32 x, split inside, or the operand pair ``pair`` = (hi, lo) with
    x None); the ordinal is passed as *ord + 2.  ``f``, ``div`` and ``ws`` default to fresh buffers of x's batch."""
    L = _ffi.lib()
    B, D = x.shape if x is not None else pair[0].shape
    blob = m._prepared(True, torch.device(DEV))
    ws = _ffi.workspace(L.cfm_cnf_tc_workspace_bytes(B, D, m.w), DEV) if ws is None else ws
    f = torch.empty(B, D, device=DEV) if f is None else f
    div = torch.empty(B, device=DEV) if div is None else div
    tt = torch.tensor([t], dtype=torch.float32, device=DEV)
    sd = torch.tensor([seed], dtype=torch.int64, device=DEV)
    nn = torch.tensor([n - 2], dtype=torch.int32, device=DEV)
    hi, lo = pair if pair is not None else (None, None)
    _ffi.check(L.cfm_cnf_tc_field_f32(
        _ffi.ptr(blob), _ffi.ptr(x), _ffi.ptr(hi), _ffi.ptr(lo), B, D, m.w, m.act, EST_CODE[est], _ffi.ptr(tt),
        _ffi.ptr(sd), _ffi.ptr(nn), 2, _ffi.ptr(f), _ffi.ptr(div), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(DEV)),
        "cfm_cnf_tc_field_f32")
    return f, div


# ---- one evaluation ---------------------------------------------------------------------------------------------------
def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def every_row_against_float64(m, mc, x, act, label):
    """Both estimators at one (t, x): div within DIV_K S and f within F_K F of the float64 field on every row; f
    bit-identical to the per-layer forward where m.vector_field takes it (w != 256 or dim < 64), within F_K F of the
    fused forward elsewhere.  Prints the worst ratio to each gate."""
    B, dim = x.shape
    t = 0.3
    with torch.no_grad():
        y = m.vector_field(t, x)
    per_layer = not (m.w == 256 and dim >= 64)
    for k, est in enumerate(ESTS):
        seed, n = 1234 + k, 9
        f, div = _field(m, x, t, est, seed, n)
        eps = torch.from_numpy(ho.device_probes(est, seed, n, np.arange(B), dim)).to(DEV)
        ref_f, ref = ho.hutch_div(mc, torch.tensor(t, dtype=torch.float64), x.double(), eps)
        F, S = ho.magnitudes(_state(mc), t, x.double(), eps, act, EPS_GEMM)
        err = (div.double() - ref).abs()
        assert bool((err <= DIV_K * S).all()), (est, float((err / S).max()))
        assert bool(((f.double() - ref_f).abs() <= F_K * F).all()), (est, float(((f.double() - ref_f).abs() / F).max()))
        print(f"margins field {label} {act} {est}: div {float((err / (DIV_K * S)).max()):.2e} "
              f"f {float(((f.double() - ref_f).abs() / (F_K * F)).max()):.3f} of the gate")
        if per_layer:  # the primal epilogue is the per-layer forward's: the same bits
            assert torch.equal(f, y)
        else:  # the fused forward
            assert float((f - y).abs().max()) <= 1e-5 * float(y.abs().max())
            assert bool(((f.double() - y.double()).abs() <= F_K * F).all())


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("B,dim,w", [(256, 784, 256), (300, 64, 128), (129, 32, 32)] + tc.FIELD_SHAPES)
def test_one_evaluation_every_row_against_float64(B, dim, w, act):
    """Also at the edges of tests/tc_sampler_cases.py: partial hidden and output chunks, 8-column N tiles, K tails,
    more tiles than CTAs in every GEMM, one-row last M tiles, 1 to 25 fold chunks."""
    B = tc.batch(B, _sms())
    m, mc = _pair(dim, w, dim + w, act)
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(B)).to(DEV)
    every_row_against_float64(m, mc, x, act, f"{B}x{dim}x{w}")


@pytest.mark.parametrize("est", ESTS)
def test_mean_over_64_seeds_is_the_exact_trace(est):
    """Unbiasedness at one evaluation: the mean over 64 fixed seeds lies within 5 standard errors of the float64 trace
    (jacrev) on each of 4 rows; the standard error is the oracle's own spread over the same probes."""
    B, dim, w = 128, 32, 32
    m, mc = _pair(dim, w, 5)
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(6)).to(DEV)
    t = torch.tensor(0.6, dtype=torch.float64, device=DEV)
    rows = np.arange(4)
    dev, orc = [], []
    for s in range(64):
        dev.append(_field(m, x, 0.6, est, 1000 + s, 0)[1][:4].double())
        eps = torch.from_numpy(ho.device_probes(est, 1000 + s, 0, rows, dim)).to(DEV)
        orc.append(ho.hutch_div(mc, t, x[:4].double(), eps)[1])
    dev, orc = torch.stack(dev), torch.stack(orc)
    exact = co.cnf_field(mc)(t, torch.cat([x[:4].double(), torch.zeros(4, 1, device=DEV, dtype=torch.float64)], 1))
    se = orc.std(0) / 8
    assert bool(((dev.mean(0) - exact[:, -1]).abs() <= 5 * se).all()), ((dev.mean(0) - exact[:, -1]) / se).tolist()


# ---- trajectories -----------------------------------------------------------------------------------------------------
class _Tracked:
    """The oracle field with its per-evaluation magnitudes (F, S) per row."""

    def __init__(self, mc, est, seed, B, D, act):
        self.mc, self.act, self.seen = mc, act, []
        self.probes = ho.Probes(est, seed, B, D, device=DEV)
        self.state = _state(mc)

    def __call__(self, t, z):
        x = z[:, :-1]
        eps = self.probes.next().to(x)
        f, div = ho.hutch_div(self.mc, t, x, eps)
        F, S = ho.magnitudes(self.state, float(t), x, eps, self.act, EPS_GEMM)
        self.seen.append((float(t), F, S))
        return torch.cat([f, div[:, None]], 1)


def _seeded(node, z, span, seed=77):
    torch.manual_seed(seed)
    with torch.no_grad():
        return node.trajectory(z, span)


def _seed_of(seed=77):
    torch.manual_seed(seed)
    return int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))


# (direction, shape): the first shape keeps the test's original ids
_EULER = [pytest.param(d, s, id=d if s == tc.EULER_SHAPES[0] else f"{d}-{s[0]}x{s[1]}x{s[2]}")
          for s in tc.EULER_SHAPES for d in ("forward", "reverse")]


@pytest.mark.parametrize("direction,shape", _EULER)
@pytest.mark.parametrize("est", ESTS)
def test_euler_trajectory_against_float64_and_plain_wide_euler(est, direction, shape):
    B, dim, w, steps = shape
    act = "selu"
    m, mc = _pair(dim, w, 11, act, scale=0.5)
    lip = ho.lipschitz(mc, act)
    assert lip < 2
    z = torch.cat([torch.randn(B, dim, generator=torch.Generator().manual_seed(12)), torch.zeros(B, 1)], 1).to(DEV)
    span = torch.linspace(0, 1, steps + 1) if direction == "forward" else torch.linspace(1, 0, steps + 1)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator=est), solver="euler")
    traj = _seeded(node, z, span)
    assert traj.shape == (steps + 1, B, dim + 1) and node.stats["nfe"] == steps and node.stats["graph"]
    field = _Tracked(mc, est, _seed_of(), B, dim, act)
    ref = co.euler_any_direction(field, z.double(), span.double().to(DEV))
    assert field.probes.n == steps
    h = (span[1:] - span[:-1]).abs().double().tolist()
    grow = math.exp(lip)
    bx = torch.zeros(B, dim, dtype=torch.float64, device=DEV)
    bl = torch.zeros(B, dtype=torch.float64, device=DEV)
    for k, (_, F, S) in enumerate(field.seen):
        bx = bx + h[k] * F_K * F + 2.0**-24 * ref[k + 1, :, :dim].abs()
        bl = bl + h[k] * DIV_K * S + 2.0**-24 * ref[k + 1, :, dim].abs()
    bx, bl = grow * bx, 2 * grow * bl  # 2: the x error's feed-through into div, second order in EPS_GEMM
    err = (traj.double() - ref).abs()
    assert bool((err[-1, :, :dim] <= bx).all()), float((err[-1, :, :dim] / bx).max())
    assert bool((err[-1, :, dim] <= bl).all()), float((err[-1, :, dim] / bl).max())
    print(f"margins euler {B}x{dim}x{w} {est} {direction}: x {float((err[-1, :, :dim] / bx).max()):.3f} "
          f"ll {float((err[-1, :, dim] / bl).max()):.2e} of the gate")
    # eager enqueue gives the bits of the graph replay
    node.use_cuda_graph = False
    assert torch.equal(_seeded(node, z, span), traj)
    if w == 256 and dim >= 64:  # the plain wide Euler takes the fused forward there
        return
    # the x columns are those of the plain wide Euler trajectory on a per-layer shape, bit for bit
    plain = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="euler")
    with torch.no_grad():
        px = plain.trajectory(z[:, :dim].contiguous(), span)
    assert torch.equal(traj[..., :dim], px)


# (direction, B): B (D + 1) = 1, 2, 3 mod 4 puts the stage outputs f = k[i] at every 4-byte offset mod 16; the first
# batch keeps the test's original ids
_DOPRI5 = [pytest.param(d, B, id=d if B == tc.DOPRI5_BATCHES[0] else f"{d}-B{B}")
           for B in tc.DOPRI5_BATCHES for d in ("forward", "reverse")]


@pytest.mark.parametrize("direction,B", _DOPRI5)
def test_dopri5_takes_the_oracle_step_sequence(direction, B):
    (dim, w), act, est = tc.DOPRI5_SHAPE, "silu", "hutch_gaussian"
    m, mc = _pair(dim, w, 21, act, scale=0.5)
    lip = ho.lipschitz(mc, act)
    z = torch.cat([torch.randn(B, dim, generator=torch.Generator().manual_seed(22)), torch.zeros(B, 1)], 1).to(DEV)
    span = torch.linspace(0, 1, 3) if direction == "forward" else torch.linspace(1, 0, 3)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator=est), solver="dopri5", atol=1e-5,
                              rtol=1e-5)
    traj = _seeded(node, z, span)
    field = _Tracked(mc, est, _seed_of(), B, dim, act)
    ref, st = co.dopri5_any_direction(field, z.double(), span.double().to(DEV), 1e-5, 1e-5)
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert field.probes.n == st["nfe"] and st["accepted"] >= 2
    Fm = torch.stack([F for _, F, _ in field.seen]).amax(0)
    Sm = torch.stack([S for _, _, S in field.seen]).amax(0)
    steps = st["accepted"] + st["rejected"]
    bx = math.exp(lip) * (25 * F_K * Fm + steps * 2.0**-23 * ref[:, :, :dim].abs().amax(0))
    bl = 2 * math.exp(lip) * (25 * DIV_K * Sm + steps * 2.0**-23 * ref[:, :, dim].abs().amax(0))
    err = (traj.double() - ref).abs()
    assert bool((err[..., :dim] <= bx).all()), float((err[..., :dim] / bx).max())
    assert bool((err[..., dim] <= bl).all()), float((err[..., dim] / bl).max())
    print(f"margins dopri5 B={B} {direction}: x {float((err[..., :dim] / bx).max()):.3f} "
          f"ll {float((err[..., dim] / bl).max()):.2e} of the gate")
    assert torch.equal(_seeded(node, z, span), traj)  # the captured step and init replay the same bits
    node.use_cuda_graph = False
    node._plans.clear()
    assert torch.equal(_seeded(node, z, span), traj)


# ---- reproducibility --------------------------------------------------------------------------------------------------
def test_rows_seeds_graphs_launches_and_in_place_weights():
    B, dim, w = 300, 64, 128
    m, _ = _pair(dim, w, 31, scale=0.5)
    z = torch.cat([torch.randn(B, dim, generator=torch.Generator().manual_seed(32)), torch.zeros(B, 1)], 1).to(DEV)
    span = torch.linspace(1, 0, 6)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator="hutch_rademacher"), solver="euler")
    a = _seeded(node, z, span)
    # a row's result does not depend on the batch it is in
    assert torch.equal(_seeded(node, z[:256].contiguous(), span), a[:, :256])
    # torch.manual_seed reproduces the trajectory; another seed draws other probes
    assert torch.equal(_seeded(node, z, span), a)
    other = _seeded(node, z, span, seed=78)
    assert torch.equal(other[..., :dim], a[..., :dim]) and not torch.equal(other[..., dim], a[..., dim])
    # eager enqueue gives the bits of the graph replay, in 1 + 11 launches per step
    node.use_cuda_graph = False
    L = _ffi.lib()
    c0 = L.cfm_launch_count()
    assert torch.equal(_seeded(node, z, span), a)
    assert L.cfm_launch_count() - c0 == 1 + 11 * (span.numel() - 1)
    node.use_cuda_graph = True
    # weights updated in place: the trajectory of a fresh net with those weights
    with torch.no_grad():
        m.net[2].weight.mul_(1.25)
        m.net[0].bias.add_(0.1)
    upd = _seeded(node, z, span)
    fresh = cfm_b200.MLP(dim=dim, w=w, time_varying=True).to(DEV)
    fresh.load_state_dict(m.state_dict())
    node2 = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(fresh, likelihood_estimator="hutch_rademacher"), solver="euler")
    assert torch.equal(upd, _seeded(node2, z, span)) and not torch.equal(upd, a)


def test_autograd_forward_has_the_same_bits_and_backward_raises():
    B, dim, w = 256, 32, 64
    m, _ = _pair(dim, w, 41)
    z = torch.cat([torch.randn(B, dim, generator=torch.Generator().manual_seed(42)), torch.zeros(B, 1)], 1).to(DEV)
    for solver in ("euler", "dopri5"):
        span = torch.linspace(1, 0, 4)
        node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator="hutch_gaussian"), solver=solver)
        ref = _seeded(node, z, span)
        zg = z.clone().requires_grad_(True)
        torch.manual_seed(77)
        traj = node.trajectory(zg, span)
        assert traj.requires_grad and torch.equal(traj.detach(), ref)
        with pytest.raises(NotImplementedError, match="Hutchinson-estimator trajectory"):
            traj.sum().backward()


def test_refusals():
    wide = cfm_b200.MLP(dim=64, w=128, time_varying=True).to(DEV)
    z = torch.zeros(256, 65, device=DEV)
    span = torch.linspace(1, 0, 3)
    with pytest.raises(NotImplementedError, match="no exact-likelihood kernel.*'hutch_gaussian' or 'hutch_rademacher'"):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(wide), solver="euler").trajectory(z, span)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(wide, likelihood_estimator="hutch_gaussian"), solver="dopri5")
    node.lockstep = True
    with pytest.raises(NotImplementedError, match="lock-step"):
        node.trajectory(z, span)
    small = cfm_b200.MLP(dim=2, w=256, time_varying=True).to(DEV)
    for est in ESTS:
        with pytest.raises(NotImplementedError, match="Hutchinson"):
            cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(small, likelihood_estimator=est),
                               solver="euler").trajectory(torch.zeros(256, 3, device=DEV), span)
    odd = cfm_b200.MLP(dim=64, out_dim=32, w=128, time_varying=True).to(DEV)
    with pytest.raises(NotImplementedError, match="out_dim=32"):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(odd, likelihood_estimator="hutch_gaussian"),
                           solver="euler").trajectory(z, span)
    with pytest.raises(ValueError):
        cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(wide, likelihood_estimator="hutch_gaussian"),
                           solver="euler").trajectory(torch.zeros(256, 64, device=DEV), span)
