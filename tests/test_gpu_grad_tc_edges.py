"""The tensor-core gradient field (csrc/grad_tc.cu) at the edges of its scale logic: every layer's weight scale in its
own binade, the prepared gradient blob byte for byte, reverse chains that grow up to and past fp16's 65504, W3 at
every power of two the chain factor meets, rows at SELU's kink, Euler at every checkpoint on uneven spans, and the
cached plans across calls that change the weights, the activation, the direction or the solver.

Gates as tests/test_gpu_grad_tc.py: GRAD_K M per entry (grad_tc_oracle.bounds), rows near the kink counted apart."""
import math

import numpy as np
import pytest
import torch

import cnf_oracle as co
import grad_tc_cases as gc
import grad_tc_oracle as go
from test_gpu_grad_tc import KINK_SHARE, _field, _node, _state, _Tracked, every_row_against_float64

import cfm_b200
from cfm_b200 import _ffi

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
GRAD_K = go.GRAD_K


def _pair(dim, w, seed, factors=(1.0, 1.0, 1.0, 1.0), act="selu"):
    m = gc.scaled_action(dim, w, seed, factors, act)
    return m.to(DEV), {k: v.double().to(DEV) for k, v in _state(m).items()}


def _x(B, dim, seed):
    return torch.randn(B, dim, generator=torch.Generator().manual_seed(seed)).to(DEV)


# ---- per-layer scales -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("factors", gc.LAYER_SCALE_SETS)
@pytest.mark.parametrize("B,dim,w", gc.LAYER_SCALE_SHAPES)
def test_per_layer_scales_every_row_against_float64(B, dim, w, factors, act):
    """s_0..s_3 and 2^k pairwise distinct (test_grad_tc_host.py asserts it): an epilogue that undoes another layer's
    scale, or a chain factor taken from another layer, is off by a power of two."""
    m, state = _pair(dim, w, gc.LAYER_SCALE_SEED, factors, act)
    every_row_against_float64(m, state, _x(B, dim, 8), act, f"{B}x{dim}x{w} layers x{factors}")


# ---- the prepared blob ------------------------------------------------------------------------------------------------
_BLOB_CASES = [pytest.param(dim, w, (1.0,) * 4, id=f"{dim}x{w}") for _, dim, w in gc.FIELD_SHAPES] + \
    [pytest.param(dim, w, f, id=f"{dim}x{w}-x{f}") for _, dim, w in gc.LAYER_SCALE_SHAPES for f in gc.LAYER_SCALE_SETS]


@pytest.mark.parametrize("dim,w,factors", _BLOB_CASES)
def test_prepared_blob_byte_for_byte(dim, w, factors):
    m, state = _pair(dim, w, dim + w, factors)
    _, gblob = m._grad_prepared(torch.device(DEV))
    got = gblob.cpu().numpy()
    want, regions = go.grad_blob({k: v.cpu() for k, v in state.items()}, dim, w)
    assert got.size >= want.size
    _, (k, k0) = go.layer_scales({k: v.cpu() for k, v in state.items()}, dim)
    assert got[:8].view(np.float32).tolist() == [float(k), float(k0)]
    for name, off, n in regions:
        bad = np.flatnonzero(got[off:off + n] != want[off:off + n])
        assert bad.size == 0, (name, int(bad[0]), bad.size)


# ---- the range of the reverse chain -----------------------------------------------------------------------------------
@pytest.mark.parametrize("act,factors,frac", gc.RANGE_CASES)
def test_range_every_row_against_float64(act, factors, frac):
    """Chains that reach frac of 65504 under the W3-only chain factor: past 1 its saturating splits clamp unless the
    chain factor bounds the whole chain."""
    B, dim, w = gc.RANGE_SHAPE
    m, state = _pair(dim, w, 7, factors, act)
    every_row_against_float64(m, state, gc.range_input(B, dim).to(DEV), act, f"range {frac} x{factors}")


def _with_w3(m, w3):
    with torch.no_grad():
        m.net[6].weight.copy_(w3)
    return m


def test_w3_powers_of_two_scale_v_exactly():
    B, dim, w = gc.W3_SHAPE
    m, state = _pair(dim, w, 91, (20.0, 20.0, 20.0, 1.0), "selu")  # a chain factor below s_3 2^-7
    x = _x(B, dim, 92)
    v = every_row_against_float64(m, state, x, "selu", "W3 base")
    w3 = m.net[6].weight.detach().clone()
    for p in gc.W3_POWERS:
        got = _field(_with_w3(m, w3 * 2.0 ** p), x)
        assert torch.equal(got, v * 2.0 ** p), p


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_w3_past_the_scale_clamp(act):
    B, dim, w = gc.W3_SHAPE
    m, _ = _pair(dim, w, 93, act=act)
    w3 = m.net[6].weight.detach()
    _with_w3(m, w3 / w3.abs().max() * gc.W3_PAST_CLAMP)
    assert float(m.net[6].weight.abs().max()) == gc.W3_PAST_CLAMP
    state = {k: v.double() for k, v in _state(m).items()}
    every_row_against_float64(m, state, _x(B, dim, 94), act, "max|W3| 2^-110")


def test_zero_w3_gives_positive_zero_and_a_still_trajectory():
    """A zero-initialised last layer: v is +0 in every entry, and Euler and dopri5 return x0 at every checkpoint, in both
    directions."""
    B, dim, w = gc.W3_SHAPE
    m, _ = _pair(dim, w, 95)
    _with_w3(m, torch.zeros_like(m.net[6].weight))
    x = _x(B, dim, 96)
    v = _field(m, x)
    assert torch.equal(v.view(torch.int32), torch.zeros_like(v, dtype=torch.int32))
    for solver in ("euler", "dopri5"):
        for span in (torch.linspace(0, 1, 5), torch.linspace(1, 0, 5)):
            with torch.no_grad():
                traj = _node(m, solver=solver, atol=1e-4, rtol=1e-4).trajectory(x, span)
            assert traj.shape == (5, B, dim)
            assert torch.equal(traj, x[None].expand_as(traj)), (solver, float(span[0]))


# ---- rows at SELU's kink ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("biases", gc.KINK_BIASES)
def test_kink_rows_take_act_prime_at_zero(biases):
    """x = 0 rows at t = 0 with zero biases: pre-activations exactly 0, where torch's SELU' (elu_backward's x <= 0
    branch) is lambda alpha.  bounds() counts these rows as kink rows (|pre| <= eps P holds with P = 0), so they are
    checked here entry by entry."""
    B, dim, w = gc.KINK_SHAPE
    m, _ = _pair(dim, w, 97)
    with torch.no_grad():
        for li in (0, 2, 4):
            b = m.net[li].bias
            b[: (w if biases == "all" else w // 2)] = 0.0
    state = {k: v.double().to(DEV) for k, v in _state(m).items()}
    x = _x(B, dim, 98)
    zero = torch.arange(B, device=DEV) % 3 == 0
    x[zero] = 0.0
    pre0 = go._forward(state, 0.0, x.double(), "selu")[0][0]
    assert bool((pre0[zero][:, : w // 2] == 0).all())
    v = _field(m, x, t=0.0)
    ref = go.field(state, 0.0, x.double(), "selu")
    M, kink = go.bounds(state, 0.0, x.double(), "selu")
    assert bool(kink[zero].all())
    err = (v.double() - ref).abs()
    ratio = float((err[zero] / (GRAD_K * M[zero])).max())
    assert ratio <= 1.0, ratio
    others = ~zero & ~kink
    r2 = float((err[others] / (GRAD_K * M[others])).max())
    assert r2 <= 1.0, r2
    assert float((kink & ~zero).double().sum()) <= KINK_SHARE * B
    print(f"margins grad kink rows {biases} biases zero: {ratio:.3f} of the gate on {int(zero.sum())} x = 0 rows")


# ---- Euler at every checkpoint ----------------------------------------------------------------------------------------
_SPANS = [pytest.param(name, d, id=f"{name}-{d}") for name in gc.SPANS for d in ("forward", "reverse")]


@pytest.mark.parametrize("name,direction", _SPANS)
def test_euler_every_checkpoint_against_float64(name, direction):
    B, dim, w = gc.SPAN_SHAPE
    act = "silu"
    m, state = _pair(dim, w, 71, act=act)
    lip = go.lipschitz({k: v.cpu() for k, v in state.items()}, act, dim)
    if lip > 1.0:
        with torch.no_grad():
            m.net[6].weight.mul_(2.0 ** math.floor(math.log2(1.0 / lip)))
        state = {k: v.double().to(DEV) for k, v in _state(m).items()}
        lip = go.lipschitz({k: v.cpu() for k, v in state.items()}, act, dim)
    pts = gc.SPANS[name] if direction == "forward" else gc.SPANS[name][::-1]
    span = torch.tensor(pts, dtype=torch.float32)
    x = _x(B, dim, 72)
    with torch.no_grad():
        traj = _node(m, solver="euler").trajectory(x, span)
    field = _Tracked(state, act)
    ref = co.euler_any_direction(field, x.double(), span.double().to(DEV))
    assert traj.shape == ref.shape and torch.equal(traj[0], x)
    h = (span[1:] - span[:-1]).abs().double().tolist()
    bound = torch.zeros(B, dim, dtype=torch.float64, device=DEV)
    worst = 0.0
    for k, (M, _) in enumerate(field.seen):
        bound = bound + h[k] * GRAD_K * M + 2.0 ** -24 * ref[k + 1].abs()
        g = math.exp(lip * abs(pts[k + 1] - pts[0])) * bound
        err = (traj[k + 1].double() - ref[k + 1]).abs()
        r = float((err / g).max())
        assert r <= 1.0, (k + 1, r)
        worst = max(worst, r)
        if h[k] == 0.0:
            assert torch.equal(traj[k + 1], traj[k]), k + 1
    print(f"margins grad euler {name} {direction}: {worst:.3f} of the bound at the worst checkpoint")


# ---- plans across calls -----------------------------------------------------------------------------------------------
def _fresh(m, solver):
    f = cfm_b200.MLP(dim=m.dim, out_dim=1, w=m.w, time_varying=True).to(DEV)
    f.load_state_dict(m.state_dict())
    f.act = m.act
    return _node(f, solver=solver, atol=1e-4, rtol=1e-4)


def _run(node, x, span):
    with torch.no_grad():
        return node.trajectory(x, span)


def test_plans_follow_weights_activation_direction_and_solver():
    """One NeuralODE called again after an in-place Adam step, a switch of activation, a reversed span and a switch of
    solver gives, bit for bit, what a freshly built net and node with the same weights give."""
    B, dim, w = 257, 72, 136
    m, _ = _pair(dim, w, 99, act="selu")
    with torch.no_grad():
        m.net[6].weight.mul_(0.25)
    x = _x(B, dim, 100)
    fwd, rev = torch.linspace(0, 1, 6), torch.linspace(1, 0, 6)
    for solver in ("euler", "dopri5"):
        node = _node(m, solver=solver, atol=1e-4, rtol=1e-4)
        first = _run(node, x, fwd)
        assert torch.equal(first, _run(_fresh(m, solver), x, fwd)), solver
        opt = torch.optim.Adam(m.parameters(), lr=1e-3)
        m(torch.randn(64, dim + 1, device=DEV)).square().sum().backward()
        opt.step()
        opt.zero_grad()
        upd = _run(node, x, fwd)
        assert not torch.equal(upd, first)
        assert torch.equal(upd, _run(_fresh(m, solver), x, fwd)), (solver, "adam")
        m.act = _ffi.ACT_SILU
        silu = _run(node, x, fwd)
        assert torch.equal(silu, _run(_fresh(m, solver), x, fwd)), (solver, "silu")
        m.act = _ffi.ACT_SELU
        assert torch.equal(_run(node, x, fwd), upd), (solver, "selu again")
        back = _run(node, x, rev)
        assert torch.equal(back, _run(_fresh(m, solver), x, rev)), (solver, "reverse")
        assert torch.equal(_run(node, x, fwd), upd), (solver, "forward again")
    node = _node(m, solver="euler", atol=1e-4, rtol=1e-4)
    e = _run(node, x, fwd)
    node.solver = "dopri5"
    d = _run(node, x, fwd)
    assert torch.equal(d, _run(_fresh(m, "dopri5"), x, fwd))
    node.solver = "euler"
    assert torch.equal(_run(node, x, fwd), e)
