"""The action-matching gradient field of wide scalar actions on the tensor cores
(``NeuralODE(torch_wrapper(GradModel(MLP(dim, out_dim=1, w, time_varying=True))))`` in the tensor-core class;
csrc/grad_tc.cu) against the float64 restatement of tests/grad_tc_oracle.py.

Error bounds.  One evaluation errs by at most GRAD_K M per entry, M the entry's magnitude chain
(grad_tc_oracle.bounds, which derives GRAD_K); rows with a SELU pre-activation within its own error of the kink at 0
leave that gate and are counted.  Trajectories add the per-evaluation bounds over the steps (|h| each; dopri5: the
largest stage-coefficient sum, 25, times the largest bound seen), times the growth exp(T Lip) with grad_tc_oracle's
Lipschitz bound, plus fp32 rounding of the state (2^-24 of it per step).  The trajectory nets have W3 scaled by a power
of two so that Lip <= 1."""
import math

import pytest
import torch

import cnf_oracle as co
import grad_tc_cases as gc
import grad_tc_oracle as go

import cfm_b200
from cfm_b200 import _ffi

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
GRAD_K = go.GRAD_K
KINK_SHARE = 0.05  # at most this share of rows may leave the tight gate (SELU only)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pair(dim, w, seed, act="selu", scale=1.0, lip_max=None):
    """(device action MLP, float64 state dict) with the same weights; ``scale`` multiplies W0..W2; with ``lip_max``, W3
    is scaled by a power of two so that the gradient field's Lipschitz bound is at most lip_max."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
    with torch.no_grad():
        for li in (0, 2, 4):
            m.net[li].weight.mul_(scale)
        if lip_max is not None:
            lip = go.lipschitz(_state(m), act, dim)
            if lip > lip_max:
                m.net[6].weight.mul_(2.0 ** math.floor(math.log2(lip_max / lip)))
    return m.to(DEV), {k: v.double().to(DEV) for k, v in _state(m).items()}


def _state(m):
    return {k: v.detach() for k, v in m.state_dict().items()}


def _field(m, x=None, t=0.3, pair=None, v=None, ws=None, B=None, t_dev=None):
    """One device evaluation through the C entry (fp32 x, split inside, or the operand pair ``pair`` = (hi, lo)) at
    time t, or at the time in the device tensor ``t_dev``."""
    L = _ffi.lib()
    B = B if B is not None else (x.shape[0] if x is not None else pair[0].shape[0])
    D = m.dim
    blob, gblob = m._grad_prepared(torch.device(DEV))
    ws = _ffi.workspace(L.cfm_grad_tc_workspace_bytes(B, D, m.w), DEV) if ws is None else ws
    v = torch.empty(B, D, device=DEV) if v is None else v
    tt = torch.tensor([t], dtype=torch.float32, device=DEV) if t_dev is None else t_dev
    hi, lo = pair if pair is not None else (None, None)
    _ffi.check(L.cfm_grad_tc_field_f32(
        _ffi.ptr(blob), _ffi.ptr(gblob), _ffi.ptr(x), _ffi.ptr(hi), _ffi.ptr(lo), B, D, m.w, m.act, _ffi.ptr(tt),
        _ffi.ptr(v), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(DEV)), "cfm_grad_tc_field_f32")
    return v


def every_row_against_float64(m, state, x, act, label, t=0.3):
    v = _field(m, x, t)
    ref = go.field(state, t, x.double(), act)
    M, kink = go.bounds(state, t, x.double(), act)
    err = (v.double() - ref).abs()
    ok = ~kink
    ratio = float((err[ok] / (GRAD_K * M[ok])).max())
    assert bool(torch.isfinite(v).all())
    assert ratio <= 1.0, (label, ratio)
    share = float(kink.double().mean())
    assert share <= KINK_SHARE, (label, share)
    print(f"margins grad field {label} {act}: {ratio:.3f} of the gate, {int(kink.sum())} kink rows of {x.shape[0]}")
    return v


# ---- one evaluation ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("B,dim,w", gc.FIELD_SHAPES)
def test_one_evaluation_every_row_against_float64(B, dim, w, act):
    """Also at the edges of tests/grad_tc_cases.py: partial chunks at N = dim and N = w, K tails, more tiles than CTAs,
    one-row last M tiles."""
    B = gc.batch(B, _sms())
    m, state = _pair(dim, w, dim + w, act)
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(B)).to(DEV)
    every_row_against_float64(m, state, x, act, f"{B}x{dim}x{w}")


@pytest.mark.parametrize("factor", gc.SCALE_FACTORS)
@pytest.mark.parametrize("B,dim,w", gc.SCALE_SHAPES)
def test_weight_scales(B, dim, w, factor):
    """W0..W2 scaled by 3, 0.2 and 11: the per-layer weight scales of both blobs and the growth of the reverse chain."""
    for act in ("selu", "silu"):
        m, state = _pair(dim, w, 7, act, scale=factor)
        x = torch.randn(B, dim, generator=torch.Generator().manual_seed(8)).to(DEV)
        every_row_against_float64(m, state, x, act, f"{B}x{dim}x{w} W0..W2 x{factor}")


# ---- bit for bit ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,dim,w", [gc.OFFSET_SHAPE, (256, 784, 256)])
def test_bits(B, dim, w):
    m, _ = _pair(dim, w, 51, "silu")
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(52)).to(DEV)
    v = _field(m, x)
    # W3 scaled by a power of two scales v by the same power, exactly; b3 does not enter
    with torch.no_grad():
        w3 = m.net[6].weight.clone()
        for p in (-12, 6):
            m.net[6].weight.copy_(w3 * 2.0 ** p)
            assert torch.equal(_field(m, x), v * 2.0 ** p), p
        m.net[6].weight.copy_(w3)
        m.net[6].bias.fill_(123.25)
    assert torch.equal(_field(m, x), v)
    # fp32 x and its split pair
    hi = x.half()
    lo = ((x - hi.float()) * 2048).half()
    assert torch.equal(_field(m, pair=(hi, lo)), v)
    # v written 1, 2 or 3 floats into a larger buffer
    for off in gc.V_OFFSETS:
        buf = torch.full((B * dim + 8,), float("nan"), device=DEV)
        out = buf[off:off + B * dim].view(B, dim)
        _field(m, x, v=out)
        assert torch.equal(out, v), off
        assert bool(buf[:off].isnan().all()) and bool(buf[off + B * dim:].isnan().all())
    # a NaN-filled or left-over workspace, and a second call
    L = _ffi.lib()
    ws = _ffi.workspace(L.cfm_grad_tc_workspace_bytes(B, dim, w), DEV)
    ws.view(torch.uint8).fill_(0xFF)  # NaN in every fp32 and fp16 slot
    assert torch.equal(_field(m, x, ws=ws), v)
    _field(m, torch.randn_like(x) * 5, ws=ws)
    assert torch.equal(_field(m, x, ws=ws), v)
    assert torch.equal(_field(m, x, ws=ws), v)
    # rows past B stay untouched
    big = torch.full((B + 5, dim), -7.5, device=DEV)
    _field(m, x, v=big[:B])
    assert torch.equal(big[:B], v) and bool((big[B:] == -7.5).all())
    # a row's value does not depend on the batch size
    assert torch.equal(_field(m, x[:128].contiguous()), v[:128])
    assert torch.equal(_field(m, x[B - 129:].contiguous()), v[B - 129:])
    # graph replay equals eager enqueue
    out = torch.empty_like(v)
    ws2 = _ffi.workspace(L.cfm_grad_tc_workspace_bytes(B, dim, w), DEV)
    t_dev = torch.tensor([0.3], device=DEV)
    _field(m, x, v=out, ws=ws2, t_dev=t_dev)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _field(m, x, v=out, ws=ws2, t_dev=t_dev)
    out.zero_()
    g.replay()
    assert torch.equal(out, v)
    # an in-place Adam update: the result of a freshly built net with those weights
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    loss = m(torch.randn(64, dim + 1, device=DEV)).square().sum()
    loss.backward()
    opt.step()
    upd = _field(m, x)
    fresh = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True).to(DEV)
    fresh.load_state_dict(m.state_dict())
    fresh.act = m.act
    assert torch.equal(upd, _field(fresh, x)) and not torch.equal(upd, v)


# ---- trajectories -----------------------------------------------------------------------------------------------------
def _node(m, **kw):
    return cfm_b200.NeuralODE(cfm_b200.torch_wrapper(cfm_b200.GradModel(m)), **kw)


class _Tracked:
    """The float64 field with the scale M of every evaluation."""

    def __init__(self, state, act):
        self.state, self.act, self.seen = state, act, []

    def __call__(self, t, x):
        M, kink = go.bounds(self.state, float(t), x, self.act)
        self.seen.append((M, kink))
        return go.field(self.state, float(t), x, self.act)


def _positive_selu_action(dim, w, seed):
    """An action whose hidden pre-activations are all positive for |x| <= ~10, t in [0, 1]: SELU is linear there, s
    is affine in x and its gradient c is constant."""
    g = torch.Generator().manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True)
    with torch.no_grad():
        m.net[0].weight.copy_(0.05 * torch.randn(w, dim + 1, generator=g))
        m.net[0].bias.copy_(3.0 + torch.rand(w, generator=g))
        for li in (2, 4):
            m.net[li].weight.copy_(0.05 * torch.rand(w, w, generator=g))
            m.net[li].bias.copy_(0.5 + torch.rand(w, generator=g))
        m.net[6].weight.copy_(0.1 * torch.randn(1, w, generator=g))
        m.net[6].bias.copy_(0.1 * torch.randn(1, generator=g))
    return m.to(DEV), {k: v.double().to(DEV) for k, v in _state(m).items()}


@pytest.mark.parametrize("solver", ["euler", "dopri5"])
def test_affine_action_gives_a_straight_trajectory(solver):
    B, dim, w = 256, 64, 128
    m, state = _positive_selu_action(dim, w, 61)
    W = [state[f"net.{li}.weight"] for li in (0, 2, 4, 6)]
    c = go.SELU_L ** 3 * (W[3] @ W[2] @ W[1] @ W[0][:, :dim])[0]  # the constant gradient
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(62)).to(DEV)
    for span in (torch.linspace(0, 1, 11), torch.linspace(1, 0, 11)):
        node = _node(m, solver=solver, atol=1e-4, rtol=1e-4)
        with torch.no_grad():
            traj = node.trajectory(x, span)
        ref = x.double()[None] + (span.double().to(DEV) - float(span[0]))[:, None, None] * c
        for t in span.tolist():
            for pre, _ in go._forward(state, t, ref[0] + (t - float(span[0])) * c, "selu"):
                assert float(pre.min()) > 0
        M, kink = go.bounds(state, 0.5, x.double(), "selu")
        assert not bool(kink.any())
        steps = node.stats["accepted"] + node.stats["rejected"]
        bound = 2 * GRAD_K * M[None] + (steps + 10) * 2.0**-23 * ref.abs().amax(0)[None]
        err = (traj.double() - ref).abs()
        assert bool((err <= bound).all()), (solver, float((err / bound).max()))
        print(f"margins affine {solver} {float(span[0])}->{float(span[-1])}: {float((err / bound).max()):.3f}")


_EULER = [pytest.param(d, s, id=f"{d}-{s[0]}x{s[1]}x{s[2]}") for s in gc.EULER_SHAPES for d in ("forward", "reverse")]


@pytest.mark.parametrize("direction,shape", _EULER)
def test_euler_trajectory_against_float64(direction, shape):
    B, dim, w = shape
    act = "silu"
    m, state = _pair(dim, w, 71, act, lip_max=1.0)
    lip = go.lipschitz({k: v.cpu() for k, v in state.items()}, act, dim)
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(72)).to(DEV)
    span = torch.linspace(0, 1, 100) if direction == "forward" else torch.linspace(1, 0, 100)
    steps = span.numel() - 1
    node = _node(m, solver="euler")
    with torch.no_grad():
        traj = node.trajectory(x, span)
    assert traj.shape == (steps + 1, B, dim) and node.stats["nfe"] == steps and node.stats["graph"]
    field = _Tracked(state, act)
    ref = co.euler_any_direction(field, x.double(), span.double().to(DEV))
    h = (span[1:] - span[:-1]).abs().double().tolist()
    bound = torch.zeros(B, dim, dtype=torch.float64, device=DEV)
    for k, (M, _) in enumerate(field.seen):
        bound = bound + h[k] * GRAD_K * M + 2.0**-24 * ref[k + 1].abs()
    bound = math.exp(lip) * bound
    err = (traj[-1].double() - ref[-1]).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    print(f"margins grad euler {B}x{dim}x{w} {direction}: {float((err / bound).max()):.3f} of the gate (Lip {lip:.2f})")
    # eager enqueue gives the bits of the graph replay, in 1 + 7 launches per step
    node.use_cuda_graph = False
    L = _ffi.lib()
    c0 = L.cfm_launch_count()
    with torch.no_grad():
        eager = node.trajectory(x, span)
    assert L.cfm_launch_count() - c0 == 1 + 7 * steps
    assert torch.equal(eager, traj) and not node.stats["graph"]


@pytest.mark.parametrize("direction", ["forward", "reverse"])
@pytest.mark.parametrize("B,dim,w", gc.DOPRI5_CASES)
def test_dopri5_takes_the_oracle_step_sequence(B, dim, w, direction):
    act = "silu"
    m, state = _pair(dim, w, 81, act, lip_max=1.0)
    lip = go.lipschitz({k: v.cpu() for k, v in state.items()}, act, dim)
    x = torch.randn(B, dim, generator=torch.Generator().manual_seed(82)).to(DEV)
    span = torch.linspace(0, 1, 3) if direction == "forward" else torch.linspace(1, 0, 3)
    node = _node(m, solver="dopri5", atol=1e-4, rtol=1e-4)
    with torch.no_grad():
        traj = node.trajectory(x, span)
    field = _Tracked(state, act)
    ref, st = co.dopri5_any_direction(field, x.double(), span.double().to(DEV), 1e-4, 1e-4)
    assert (node.stats["nfe"], node.stats["accepted"], node.stats["rejected"]) == \
        (st["nfe"], st["accepted"], st["rejected"])
    assert node.stats["graph"]
    Mm = torch.stack([M for M, _ in field.seen]).amax(0)
    steps = st["accepted"] + st["rejected"]
    bound = math.exp(lip) * (25 * GRAD_K * Mm + steps * 2.0**-23 * ref.abs().amax(0))
    err = (traj.double() - ref).abs()
    assert bool((err <= bound).all()), float((err / bound).max())
    print(f"margins grad dopri5 {B}x{dim}x{w} {direction}: {float((err / bound).max()):.3f} of the gate, "
          f"nfe {st['nfe']}")
    with torch.no_grad():
        assert torch.equal(node.trajectory(x, span), traj)  # the captured step and init replay the same bits
        node.use_cuda_graph = False
        node._plans.clear()
        assert torch.equal(node.trajectory(x, span), traj)


def test_refusals_launch_nothing():
    L = _ffi.lib()
    span = torch.linspace(0, 1, 3)
    before = L.cfm_launch_count()
    for B, dim, w in [(127, 64, 128), (1024, 64, 36), (1024, 60, 128), (1024, 16, 64)]:
        m = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True).to(DEV)
        for solver in ("euler", "dopri5"):
            with pytest.raises(NotImplementedError, match="no gradient-field kernel.*tensor-core class"):
                _node(m, solver=solver).trajectory(torch.zeros(B, dim, device=DEV), span)
    assert L.cfm_launch_count() == before
    node = _node(cfm_b200.MLP(dim=64, out_dim=1, w=128, time_varying=True).to(DEV), solver="dopri5")
    node.lockstep = True
    with pytest.raises(NotImplementedError, match="lock-step"):
        node.trajectory(torch.zeros(256, 64, device=DEV), span)
    with pytest.raises(NotImplementedError, match="out_dim=2"):
        _node(cfm_b200.MLP(dim=64, out_dim=2, w=128, time_varying=True).to(DEV)).trajectory(
            torch.zeros(256, 64, device=DEV), span)
