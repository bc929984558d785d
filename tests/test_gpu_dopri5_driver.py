"""The multi-kernel dopri5 driver (csrc/rk.cu + cfm_b200/ode.py::_dopri5/_enqueue_step/_enqueue_init/_plan/_euler), the
one every model too large for the one-launch kernel goes through, on every path it takes.

A. Whole trajectories against the torchdyn restatement (oracle/vector_field.py): same (nfe, accepted, rejected) and
   EVERY checkpoint within 1e-4 max(1, |ref|) of the fp32 oracle, the last state within 5e-3 of a float64 run at 1e-9.
   The step sequence is a discrete function of fp32 error ratios, so every case asserts that the oracle's recorded
   ratios stay 1e-3 away from 1: with that margin a different count is a defect, not rounding.  Three model classes
   put all three MLP back ends under the driver: SIMT with element counts that are not multiples of 4 (the scalar path
   of every elementwise kernel), the per-layer tensor-core MLP, and the fused w = 256 kernel with its split operands.
   Decreasing spans, Euler, rejected (and rejected clipped) steps, long / dense / non-uniform spans, the burst
   settings, plan reuse with something changed, graph against eager stepping, higher-rank inputs.
B. The kernels one by one through the C ABI against float64 (and, for the one-thread controller, against an fp32
   restatement of torchdyn's loop body acting on the same state struct): stage inputs at every stage and at sizes on
   both the 128-bit and the scalar path, the error norm, each branch of cfm_rk_control, the commit, the Hairer initial
   step, zero and constant fields end to end, and the argument refusals.

Every test forces the driver under test (``use_fused_small = False``) and asserts the one-launch kernel did not run."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

import cnf_oracle as co
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
f32 = np.float32

# (dim, w, B, act): SIMT with 3 B % 4 == 3 and 2 B % 4 == 2 (w = 50 has no one-launch kernel either), the per-layer
# tensor-core MLP, the fused w = 256 kernel at an aligned and a ragged last K chunk
SIMT3, SIMT2, TC128, FUSED64, FUSED200 = ((3, 64, 1001, "selu"), (2, 50, 1001, "silu"), (64, 128, 1500, "silu"),
                                          (64, 256, 1000, "selu"), (200, 256, 300, "silu"))
CLASSES = [SIMT3, SIMT2, TC128, FUSED64, FUSED200]
_ids = lambda c: f"{c[0]}-{c[1]}-{c[2]}-{c[3]}"  # noqa: E731

REVERSE_SPANS = {"1to0x2": torch.linspace(1, 0, 2), "1to0x9": torch.linspace(1, 0, 9),
                 "nonuniform": torch.tensor([0.875, 0.375, 0.125])}  # (binary fractions: t + dt lands on them exactly)
SPANS = {"100pts": torch.linspace(0, 1, 100), "40pts": torch.linspace(0, 1, 40), "300pts": torch.linspace(0, 1, 300),
         "near_pairs": torch.tensor([0.0, 1e-3, 0.5, 0.5 + 1e-4, 1.0]), "from_quarter": torch.tensor([0.25, 0.6, 2.0])}
# last-layer gain and span with which the controller rejects at least twice (asserted), in the direction that keeps
# the flow's growth, and with it the amplification of fp32 rounding, moderate
STIFF = {SIMT3: (150.0, torch.linspace(1, 0, 3)), SIMT2: (120.0, torch.linspace(0, 1, 4)),
         TC128: (120.0, torch.linspace(0, 1, 3)), FUSED64: (50.0, torch.linspace(0, 1, 4)),
         FUSED200: (150.0, torch.linspace(1, 0, 3))}
# tolerance at which the plan-reuse case needs more steps than at 1e-4
TIGHT = {SIMT3: 1e-6, FUSED64: 1e-6}
SEED = 3


def _field(dim, w, act="selu", gain=1.0, seed=SEED):
    """(cfm_b200.MLP on the CPU, fp32 oracle MLP) with the same weights; ``gain`` scales the last layer."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
    with torch.no_grad():
        m.net[6].weight.mul_(gain)
    mc = vf.make_mlp(dim, w=w, time_varying=True)
    mc.load_state_dict(m.state_dict())
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            mc.net[k] = torch.nn.SiLU()
    return m, mc


def _sync_oracle(mc, m):
    mc.load_state_dict({k: v.detach().cpu() for k, v in m.state_dict().items()})


def _x(B, dim, seed=9, scale=1.0):
    return torch.randn(B, dim, generator=torch.Generator().manual_seed(seed)) * scale


def _f(mc):
    return lambda t, z: vf.wrapped_forward(mc, t, z)


def _oracle(mc, x, span, atol=1e-4, rtol=1e-4):
    """fp32 oracle run with its step record; asserts what makes its step sequence reproducible on other arithmetic:
    no error ratio within 1e-3 of 1, and the same counts from a float64 run of the same controller.  (The second
    matters on expansive fields: after a sliver of a step onto a checkpoint the error ratio is rounding noise, the
    step factor 0.9 ratio^-0.2 carries it into dt, and a later ratio can end up on the other side of 1.)"""
    rec = []
    with torch.no_grad():
        ref, st = co.dopri5_any_direction(_f(mc), x, span, atol, rtol, record=rec)
        _, st64 = co.dopri5_any_direction(_f(copy.deepcopy(mc).double()), x.double(), span.double(), atol, rtol)
    gap = min(abs(r["ratio"] - 1.0) for r in rec)
    assert gap >= 1e-3, f"an error ratio within {gap:.1e} of 1: pick another seed for this case"
    assert st == st64, f"step counts depend on rounding ({st} in fp32, {st64} in float64): pick another case"
    # torchdyn records a checkpoint only when t + dt == t_span[ckpt] holds in fp32, so it can lose one to rounding (the
    # device snaps t onto it instead, see test_checkpoint_the_oracle_loses_to_rounding); these cases need them all
    assert ref.shape[0] == len(span), "the oracle lost a checkpoint to rounding: pick another span"
    return ref, st, rec


def _tight_last(mc, x, span):
    """Last state of a float64 oracle run at 1e-9 tolerances."""
    m64 = copy.deepcopy(mc).double()
    with torch.no_grad():
        ref, _ = co.dopri5_any_direction(_f(m64), x.double(), span.double(), 1e-9, 1e-9)
    assert ref.shape[0] == len(span)
    return ref[-1]


def _node(m, solver="dopri5", atol=1e-4, rtol=1e-4):
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver=solver, sensitivity="adjoint", atol=atol, rtol=rtol)
    node.use_fused_small = False
    return node


def _counts(stats):
    return stats["nfe"], stats["accepted"], stats["rejected"]


def _run(node, x, span, ref, st):
    """One device trajectory gated against an oracle run: counts equal, every checkpoint within 1e-4."""
    traj = node.trajectory(x.to(DEV), span)
    assert not node.stats.get("fused")
    assert traj.shape == ref.shape
    assert _counts(node.stats) == _counts(st)
    err = (traj.cpu() - ref).abs().amax(dim=(1, 2))
    assert (err <= 1e-4 * max(1.0, ref.abs().max().item())).all(), err
    return traj


# ================================================================================================ A. whole trajectories
@pytest.mark.parametrize("span", list(REVERSE_SPANS), ids=list(REVERSE_SPANS))
@pytest.mark.parametrize("cls", CLASSES, ids=_ids)
def test_decreasing_span_against_the_oracle(cls, span):
    dim, w, B, act = cls
    span = REVERSE_SPANS[span]
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    ref, st, _ = _oracle(mc, x, span)
    node = _node(m)
    traj = _run(node, x, span, ref, st)
    assert node.stats["t"] == float(span[-1])  # with its sign: the driver integrated -t_span
    assert torch.equal(traj[0].cpu(), x)
    assert (traj[-1].cpu().double() - _tight_last(mc, x, span)).abs().max() < 5e-3
    # the second call replays the captured step of the reversed field and gives the same bits
    stats = dict(node.stats)
    again = node.trajectory(x.to(DEV), span)
    assert node.stats["graph"] and torch.equal(again, traj)
    assert {k: v for k, v in node.stats.items() if k != "graph"} == {k: v for k, v in stats.items() if k != "graph"}


@pytest.mark.parametrize("cls", [SIMT3, FUSED64], ids=_ids)
def test_checkpoint_the_oracle_loses_to_rounding(cls):
    """Over [0.8, 0.35, 0.1] fp32 gives t + (t_end - t) > t_end on the last step: torchdyn's exact comparison then
    records nothing and leaves the loop, one point short.  The controller snaps a clipped step onto its checkpoint
    (rk_control.cuh), so the device returns every point: the oracle's own up to there, and a last one that the
    float64 run confirms."""
    dim, w, B, act = cls
    span = torch.tensor([0.8, 0.35, 0.1])
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    rec = []
    with torch.no_grad():
        ref, st = co.dopri5_any_direction(_f(mc), x, span, 1e-4, 1e-4, record=rec)
    assert ref.shape[0] == 2 and rec[-1]["clipped"] and min(abs(r["ratio"] - 1.0) for r in rec) >= 1e-3
    node = _node(m)
    traj = node.trajectory(x.to(DEV), span)
    assert not node.stats.get("fused") and traj.shape[0] == 3 and _counts(node.stats) == _counts(st)
    assert node.stats["t"] == float(span[-1])
    assert (traj[:2].cpu() - ref).abs().max() <= 1e-4 * max(1.0, ref.abs().max().item())
    assert (traj[-1].cpu().double() - _tight_last(mc, x, span)).abs().max() < 5e-3


@pytest.mark.parametrize("cls", CLASSES, ids=_ids)
def test_forward_then_backward_returns_to_the_start(cls):
    dim, w, B, act = cls
    m, _ = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim).to(DEV)
    node = _node(m, atol=1e-6, rtol=1e-6)
    there = node.trajectory(x, torch.linspace(0, 1, 3))
    assert not node.stats.get("fused") and node.stats["t"] == 1.0
    back = node.trajectory(there[-1], torch.linspace(1, 0, 3))
    assert not node.stats.get("fused") and node.stats["t"] == 0.0
    assert (back[-1] - x).abs().max() <= 2e-4 * max(1.0, x.abs().max().item())
    assert (back[1] - there[1]).abs().max() <= 2e-4 * max(1.0, x.abs().max().item())


@pytest.mark.parametrize("cls", [SIMT3, SIMT2, (5, 256, 7, "selu")], ids=_ids)
def test_euler_multi_kernel_on_unaligned_checkpoints(cls):
    """B D % 4 != 0: traj[n], the MLP's input and output, is only 4- or 8-byte aligned for odd n."""
    dim, w, B, act = cls
    assert (B * dim) % 4 != 0
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    for span in (torch.tensor([1.0, 0.9, 0.4, 0.35, 0.0]), torch.tensor([0.0, 0.05, 0.5, 0.55, 0.8, 1.5])):
        node = _node(m, solver="euler")
        traj = node.trajectory(x.to(DEV), span)
        assert not node.stats.get("fused") and _counts(node.stats) == (len(span) - 1, len(span) - 1, 0)
        with torch.no_grad():
            ref = vf.euler_trajectory(_f(mc), x, span)  # a negative step needs no reversed field
            ref64 = vf.euler_trajectory(_f(copy.deepcopy(mc).double()), x.double(), span.double())
        assert traj.shape == ref.shape
        assert (traj.cpu() - ref).abs().max() <= 2e-5 * max(1.0, ref.abs().max().item())
        assert (traj.cpu().double() - ref64).abs().max() <= 2e-5 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("cls", CLASSES, ids=_ids)
def test_stiff_field_rejected_steps(cls):
    dim, w, B, act = cls
    gain, span = STIFF[cls]
    m, mc = _field(dim, w, act, gain=gain)
    m = m.to(DEV)
    x = _x(B, dim)
    ref, st, rec = _oracle(mc, x, span)
    assert st["rejected"] >= 2 and sum(r["ratio"] > 1.0 for r in rec) == st["rejected"], st
    _run(_node(m), x, span, ref, st)


@pytest.mark.parametrize("cls,gain,span", [(SIMT3, 50.0, torch.linspace(0, 1, 7)), (FUSED64, 70.0, torch.linspace(1, 0, 5)),
                                           (FUSED200, 150.0, torch.linspace(1, 0, 5))],
                         ids=["3-64-forward", "64-256-reverse", "200-256-reverse"])
def test_rejected_clipped_step(cls, gain, span):
    """A stiff field over several checkpoints: a step clipped onto a checkpoint is rejected, and the controller still
    applies dt = dt_old - dt although nothing was recorded."""
    dim, w, B, act = cls
    m, mc = _field(dim, w, act, gain=gain)
    m = m.to(DEV)
    x = _x(B, dim)
    ref, st, rec = _oracle(mc, x, span)
    assert any(r["clipped"] and not r["accepted"] for r in rec), "no rejected clipped step: the case covers nothing"
    assert any(r["clipped"] and r["accepted"] for r in rec) and any(not r["clipped"] for r in rec)
    _run(_node(m), x, span, ref, st)


@pytest.mark.parametrize("span", list(SPANS), ids=list(SPANS))
@pytest.mark.parametrize("cls", [SIMT3, TC128, FUSED64], ids=_ids)
def test_long_dense_and_nonuniform_spans(cls, span):
    dim, w, B, act = cls
    name, span = span, SPANS[span]
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    ref, st, rec = _oracle(mc, x, span)
    if name == "300pts":  # spacing far below the natural step: every step is clipped and dt_old is carried along
        assert sum(not r["clipped"] for r in rec) <= 1 and st["accepted"] == 299  # (the t_end clip is not flagged)
    if name == "from_quarter":  # the natural step is far below the spacing: unclipped steps, then the t_end clip
        assert sum(not r["clipped"] for r in rec) >= 2 and rec[0]["t"] == 0.25
    node = _node(m)
    traj = _run(node, x, span, ref, st)
    assert node.stats["t"] == float(span[-1])
    if name in ("40pts", "near_pairs", "from_quarter"):
        assert (traj[-1].cpu().double() - _tight_last(mc, x, span)).abs().max() < 5e-3


def test_readme_row_shape_over_its_100_point_span():
    """MLP 785-256-256-256-784 on a 100-point span (a reduced batch keeps the CPU oracle affordable)."""
    m, mc = _field(784, 256, "selu", seed=0)
    m = m.to(DEV)
    x = _x(200, 784)
    span = torch.linspace(0, 1, 100)
    ref, st, _ = _oracle(mc, x, span)
    _run(_node(m), x, span, ref, st)


@pytest.mark.parametrize("cls", [SIMT3, FUSED64], ids=_ids)
def test_burst_settings_change_nothing(cls):
    """Steps enqueued behind the device-side ``done`` flag are no-ops in all 15 kernels of a step (the gated fused
    MLP included) and are not counted."""
    dim, w, B, act = cls
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    span = torch.linspace(0, 1, 6)
    ref, st, _ = _oracle(mc, x, span)
    outs = []
    for lo, hi in ((1, 1), (4, 32), (32, 64)):
        node = _node(m)
        node.min_burst, node.max_burst = lo, hi
        first = _run(node, x, span, ref, st)
        stats = dict(node.stats)
        second = _run(node, x, span, ref, st)  # now with the step count predicted from the first call
        assert torch.equal(first, second)
        outs.append((first, {k: v for k, v in stats.items() if k != "graph"}))
    for traj, stats in outs[1:]:
        assert torch.equal(traj, outs[0][0]) and stats == outs[0][1]


@pytest.mark.parametrize("cls", [SIMT3, FUSED64], ids=_ids)
def test_plan_reuse_with_something_changed(cls):
    dim, w, B, act = cls
    m, mc = _field(dim, w, act, gain=3.0)
    m = m.to(DEV)
    node = _node(m)
    span = torch.linspace(0, 1, 4)
    x1 = _x(B, dim, seed=11)
    ref1, st1, _ = _oracle(mc, x1, span)
    traj1 = _run(node, x1, span, ref1, st1)
    keep = traj1.clone()
    plan = next(iter(node._plans.values()))
    steps = lambda st: st["accepted"] + st["rejected"]  # noqa: E731
    # tolerances are not part of the plan, they travel in the state struct; tightened, the same plan needs more steps
    # than its previous call predicted (the top-up bursts) ...
    node.atol = node.rtol = tight = TIGHT[cls]
    ref2, st2, _ = _oracle(mc, x1, span, tight, tight)
    assert steps(st2) > steps(st1)
    _run(node, x1, span, ref2, st2)
    # ... and, loosened again on new data, fewer (surplus steps are no-ops behind `done`)
    node.atol = node.rtol = 1e-4
    x3 = _x(B, dim, seed=12, scale=6.0)
    ref3, st3, _ = _oracle(mc, x3, span)
    assert steps(st3) < steps(st2)
    _run(node, x3, span, ref3, st3)
    assert next(iter(node._plans.values())) is plan and node.stats["graph"]
    # same n_span, other values and another t0: the device span is refreshed under the captured init graph
    span_b = torch.tensor([0.3, 0.35, 0.9, 1.6])
    ref4, st4, _ = _oracle(mc, x1, span_b)
    _run(node, x1, span_b, ref4, st4)
    assert next(iter(node._plans.values())) is plan and node.stats["t"] == float(span_b[-1])
    # weights updated in place, as optimizer.step() does: new plan, new blob, and a new reversed field
    back = torch.linspace(1, 0, 4)
    refb0, stb0, _ = _oracle(mc, x1, back)
    _run(node, x1, back, refb0, stb0)
    g = torch.Generator().manual_seed(5)
    with torch.no_grad():
        for p in m.parameters():
            p.add_((0.05 * torch.randn(p.shape, generator=g)).to(DEV))
    _sync_oracle(mc, m)
    ref6, st6, _ = _oracle(mc, x1, span)
    assert (ref6 - ref1).abs().max() > 1e-2  # the update matters at the gate's scale
    _run(node, x1, span, ref6, st6)
    refb, stb, _ = _oracle(mc, x1, back)
    assert (refb - refb0).abs().max() > 1e-2
    _run(node, x1, back, refb, stb)
    # the activation flipped on the module
    m.act = _ffi.ACT_SILU if act == "selu" else _ffi.ACT_SELU
    for k in (1, 3, 5):
        mc.net[k] = torch.nn.SiLU() if act == "selu" else torch.nn.SELU()
    ref7, st7, _ = _oracle(mc, x1, span)
    _run(node, x1, span, ref7, st7)
    ref8, st8, _ = _oracle(mc, x1, back)
    _run(node, x1, back, ref8, st8)
    assert torch.equal(traj1, keep)  # an earlier result is the caller's own memory


def test_mlp_algo_flipped_on_the_module_rebuilds_the_plan():
    dim, w, B, act = TC128
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    span = torch.linspace(0, 1, 3)
    ref, st, _ = _oracle(mc, x, span)
    node = _node(m)
    tc = _run(node, x, span, ref, st)
    assert next(iter(node._plans.values()))["xs_hi"] is not None
    m.mlp_algo = 1
    simt = _run(node, x, span, ref, st)
    assert next(iter(node._plans.values()))["xs_hi"] is None
    assert not torch.equal(tc, simt)  # two different kernels did run
    back = torch.linspace(1, 0, 3)
    refb, stb, _ = _oracle(mc, x, back)
    _run(node, x, back, refb, stb)  # the reversed field follows the module's mlp_algo
    assert next(iter(node._plans.values()))["xs_hi"] is None


@pytest.mark.parametrize("cls,span", [(SIMT3, torch.linspace(0, 1, 5)), (SIMT2, torch.linspace(1, 0, 4)),
                                      (FUSED200, torch.tensor([0.85, 0.4, 0.05]))],
                         ids=["3-64-odd-forward", "2-50-odd-reverse", "200-256-reverse"])
def test_graph_and_eager_stepping_give_identical_bits(cls, span):
    dim, w, B, act = cls
    m, _ = _field(dim, w, act, gain=4.0)
    m = m.to(DEV)
    x = _x(B, dim).to(DEV)
    outs = []
    for graph in (True, False):
        node = _node(m, atol=1e-5, rtol=1e-5)
        node.use_cuda_graph = graph
        node.trajectory(x, span)
        outs.append((node.trajectory(x, span), dict(node.stats)))
        assert node.stats["graph"] == graph and not node.stats.get("fused")
    (o_g, s_g), (o_e, s_e) = outs
    assert torch.equal(o_g, o_e)
    assert {k: v for k, v in s_g.items() if k != "graph"} == {k: v for k, v in s_e.items() if k != "graph"}


def test_higher_rank_and_non_contiguous_input():
    dim, w, B, act = FUSED64
    m, mc = _field(dim, w, act)
    m = m.to(DEV)
    x = _x(B, dim)
    span = torch.linspace(0, 1, 3)
    ref, st, _ = _oracle(mc, x, span)
    node = _node(m)
    flat = _run(node, x, span, ref, st)
    img = node.trajectory(x.reshape(B, 1, 8, 8).to(DEV), span)
    assert img.shape == (3, B, 1, 8, 8) and torch.equal(img.reshape(3, B, dim), flat)
    wide = torch.zeros(B, 2 * dim)
    wide[:, ::2] = x
    strided = wide.to(DEV)[:, ::2]
    assert not strided.is_contiguous()
    assert torch.equal(node.trajectory(strided, span), flat)
    turned = x.reshape(B, 8, 8).to(DEV).transpose(1, 2)  # rank 3 and non-contiguous: other rows of the same field
    assert not turned.is_contiguous()
    assert torch.equal(node.trajectory(turned, span),
                       node.trajectory(turned.reshape(B, dim), span).reshape(3, B, 8, 8))


# ============================================================================================ B. the kernels one by one
A = [[float(a) for a in row] + [0.0] * (6 - len(row)) for row in vf._A]
E = [float(e) for e in vf._BERR]
STATE_FIELDS = [n for n, _ in _ffi.RkState._fields_]


def _state(**kw):
    st = _ffi.RkState()
    st.t, st.dt, st.t_end, st.atol, st.rtol = 0.25, 0.0625, 1.0, 1e-4, 1e-4
    st.n_span, st.ckpt, st.save_slot = 2, 1, -1
    for k, v in kw.items():
        setattr(st, k, v)
    return st


def _up(st):
    return torch.frombuffer(bytearray(bytes(st)), dtype=torch.uint8).to(DEV)


def _down(buf):
    return _ffi.RkState.from_buffer_copy(bytes(buf.cpu().numpy().tobytes()))


def _sp():
    return _ffi.stream_ptr(torch.device(DEV))


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sizes():
    """Element counts on the 128-bit path (multiples of 4) and on the scalar one, down to a single element and up to
    one past what a full grid covers in one pass of its grid-stride loop (8 CTAs per SM x 256 threads x 8 elements)."""
    wrap = 8 * 256 * 8 * _sms()
    return [1, 3, 5, 1024, 1026, 513 * 64, wrap + 4 * 999, wrap + 4 * 999 + 1]


def _rand(numel, seed, n_k=7):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(numel, generator=g), torch.randn(n_k, numel, generator=g)


@pytest.mark.parametrize("stage", [1, 2, 3, 4, 5, 6])
def test_stage_input_every_stage_and_size(stage):
    L = _ffi.lib()
    dt, t = 0.0625, 0.25
    for numel in _sizes():
        x, k = _rand(numel, stage)
        xd, kd, st = x.to(DEV), k.to(DEV), _up(_state(dt=dt, t=t))
        out = torch.full((numel,), 7.0, device=DEV)
        hi, lo = (torch.zeros(numel, dtype=torch.float16, device=DEV) for _ in range(2))
        errp, t_s = torch.full((numel,), 7.0, device=DEV), torch.zeros(1, device=DEV)
        _ffi.check(L.cfm_rk_stage_input(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(kd), _ffi.ptr(out), _ffi.ptr(hi),
                                        _ffi.ptr(lo), _ffi.ptr(t_s), _ffi.ptr(errp) if stage == 6 else None, numel,
                                        stage, _sp()), "cfm_rk_stage_input")
        ref = x.double() + dt * sum(A[stage][j] * k[j].double() for j in range(stage))
        scale = max(1.0, ref.abs().max().item())
        assert (out.cpu().double() - ref).abs().max() <= 4e-6 * scale, numel
        assert ((hi.float() + lo.float() / 2048.0) - out).abs().max().item() <= 2.0 ** -21 * scale, numel
        assert abs(t_s.item() - (t + vf._C[stage] * dt)) <= 1e-7
        if stage == 6:
            ep = sum(E[j] * k[j].double() for j in range(6))
            assert (errp.cpu().double() - ep).abs().max() <= 4e-6 * max(1.0, ep.abs().max().item()), numel
        # fp32 output alone (the SIMT driver's call) gives the same bits
        out2 = torch.full((numel,), 7.0, device=DEV)
        _ffi.check(L.cfm_rk_stage_input(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(kd), _ffi.ptr(out2), None, None, None,
                                        None, numel, stage, _sp()), "cfm_rk_stage_input")
        assert torch.equal(out2, out)
        assert _down(st).t == t and _down(st).dt == dt  # the state is read-only here


@pytest.mark.parametrize("numel", [5, 1024, 1026])
def test_stage_input_after_the_end_writes_nothing(numel):
    L = _ffi.lib()
    x, k = _rand(numel, 1)
    st = _up(_state(done=1))
    out, errp = torch.full((numel,), 7.0, device=DEV), torch.full((numel,), 7.0, device=DEV)
    hi, lo = (torch.full((numel,), 7.0, dtype=torch.float16, device=DEV) for _ in range(2))
    t_s = torch.full((1,), 7.0, device=DEV)
    for stage in (1, 6):
        _ffi.check(L.cfm_rk_stage_input(_ffi.ptr(st), _ffi.ptr(x.to(DEV)), _ffi.ptr(k.to(DEV)), _ffi.ptr(out),
                                        _ffi.ptr(hi), _ffi.ptr(lo), _ffi.ptr(t_s), _ffi.ptr(errp) if stage == 6 else
                                        None, numel, stage, _sp()), "cfm_rk_stage_input")
    for buf in (out, errp, hi, lo, t_s):
        assert (buf == 7.0).all()


def _err_sum(x, xnew, k, dt, atol, rtol):
    e = dt * sum(E[j] * k[j].double() for j in range(7))
    tol = atol + rtol * torch.maximum(x.double().abs(), xnew.double().abs())
    return float(((e / tol) ** 2).sum())


def test_error_norm_with_and_without_the_stage6_partial():
    L = _ffi.lib()
    dt, atol, rtol = 0.0625, 1e-4, 3e-4
    for numel in _sizes():
        x, k = _rand(numel, 21)
        xnew = x + 0.1 * _rand(numel, 22)[0]
        xd, kd, nd = x.to(DEV), k.to(DEV), xnew.to(DEV)
        ref = _err_sum(x, xnew, k, dt, atol, rtol)
        # the partial as the stage-6 kernel writes it
        st = _up(_state(dt=dt, atol=atol, rtol=rtol))
        out, errp = torch.empty(numel, device=DEV), torch.empty(numel, device=DEV)
        _ffi.check(L.cfm_rk_stage_input(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(kd), _ffi.ptr(out), None, None, None,
                                        _ffi.ptr(errp), numel, 6, _sp()), "cfm_rk_stage_input")
        got = []
        for part in (None, errp):
            st = _up(_state(dt=dt, atol=atol, rtol=rtol))
            _ffi.check(L.cfm_rk_error_norm(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(nd), _ffi.ptr(kd), _ffi.ptr(part),
                                           numel, _sp()), "cfm_rk_error_norm")
            one = _down(st).err_acc
            assert abs(one - ref) <= 1e-6 * ref, (numel, part is not None)
            # a second call adds onto the accumulator
            _ffi.check(L.cfm_rk_error_norm(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(nd), _ffi.ptr(kd), _ffi.ptr(part),
                                           numel, _sp()), "cfm_rk_error_norm")
            assert abs(_down(st).err_acc - 2 * ref) <= 2e-6 * ref
            got.append(one)
            # past the end the accumulator is left alone
            st = _up(_state(dt=dt, atol=atol, rtol=rtol, done=1, err_acc=0.375))
            _ffi.check(L.cfm_rk_error_norm(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(nd), _ffi.ptr(kd), _ffi.ptr(part),
                                           numel, _sp()), "cfm_rk_error_norm")
            assert _down(st).err_acc == 0.375
        assert abs(got[0] - got[1]) <= 1e-6 * ref


# ---- the one-thread controller: torchdyn's loop body (oracle/vector_field.py::dopri5_trajectory) on an RkState, every
# scalar rounded to fp32 in the kernel's order
def _ref_prestep(s, span):
    if not (s["t"] < s["t_end"]):
        s["done"] = 1
        return
    if f32(s["t"] + s["dt"]) > s["t_end"]:
        s["dt"] = f32(s["t_end"] - s["t"])
    if s["ckpt"] < s["n_span"] and f32(s["t"] + s["dt"]) > span[s["ckpt"]]:
        s["dt_old"], s["ckpt_flag"] = s["dt"], 1
        s["dt"] = f32(span[s["ckpt"]] - s["t"])


def _ref_control(s, span, numel):
    """Returns whether the adapted dt went through pow (then it is compared to a few ulp, not bit for bit)."""
    if s["done"]:
        s["commit"] = 0
        return False
    ratio = f32(np.sqrt(np.float64(s["err_acc"]) / np.float64(numel)))
    s["err_acc"], s["ratio"] = 0.0, ratio
    s["nfe"] += 6
    accept = bool(ratio <= f32(1))
    s["save_slot"] = -1
    if accept:
        tn = f32(s["t"] + s["dt"])
        if s["ckpt"] < s["n_span"] and (tn == span[s["ckpt"]] or s["ckpt_flag"]):
            tn = span[s["ckpt"]]
            s["save_slot"] = s["ckpt"]
            s["ckpt"] += 1
        s["t"] = tn
        s["accepted"] += 1
    else:
        s["rejected"] += 1
    dt = s["dt"]
    if s["ckpt_flag"]:
        dt, s["ckpt_flag"] = f32(s["dt_old"] - dt), 0
    inexact = False
    if ratio == 0:
        dt = f32(dt * f32(10))
    else:
        lo = f32(1) if ratio < 1 else f32(0.2)
        raw = f32(f32(0.9) / f32(np.power(np.float64(ratio), np.float64(f32(0.2)))))
        factor = min(f32(10), max(raw, lo))
        inexact = factor == raw and ratio != 1
        dt = f32(dt * factor)
    s["dt"] = dt
    _ref_prestep(s, span)
    s["commit"] = 1 if accept else 0
    return inexact


def _as_dict(st):
    d = {}
    for name, ctype in _ffi.RkState._fields_:
        v = getattr(st, name)
        d[name] = f32(v) if ctype is C.c_float else v
    return d


SPAN5 = [0.0, 0.25, 0.5, 0.75, 1.0]
# name -> (state fields, ratio the error sum encodes, span)
CONTROL_CASES = {
    "ratio_zero_grows_tenfold": (dict(t=0.1, dt=0.01, ckpt=1), 0.0, SPAN5),
    "ratio_exactly_one_is_accepted": (dict(t=0.1, dt=0.01, ckpt=1), 1.0, SPAN5),
    "ratio_tiny_factor_capped_at_ten": (dict(t=0.1, dt=0.001, ckpt=1), 1e-8, SPAN5),
    "ratio_below_one_factor_floored_at_one": (dict(t=0.1, dt=0.01, ckpt=1), 0.8, SPAN5),
    "ratio_below_one_grows_by_pow": (dict(t=0.1, dt=0.01, ckpt=1), 0.05, SPAN5),
    "rejected_shrinks_by_pow": (dict(t=0.1, dt=0.05, ckpt=1), 50.0, SPAN5),
    "rejected_floor_of_a_fifth": (dict(t=0.1, dt=0.05, ckpt=1), 1e4, SPAN5),
    "rejected_clipped_step_restores_dt_old": (dict(t=0.2, dt=0.05, dt_old=0.09, ckpt_flag=1, ckpt=1), 3.0, SPAN5),
    "rejected_clipped_step_floor": (dict(t=0.2, dt=0.05, dt_old=0.3, ckpt_flag=1, ckpt=1), 1e5, SPAN5),
    "accepted_clipped_step_snaps_onto_the_checkpoint": (dict(t=0.2, dt=0.0500001, dt_old=0.09, ckpt_flag=1, ckpt=1),
                                                        0.3, SPAN5),
    "accepted_clipped_step_ratio_zero": (dict(t=0.2, dt=0.05, dt_old=0.09, ckpt_flag=1, ckpt=1), 0.0, SPAN5),
    "accepted_step_lands_on_a_checkpoint_unclipped": (dict(t=0.25, dt=0.25, ckpt=2), 0.5, SPAN5),
    "next_step_clipped_to_the_checkpoint": (dict(t=0.3, dt=0.15, ckpt=2), 0.01, SPAN5),
    "next_step_clipped_to_t_end": (dict(t=0.8, dt=0.1, ckpt=5, n_span=5), 0.01, SPAN5),
    "last_checkpoint_reached_sets_done": (dict(t=0.9, dt=0.1, dt_old=0.2, ckpt_flag=1, ckpt=4, n_span=5), 0.4, SPAN5),
    "rejected_last_step_is_not_done": (dict(t=0.9, dt=0.1, dt_old=0.2, ckpt_flag=1, ckpt=4, n_span=5), 2.0, SPAN5),
    "past_the_end_only_clears_commit": (dict(t=1.0, dt=0.1, ckpt=5, n_span=5, done=1, commit=1, save_slot=4,
                                             accepted=9, rejected=2, nfe=68), 0.5, SPAN5),
    "span_not_starting_at_zero": (dict(t=-0.35, dt=0.2, t_end=-0.1, ckpt=2, n_span=3), 0.2, [-0.8, -0.35, -0.1]),
}


@pytest.mark.parametrize("name", list(CONTROL_CASES))
def test_control_branch_by_branch(name):
    L = _ffi.lib()
    fields, ratio, span = CONTROL_CASES[name]
    numel = 3003
    st = _state(n_span=len(span), t_end=span[-1], accepted=3, rejected=1, nfe=26)
    for k, v in fields.items():
        setattr(st, k, v)
    st.err_acc = float(np.float64(ratio) ** 2 * numel)
    span32 = np.asarray(span, dtype=np.float32)
    ref = _as_dict(st)
    inexact = _ref_control(ref, span32, numel)
    if not ref["done"] or not fields.get("done"):
        # the error sum does encode the ratio the case is about (1 and 0 exactly)
        assert ref["ratio"] == pytest.approx(ratio, rel=1e-6) and (ratio not in (0.0, 1.0) or ref["ratio"] == ratio)
    buf = _up(st)
    _ffi.check(L.cfm_rk_control(_ffi.ptr(buf), _ffi.ptr(torch.from_numpy(span32).to(DEV)), numel, _sp()),
               "cfm_rk_control")
    got = _as_dict(_down(buf))
    for field in STATE_FIELDS:
        if inexact and field in ("dt", "dt_old"):  # device powf is not numpy's pow to the last bit
            assert got[field] == pytest.approx(ref[field], rel=2e-6), field
        else:
            assert got[field] == ref[field], (field, got[field], ref[field])
    if not fields.get("done"):
        assert got["err_acc"] == 0.0 and got["nfe"] == 32


def test_control_case_table_reaches_every_branch():
    """The table above, run through the fp32 restatement alone: which branches its cases take."""
    seen = set()
    for name, (fields, ratio, span) in CONTROL_CASES.items():
        st = _state(n_span=len(span), t_end=span[-1])
        for k, v in fields.items():
            setattr(st, k, v)
        st.err_acc = float(np.float64(ratio) ** 2 * 3003)
        s0 = _as_dict(st)
        s = dict(s0)
        _ref_control(s, np.asarray(span, dtype=np.float32), 3003)
        if s0["done"]:
            seen.add("past_end")
            continue
        acc = s["accepted"] > s0["accepted"]
        seen.add(("accept" if acc else "reject") + ("_clipped" if s0["ckpt_flag"] else ""))
        seen.add("ratio0" if s["ratio"] == 0 else "ratio1" if s["ratio"] == 1 else "")
        if acc and s["save_slot"] >= 0:
            seen.add("saved_clipped" if s0["ckpt_flag"] else "saved_exact")
        if s["done"]:
            seen.add("done")
        if s["ckpt_flag"]:
            seen.add("next_clipped")
        elif not s["done"] and f32(s["t"] + s["dt"]) == s["t_end"]:
            seen.add("next_to_end")
    assert {"past_end", "accept", "reject", "accept_clipped", "reject_clipped", "ratio0", "ratio1", "saved_clipped",
            "saved_exact", "done", "next_clipped", "next_to_end"} <= seen


@pytest.mark.parametrize("numel", [5, 1026, 4096])
def test_commit(numel):
    L = _ffi.lib()
    g = torch.Generator().manual_seed(numel)
    x, xnew = torch.randn(numel, generator=g), torch.randn(numel, generator=g)
    k, traj = torch.randn(7, numel, generator=g), torch.randn(4, numel, generator=g)
    for commit, slot in ((0, 2), (1, -1), (1, 2), (1, 0), (1, 3)):
        xd, kd, td, nd = x.to(DEV), k.to(DEV), traj.to(DEV), xnew.to(DEV)
        st = _up(_state(commit=commit, save_slot=slot, n_span=4))
        _ffi.check(L.cfm_rk_commit(_ffi.ptr(st), _ffi.ptr(xd), _ffi.ptr(nd), _ffi.ptr(kd), _ffi.ptr(td), numel, _sp()),
                   "cfm_rk_commit")
        ex, ek, et = x.clone(), k.clone(), traj.clone()
        if commit:
            ex, ek[0] = xnew, k[6]  # FSAL: k7 is the next step's k1
            if slot >= 0:
                et[slot] = xnew
        assert torch.equal(xd.cpu(), ex) and torch.equal(kd.cpu(), ek) and torch.equal(td.cpu(), et), (commit, slot)
        assert torch.equal(nd.cpu(), xnew)


def _init_on_device(x, f0, f1, t0, span, atol, rtol, halves=1):
    """The four-call Hairer initial step; ``halves`` = 2 splits the rows in two and adds the partial sums as the
    lock-step driver's all-reduce does.  Returns (state, x_probe, t_probe, scratch after phase 0)."""
    L = _ffi.lib()
    numel = x.numel()
    cut = [0, numel] if halves == 1 else [0, numel // 2 + 1, numel]
    st = _up(_state(t=t0, dt=0.0, t_end=span[-1], atol=atol, rtol=rtol, n_span=len(span), ckpt=0, done=1, ckpt_flag=1))
    span_d = torch.tensor(span, dtype=torch.float32, device=DEV)
    parts = [(x[a:b].contiguous().to(DEV), f0[a:b].contiguous().to(DEV), f1[a:b].contiguous().to(DEV))
             for a, b in zip(cut[:-1], cut[1:])]
    scratch = torch.zeros(4, dtype=torch.float64, device=DEV)
    for xp, f0p, _ in parts:
        part = torch.full((4,), 5.0, dtype=torch.float64, device=DEV)  # phase 0 clears its scratch itself
        _ffi.check(L.cfm_rk_init_sums(_ffi.ptr(st), _ffi.ptr(xp), _ffi.ptr(f0p), None, _ffi.ptr(part), xp.numel(), 0,
                                      _sp()), "cfm_rk_init_sums")
        scratch += part
    sums0 = scratch.cpu().clone()
    probes, t_probe = [], torch.zeros(1, device=DEV)
    for xp, f0p, _ in parts:
        probes.append(torch.empty_like(xp))
        _ffi.check(L.cfm_rk_init_probe(_ffi.ptr(st), _ffi.ptr(xp), _ffi.ptr(f0p), _ffi.ptr(probes[-1]),
                                       _ffi.ptr(t_probe), _ffi.ptr(scratch), xp.numel(), numel, _sp()),
                   "cfm_rk_init_probe")
    for xp, f0p, f1p in parts:  # phase 1 adds into scratch[2]
        _ffi.check(L.cfm_rk_init_sums(_ffi.ptr(st), _ffi.ptr(xp), _ffi.ptr(f0p), _ffi.ptr(f1p), _ffi.ptr(scratch),
                                      xp.numel(), 1, _sp()), "cfm_rk_init_sums")
    _ffi.check(L.cfm_rk_init_finish(_ffi.ptr(st), _ffi.ptr(span_d), _ffi.ptr(scratch), numel, _sp()),
               "cfm_rk_init_finish")
    return _down(st), torch.cat(probes).cpu(), t_probe.item(), sums0, scratch.cpu()


INIT_CASES = {
    # name: (x scale, f0 scale, f1 - f0 scale, expected dt in fp32 or None for "compare with the oracle's init_step")
    "random": (1.0, 1.0, 1e-3, None),           # h1 < 100 h0
    "curved": (1.0, 0.3, 5.0, None),            # d2 > d1 decides h1
    "steep_flat": (1.0, 20.0, 0.0, None),       # f1 == f0 and a large field: 100 h0 < h1
    "x_zero": (0.0, 1.0, 1e-4, f32(100) * f32(1e-6)),     # d0 < 1e-5: h0 = 1e-6, dt = min(100 h0, h1) = 100 h0
    "f_tiny": (1.0, 1e-10, 1e-12, f32(100) * f32(1e-6)),  # d1 < 1e-5: h0 = 1e-6
    "zero_field": (1.0, 0.0, 0.0, f32(1e-6)),   # d1, d2 <= 1e-15: h1 = max(1e-6, 1e-3 h0) = 1e-6 < 100 h0
}


@pytest.mark.parametrize("halves", [1, 2], ids=["whole", "two_shards"])
@pytest.mark.parametrize("numel", [5, 1026, 513 * 64])
@pytest.mark.parametrize("name", list(INIT_CASES))
def test_initial_step(name, numel, halves):
    if halves == 2 and numel < 1000:
        pytest.skip("the sharded form is checked at the two larger sizes")
    sx, sf, sd, want = INIT_CASES[name]
    g = torch.Generator().manual_seed(numel)
    x = sx * torch.randn(numel, generator=g)
    f0 = sf * torch.randn(numel, generator=g)
    f1 = f0 + sd * torch.randn(numel, generator=g)
    t0, span, atol, rtol = 0.125, [0.125, 50.0, 100.0], 1e-4, 2e-4
    st, probe, t_probe, sums0, sums = _init_on_device(x, f0, f1, t0, span, atol, rtol, halves)
    scale = atol + x.double().abs() * rtol
    for got, ref in ((sums0[0], ((x.double() / scale) ** 2).sum()), (sums0[1], ((f0.double() / scale) ** 2).sum()),
                     (sums[2], (((f1.double() - f0.double()) / scale) ** 2).sum())):
        assert abs(float(got) - float(ref)) <= 2e-6 * float(ref) + 1e-300
    assert float(sums0[2]) == 0.0 and float(sums0[3]) == 0.0
    seen = []

    def f(t, z):
        seen.append((float(t), z.clone()))
        return f1

    dt_ref = float(vf.init_step(f, f0, x, torch.tensor(t0), 5, atol, rtol))
    h0 = seen[0][0] - t0
    assert t_probe == pytest.approx(seen[0][0], rel=1e-6)
    assert (probe - seen[0][1]).abs().max() <= 1e-6 * max(1.0, x.abs().max().item())
    if want is not None:  # the constant branches give their constants bit for bit
        assert st.dt_old == float(f32(1e-6)) and st.dt == float(want), (st.dt_old, st.dt)
        assert dt_ref == pytest.approx(float(want), rel=1e-5)
    else:
        assert st.dt_old == pytest.approx(h0, rel=1e-4) and st.dt == pytest.approx(dt_ref, rel=1e-5)
    assert (st.t, st.nfe, st.ckpt, st.ckpt_flag, st.done, st.accepted, st.rejected) == (t0, 2, 1, 0, 0, 0, 0)


def test_initial_step_runs_the_pre_step_of_the_first_step():
    """dt above the first checkpoint is clipped onto it at once; a span that is already over is done."""
    g = torch.Generator().manual_seed(0)
    x, f0 = torch.randn(1026, generator=g), torch.randn(1026, generator=g)
    wide, *_ = _init_on_device(x, f0, f0, 0.0, [0.0, 100.0], 1e-4, 1e-4)
    near, *_ = _init_on_device(x, f0, f0, 0.0, [0.0, 1e-3, 100.0], 1e-4, 1e-4)
    assert wide.ckpt_flag == 0 and wide.dt > 1e-3
    assert near.ckpt_flag == 1 and near.dt == float(f32(1e-3)) and near.done == 0
    assert near.dt_old == pytest.approx(wide.dt, rel=1e-6)  # (the float64 sums are added in no fixed order)
    over, *_ = _init_on_device(x, f0, f0, 1.0, [1.0, 1.0], 1e-4, 1e-4)
    assert over.done == 1


@pytest.mark.parametrize("cls", [SIMT3, FUSED64], ids=_ids)
@pytest.mark.parametrize("field", ["zero", "constant"])
def test_zero_and_constant_fields_end_to_end(cls, field):
    dim, w, B, act = cls
    m, mc = _field(dim, w, act)
    b = torch.linspace(-1.0, 2.0, dim) if field == "constant" else torch.zeros(dim)
    with torch.no_grad():
        for p in m.parameters():
            p.zero_()
        m.net[6].bias.copy_(b)
    _sync_oracle(mc, m)
    m = m.to(DEV)
    x = _x(B, dim)
    span = torch.tensor([0.0, 0.3, 1.0])
    # tolerances at which the rounding residue of sum_j e_j b (the e_j sum to zero) keeps the step factor at its cap of
    # 10, i.e. ratio < (0.9 / 10)^5: the step sequence then does not depend on that residue
    tol = 1e-2
    rec = []
    with torch.no_grad():
        ref, st = vf.dopri5_trajectory(_f(mc), x, span, tol, tol, record=rec)
    assert st["rejected"] == 0 and max(r["ratio"] for r in rec) < 1e-6
    node = _node(m, atol=tol, rtol=tol)
    traj = node.trajectory(x.to(DEV), span)
    assert not node.stats.get("fused") and _counts(node.stats) == _counts(st)
    exact = x.double()[None] + span.double()[:, None, None] * b.double()
    if field == "zero":
        # ratio == 0 on every step: dt = 1e-6 grows tenfold until the checkpoints clip it; x never moves
        assert all(r["ratio"] == 0.0 for r in rec) and node.stats["last_ratio"] == 0.0
        assert [r["dt"] for r in rec[:5]] == pytest.approx([1e-6, 1e-5, 1e-4, 1e-3, 1e-2], rel=1e-5)
        assert torch.equal(traj.cpu(), x[None].expand(3, -1, -1))
    else:
        assert (traj.cpu().double() - exact).abs().max() <= 4e-6 * exact.abs().max()
    assert (traj.cpu() - ref).abs().max() <= 1e-5 * max(1.0, ref.abs().max().item())


def test_argument_refusals_launch_nothing():
    L = _ffi.lib()
    n = 64
    st = _up(_state())
    x, xn, out, errp = (torch.zeros(n + 4, device=DEV) for _ in range(4))
    k, traj = torch.zeros(7, n, device=DEV), torch.zeros(2, n, device=DEV)
    hi, lo = (torch.zeros(n, dtype=torch.float16, device=DEV) for _ in range(2))
    span, t_s = torch.tensor([0.0, 1.0], device=DEV), torch.zeros(1, device=DEV)
    scratch = torch.zeros(4, dtype=torch.float64, device=DEV)
    p, sp, nul = _ffi.ptr, _sp(), None
    off = C.c_void_p(x.data_ptr() + 4)  # a valid address, 4-byte aligned only
    bad = {
        "stage_input: no state": lambda: L.cfm_rk_stage_input(nul, p(x), p(k), p(out), nul, nul, p(t_s), nul, n, 1, sp),
        "stage_input: no x": lambda: L.cfm_rk_stage_input(p(st), nul, p(k), p(out), nul, nul, p(t_s), nul, n, 1, sp),
        "stage_input: no k": lambda: L.cfm_rk_stage_input(p(st), p(x), nul, p(out), nul, nul, p(t_s), nul, n, 1, sp),
        "stage_input: no output": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), nul, nul, nul, p(t_s), nul, n, 1, sp),
        "stage_input: numel 0": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), nul, nul, p(t_s), nul, 0, 1, sp),
        "stage_input: stage 0": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), nul, nul, p(t_s), nul, n, 0, sp),
        "stage_input: stage 7": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), nul, nul, p(t_s), nul, n, 7, sp),
        "stage_input: error partial at stage 5": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), nul, nul,
                                                                              p(t_s), p(errp), n, 5, sp),
        "stage_input: hi without lo": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), p(hi), nul, p(t_s), nul,
                                                                   n, 1, sp),
        "stage_input: lo without hi": lambda: L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), nul, p(lo), p(t_s), nul,
                                                                   n, 1, sp),
        "stage_input: misaligned x": lambda: L.cfm_rk_stage_input(p(st), off, p(k), p(out), nul, nul, p(t_s), nul, n,
                                                                  1, sp),
        "error_norm: no xnew": lambda: L.cfm_rk_error_norm(p(st), p(x), nul, p(k), nul, n, sp),
        "error_norm: numel 0": lambda: L.cfm_rk_error_norm(p(st), p(x), p(xn), p(k), nul, 0, sp),
        "control: no span": lambda: L.cfm_rk_control(p(st), nul, n, sp),
        "control: numel 0": lambda: L.cfm_rk_control(p(st), p(span), 0, sp),
        "commit: no traj": lambda: L.cfm_rk_commit(p(st), p(x), p(xn), p(k), nul, n, sp),
        "commit: numel 0": lambda: L.cfm_rk_commit(p(st), p(x), p(xn), p(k), p(traj), 0, sp),
        "init_sums: phase 1 without f1": lambda: L.cfm_rk_init_sums(p(st), p(x), p(xn), nul, p(scratch), n, 1, sp),
        "init_sums: phase 2": lambda: L.cfm_rk_init_sums(p(st), p(x), p(xn), p(xn), p(scratch), n, 2, sp),
        "init_probe: global count below the local one": lambda: L.cfm_rk_init_probe(p(st), p(x), p(xn), p(out), p(t_s),
                                                                                    p(scratch), n, n - 1, sp),
        "init_finish: no scratch": lambda: L.cfm_rk_init_finish(p(st), p(span), nul, n, sp),
        "axpy: numel 0": lambda: L.cfm_axpy_f32(p(x), p(xn), 0.5, p(out), 0, sp),
    }
    before = L.cfm_launch_count()
    for what, call in bad.items():
        assert call() != 0, what
        assert _ffi.last_error(), what
    assert L.cfm_launch_count() == before
    torch.cuda.synchronize()
    assert bytes(_down(st)) == bytes(_state())
    # the same calls with good arguments do launch
    assert L.cfm_rk_stage_input(p(st), p(x), p(k), p(out), nul, nul, p(t_s), nul, n, 1, sp) == 0
    assert L.cfm_launch_count() == before + 1
