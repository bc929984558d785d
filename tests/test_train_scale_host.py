"""The absolute-scale oracles of the training gradients (tests/train_scale_oracle.py, tests/wide_train_oracle.py)
without a device: each scale bounds its gradient entry by entry and bounds the error of an fp32 evaluation on the CPU
by a small multiple of itself, and the gates of tests/test_gpu_training_rows.py can see one row lost or counted twice
at every batch and position those tests use on 132 SMs, on their own models and inputs
(tests/training_rows_cases.py)."""
import pytest
import torch

import action_oracle as ao
import cnf_train_oracle as cto
import train_scale_oracle as so
import training_rows_cases as rc

import cfm_b200

FP32_BOUND = 1e-5  # an fp32 evaluation errs by far less than this of each entry's scale


def _state(dim, out_dim, w, seed):
    torch.manual_seed(seed)
    return cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True).state_dict()


def _action_inputs(B, dim, seed):
    g = torch.Generator().manual_seed(seed)
    x0, x1 = torch.randn(B, dim, generator=g) * 1.5, torch.randn(B, dim, generator=g) * 1.5 + 1.0
    t = torch.rand(B, 1, generator=g)
    return t * x1 + (1 - t) * x0, t, x0, x1


def _worst(got, ref, scales):
    worst = 0.0
    for g, r, sc in zip(got, ref, scales):
        assert sc.shape == r.shape and (r.abs() <= sc * (1 + 1e-12)).all()
        err = (g.double() - r).abs()
        assert (err[sc == 0] == 0).all()
        worst = max(worst, (err / sc.clamp_min(1e-300)).max().item())
    return worst


def _fp32_action_grads(state, dim, w, xt, t, x0, x1, act):
    """The notebook's lines with torch's double backward, in fp32 on the CPU."""
    m = ao.make_action(state, dim, w, act).float()
    B = xt.shape[0]
    xt, t = xt.float().clone().requires_grad_(True), t.reshape(B, 1).float().clone().requires_grad_(True)
    st = torch.sum(m(torch.cat([xt, t], -1)))
    dsdx, dsdt = torch.autograd.grad(st, (xt, t), create_graph=True)
    a0 = m(torch.cat([x0.float(), torch.zeros(B, 1)], -1))
    a1 = m(torch.cat([x1.float(), torch.ones(B, 1)], -1))
    loss = (a0 - a1 + 0.5 * (dsdx ** 2).sum(1, keepdims=True) + dsdt).mean()
    return torch.autograd.grad(loss, list(m.parameters()), allow_unused=True)


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim,w", [(2, 32), (8, 64)])
@pytest.mark.parametrize("B", [1, 5, 300])
def test_action_scales_bound_the_gradient_and_an_fp32_run(B, dim, w, act):
    state = _state(dim, 1, w, seed=B + dim)
    xt, t, x0, x1 = _action_inputs(B, dim, seed=B)
    _, rg = ao.action_matching_loss_and_grads(state, dim, w, xt, t, x0, x1, act)
    scales = so.action_grad_scales(state, xt, t, x0, x1, act)
    g32 = _fp32_action_grads(state, dim, w, xt, t, x0, x1, act)
    g32 = [torch.zeros_like(r) if g is None else g for g, r in zip(g32, rg)]
    g32[7] = torch.zeros(1)  # b3 enters neither a0 - a1 nor ds: its gradient is exactly 0, as is its scale
    assert scales[7].item() == 0.0
    worst = _worst(g32, rg, scales)
    assert 0 < worst < FP32_BOUND, worst


def test_action_scales_are_the_gradient_when_no_term_cancels():
    """Positive weights, inputs and times, SELU: every pre-activation is positive, act' is the constant lambda and
    act'' is 0, so the act'' terms vanish and every other term is non-negative but for end 1's minus sign: the scales
    are the gradient of the loss with end 1 added."""
    dim, w = 3, 32
    state = {k: v.abs() for k, v in _state(dim, 1, w, seed=3).items()}
    xt, t, x0, x1 = (v.abs() for v in _action_inputs(6, dim, seed=4))
    sc = so.action_grad_scales(state, xt, t, x0, x1, "selu")
    mc = ao.make_action(state, dim, w, "selu")
    a0, a1, dsdx, dsdt = ao.terms(mc, xt, t, x0, x1)
    loss = (a0 + a1 + 0.5 * (dsdx ** 2).sum(1, keepdims=True) + dsdt).mean()
    for r, s in zip(torch.autograd.grad(loss, list(mc.parameters()))[:7], sc[:7]):
        assert torch.allclose(r, s, rtol=1e-10, atol=0)


def _random_states(n_span, B, dim, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n_span, B, dim + 1, generator=g, dtype=torch.float64),
            torch.randn(n_span, B, dim + 1, generator=g, dtype=torch.float64))


def _fp32_cnf_backward(state, traj, t_span, G, act):
    """restated_backward's discrete adjoint evaluated in fp32 (phi_grads in fp32, the adjoint summed in fp32)."""
    Ws, bs = cto._params(state)
    Ws, bs = [W.float() for W in Ws], [b.float() for b in bs]
    traj, G, ts = traj.float(), G.float(), t_span.float()
    dim = traj.shape[2] - 1
    grads = [torch.zeros_like(p) for pair in zip(Ws, bs) for p in pair]
    adj = G[-1].clone()
    for n in range(traj.shape[0] - 2, -1, -1):
        h = ts[n + 1] - ts[n]
        gx, g = cto.phi_grads(Ws, bs, traj[n][:, :dim], ts[n], h * adj[:, :dim], h * adj[:, dim], act)
        for acc, v in zip(grads, g):
            acc += v
        adj = G[n] + adj + torch.cat([gx, torch.zeros_like(gx[:, :1])], 1)
    return grads, adj


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim,w", [(2, 32), (8, 64)])
@pytest.mark.parametrize("B", [1, 5, 300])
def test_cnf_scales_bound_the_gradient_and_an_fp32_run(B, dim, w, act):
    state = _state(dim, dim, w, seed=10 + B + dim)
    traj, G = _random_states(4, B, dim, seed=B)
    span = torch.linspace(1, 0, 4)
    rp, rz = cto.restated_backward(state, traj, span, G, act, h32=True)
    sp, sz = so.cnf_grad_scales(state, traj, span, G, act)
    gp, gz = _fp32_cnf_backward(state, traj, span, G, act)
    worst = _worst(list(gp) + [gz], list(rp) + [rz], list(sp) + [sz])
    assert 0 < worst < FP32_BOUND, worst


def test_cnf_scales_are_the_gradient_when_no_term_cancels():
    """One Euler step, positive weights, states and cotangents, SELU: act'' is 0 and every term is non-negative."""
    dim, w = 2, 32
    state = {k: v.abs() for k, v in _state(dim, dim, w, seed=5).items()}
    traj, G = (v.abs() for v in _random_states(2, 7, dim, seed=6))
    span = torch.tensor([0.0, 0.5])
    rp, rz = cto.restated_backward(state, traj, span, G, "selu")
    sp, sz = so.cnf_grad_scales(state, traj, span, G, "selu")
    for r, s in zip(list(rp) + [rz], list(sp) + [sz]):
        assert torch.allclose(r, s, rtol=1e-10, atol=0)


# ---- the gates can see one row ---------------------------------------------------------------------------------------
H100_SMS = 132


def _exceeds(change, scales, gate):
    return max((c.abs()[s > 0] / s[s > 0]).max().item() for c, s in zip(change, scales) if (s > 0).any()) > gate


def _flow_cases(act):
    """(model, [(B, seed, positions)]) of the GPU tests' one-row flow-matching cases"""
    for w in (32, 64):
        yield rc.flow_small_model(w, act), [(B, B + w, rc.positions_on(B, rc.TILE, H100_SMS))
                                            for B in rc.small_batches(H100_SMS)]
    dim, w, out_dim = rc.TC_SHAPE
    yield rc.flow_tc_model(act), [(B, B, rc.tc_positions(B, dim, w, out_dim)) for B, _ in rc.TC_BATCHES]


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_one_row_gates_see_a_lost_or_doubled_row_in_every_flow_matching_case(act):
    """A one-row call's gradient is that row's: losing the row leaves 0, counting it twice doubles it.  Either moves
    the gradient by the row's own gradient, which must exceed the gate of its own scale on some entry, at every row
    the GPU tests isolate."""
    for m, cases in _flow_cases(act):
        state = rc.state_of(m)
        for B, seed, positions in cases:
            xt, t, ut = rc.flow_batch(m, B, seed, act)
            for r in positions.values():
                _, rg, sc = rc.one_row_flow_reference(state, m.dim, m.out_dim, m.w, xt, t, ut, r, act)
                assert _exceeds(rg, sc, rc.ROW_GATE), (m.w, B, r)


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_one_row_gates_see_a_lost_or_doubled_row_in_every_cnf_case(act):
    """The same for the CNF cases, on float64 Euler states of the GPU tests' initial states (the device's fp32 states
    are within rounding of them)."""
    span = rc.cnf_span()
    for dim, w in ((2, 32), (2, 64), (8, 64)):
        state = rc.state_of(rc.cnf_model(dim, w, act))
        for R, B in rc.cnf_batches(dim, w):
            positions = rc.positions_on(B, R, H100_SMS)
            z, Gdraw = rc.cnf_inputs(state, dim, w, act, B, positions)
            traj = rc.euler_states(state, dim, w, act, z, span)
            for r in positions.values():
                G = torch.zeros_like(Gdraw)
                G[:, r] = Gdraw[:, r]
                ref, scales = rc.one_row_cnf_reference(state, traj, span, G, r, act)
                assert _exceeds(ref, scales, rc.ROW_GATE), (dim, w, B, r)


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("w", [32, 64])
def test_swap_gate_sees_a_lost_or_doubled_row_in_every_action_case(w, act):
    """Swapping row r for row q changes the gradient by (g_q - g_r) / B.  A kernel that loses row r (or counts it
    twice) in both calls shows a change of 0 (or twice it): off by the whole change, which must exceed the gate of
    both calls' scales on some entry, at every batch and row the GPU test swaps."""
    dim = 2
    m = rc.action_model(w, act)
    state = rc.state_of(m)
    for B in rc.small_batches(H100_SMS):
        xt, t, x0, x1 = rc.action_batch(m, B, seed=B + w, act=act)
        S = so.action_grad_scales(state, xt, t, x0, x1, act)
        grads, scales = rc.action_row_terms(state, dim, w, xt, t, x0, x1, act)
        for r in rc.positions_on(B, rc.TILE, H100_SMS).values():
            change, both = rc.swap_reference(S, grads, scales, B, r, rc.swap_partner(B, r))
            assert _exceeds(change, both, rc.SWAP_GATE), (B, r)


def test_positions_on_132_sms():
    """The restated launch rules give the positions the GPU tests are named for on an H100's 132 SMs."""
    B1, B2 = rc.small_batches(H100_SMS)
    assert (B1, B2) == (37, 2133)
    assert rc.positions_on(B1, 16, H100_SMS) == {
        "first row of a warp pair": 0, "second row of a warp pair": 1, "last row of a tile": 15,
        "first row of CTA G-1": 32, "lone valid row of an odd partial tile": 36, "batch's last row": 36}
    p = rc.positions_on(B2, 16, H100_SMS)
    assert p["first row of CTA G-1"] == 2096 and p["first row of CTA 0's second pass"] == 2112 and p[
        "lone valid row of an odd partial tile"] == 2132
    assert [R for R, _ in rc.cnf_batches(2, 64)] == [2, 4, 8, 16]
    assert [R for R, _ in rc.cnf_batches(8, 64)] == [2, 4, 8, 8]
    assert rc.slicing(40003, 256, 66) == (79, 8) and rc.slicing(5001, 256, 257) == (20, 4)


def test_positions_on_a_part_with_fewer_sms_cover_both_co_resident_grids():
    """With 60 SMs a folded launch of 134 tiles gets 60 or 120 CTAs as 1 or 2 fit per SM: the tests take the
    positions of both grids."""
    assert rc.co_resident_grids(2133, 16, 60) == [60, 120]
    p = rc.positions_on(2133, 16, 60)
    assert p["first row of CTA G-1 (G=60)"] == 944 and p["first row of CTA G-1 (G=120)"] == 1904
    assert p["first row of CTA 0's second pass (G=60)"] == 960 and p["first row of CTA 0's second pass (G=120)"] == 1920
    assert rc.co_resident_grids(37, 16, 60) == [3]
