"""One-row gradients of the four training kernels at every structural position of their row loops, and the largest
batches, each gradient entry gated against its own float64 absolute scale.

A kernel that drops a row, counts one twice or reads a neighbour's row moves a full-batch gradient by about 1 / B of
its scale, which at large batches is below any gate rounding allows.  So each case isolates one row r:

* flow matching (both classes): row_scale is 1 on row r and 0 elsewhere.  The other rows then add exact zeros to every
  gradient, but their ut^2 still enters the loss, which is checked too;
* the CNF backward: a cotangent dL/dtraj that is non-zero on row r only; every other row's input gradient is exactly 0;
* action matching (no row_scale): row r's (xt, t, x0, x1) is swapped for row q's, and the change of the device
  gradient is compared with the float64 change (g_q - g_r) / B, gated on the scales of both calls.

The launch rules, the positions they give on this device's SM count, the models, inputs and gates live in
tests/training_rows_cases.py, where tests/test_train_scale_host.py checks without a device that the gates see one
row lost or counted twice on these same inputs.  The achieved errors are in DESIGN.md sections 3.12-3.15."""
import pytest
import torch

import action_oracle as ao
import cnf_train_oracle as cto
import train_scale_oracle as so
import training_rows_cases as rc
import wide_train_oracle as wo
from oracle import train as ot

import cfm_b200

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

LOSS_REL = 2e-6     # the loss, of loss + mean(ut^2) (test_gpu_train.py's gate)
BIG_GATE = 5e-7     # the full-batch gradients at 2^18 and 2^20 rows, of each entry's absolute scale
GRAD_REL = 2e-5     # and of their tensor's max-abs (test_gpu_train.py's gate)


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _entry_gap(got, ref, scales):
    """worst |got - ref| / scale over every entry of every tensor (an entry of scale 0 must be exact)"""
    worst = 0.0
    for g, r, sc in zip(got, ref, scales):
        err = (g.detach().cpu().double() - r).abs()
        assert torch.isfinite(err).all()
        assert (err[sc == 0] == 0).all()
        worst = max(worst, (err / sc.clamp_min(1e-300)).max().item())
    return worst


# ---- flow matching: one row per call ---------------------------------------------------------------------------------
def _flow_rows(m, act, B, positions, seed):
    xt, t, ut = rc.flow_batch(m, B, seed, act)
    state = rc.state_of(m)
    m = m.to(DEV)
    xd, td, ud = xt.to(DEV), t.to(DEV), ut.to(DEV)
    worst = 0.0
    for name, r in positions.items():
        s = torch.zeros(B, device=DEV)
        s[r] = 1.0
        m.zero_grad(set_to_none=True)
        loss = cfm_b200.flow_matching_loss(m, xd, td, ud, row_scale=s)
        loss.backward()
        rl, rg, sc = rc.one_row_flow_reference(state, m.dim, m.out_dim, m.w, xt, t, ut, r, act)
        lscale = rl + ut.double().pow(2).mean().item()
        assert abs(loss.item() - rl) <= LOSS_REL * lscale, (B, name, r, loss.item(), rl)
        gap = _entry_gap([p.grad for p in m.parameters()], rg, sc)
        assert gap <= rc.ROW_GATE, (B, name, r, gap)
        worst = max(worst, gap)
    return worst


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("w", [32, 64])
def test_flow_matching_small_class_one_row_at_every_tile_and_cta_position(w, act):
    m = rc.flow_small_model(w, act)
    sms = sm_count()
    worst = 0.0
    for B in rc.small_batches(sms):
        worst = max(worst, _flow_rows(m, act, B, rc.positions_on(B, rc.TILE, sms), seed=B + w))
    print(f"margins rows small w={w} {act}: grad/abs-scale {worst:.2e} (gate {rc.ROW_GATE:.0e})")


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_flow_matching_tensor_core_class_one_row_at_every_tile_chunk_and_slice_edge(act):
    """B = 5001: every slice count set by occupancy; B = 40003: by the 8-chunk cap.  Neither is a multiple of 8, so
    the last row sits next to the padding of the transposed operands."""
    dim, w, out_dim = rc.TC_SHAPE
    m = rc.flow_tc_model(act)
    worst = 0.0
    for B, regime in rc.TC_BATCHES:
        for l, (n0, n1) in enumerate(((w, dim + 2), (w, w + 1), (w, w + 1), (out_dim, w + 1))):
            slices, chunks = rc.slicing(B, n0, n1)
            assert (chunks == rc.SLICE_MAX_CHUNKS) == (regime == "cap"), (B, l, slices, chunks)
        assert B % 8 != 0
        worst = max(worst, _flow_rows(m, act, B, rc.tc_positions(B, dim, w, out_dim), seed=B))
    print(f"margins rows tc {act}: grad/abs-scale {worst:.2e} (gate {rc.ROW_GATE:.0e})")


# ---- action matching: one row swapped per call -----------------------------------------------------------------------
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("w", [32, 64])
def test_action_matching_row_swap_at_every_tile_and_cta_position(w, act):
    dim = 2
    m = rc.action_model(w, act)
    state = rc.state_of(m)
    sms = sm_count()
    worst = 0.0
    for B in rc.small_batches(sms):
        xt, t, x0, x1 = rc.action_batch(m, B, seed=B + w, act=act)
        m = m.to(DEV)
        base = [v.to(DEV) for v in (xt, t, x0, x1)]
        m.zero_grad(set_to_none=True)
        cfm_b200.action_matching_loss(m, *base).backward()
        g0 = [p.grad.clone() for p in m.parameters()]
        S = so.action_grad_scales(state, xt, t, x0, x1, act)
        grads, scales = rc.action_row_terms(state, dim, w, xt, t, x0, x1, act)
        for name, r in rc.positions_on(B, rc.TILE, sms).items():
            q = rc.swap_partner(B, r)
            swapped = [v.clone() for v in base]
            for v in swapped:
                v[r] = v[q]
            m.zero_grad(set_to_none=True)
            cfm_b200.action_matching_loss(m, *swapped).backward()
            change = [p.grad - a for p, a in zip(m.parameters(), g0)]
            ref, both = rc.swap_reference(S, grads, scales, B, r, q)
            gap = _entry_gap(change, ref, both)
            assert gap <= rc.SWAP_GATE, (B, name, r, q, gap)
            worst = max(worst, gap)
    print(f"margins rows action w={w} {act}: change/abs-scale {worst:.2e} (gate {rc.SWAP_GATE:.0e})")


# ---- the CNF backward: one row's cotangent per call ------------------------------------------------------------------
@pytest.mark.parametrize("dim,w,act", [(2, 32, "selu"), (2, 32, "silu"), (2, 64, "selu"), (2, 64, "silu"),
                                       (8, 64, "selu"), (8, 64, "silu")])
def test_cnf_backward_one_row_at_every_tile_height_and_position(dim, w, act):
    m = rc.cnf_model(dim, w, act)
    state = rc.state_of(m)
    m = m.to(DEV)
    sms = sm_count()
    batches = rc.cnf_batches(dim, w)
    assert [R for R, _ in batches] == [2, 4, 8, 8 if (dim, w) == (8, 64) else 16], batches
    span = rc.cnf_span()
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver="euler")
    worst = 0.0
    for R, B in batches:
        positions = rc.positions_on(B, R, sms)
        z, Gdraw = rc.cnf_inputs(state, dim, w, act, B, positions)
        z = z.to(DEV).requires_grad_(True)
        traj = node.trajectory(z, span)
        near = cto.kink_rows(state, traj.detach().cpu(), span) if act == "selu" else torch.zeros(B, dtype=torch.bool)
        for name, r in positions.items():
            assert not near[r], (B, name, r)
            G = torch.zeros_like(traj)
            G[:, r] = Gdraw[:, r].to(DEV)
            got = torch.autograd.grad(traj, list(m.parameters()) + [z], G, retain_graph=True)
            ref, scales = rc.one_row_cnf_reference(state, traj.detach(), span, G, r, act)
            gz = got[-1]
            assert torch.count_nonzero(gz[torch.arange(B, device=DEV) != r]) == 0, (B, name, r)
            gap = _entry_gap(list(got[:-1]) + [gz[r:r + 1]], ref, scales)
            assert gap <= rc.ROW_GATE, (R, B, name, r, gap)
            worst = max(worst, gap)
    print(f"margins rows cnf dim={dim} w={w} {act}: grad/abs-scale {worst:.2e} (gate {rc.ROW_GATE:.0e})")


# ---- the largest batches ---------------------------------------------------------------------------------------------
CHUNK = 1 << 16


def chunked_flow_reference(state, dim, out_dim, w, xt, t, ut, act):
    """(loss, gradients, scales) in float64 of the B-row flow-matching loss, summed over CHUNK-row slices: every
    gradient and scale is linear in the rows' terms with the factor 1 / B."""
    B = xt.shape[0]
    loss, grads, scales = 0.0, None, None
    for lo in range(0, B, CHUNK):
        sl = slice(lo, min(B, lo + CHUNK))
        n = sl.stop - lo
        rl, rg = ot.loss_and_grads(state, dim, out_dim, w, xt[sl], t[sl], ut[sl], act=act)
        sc = wo.grad_scales(state, dim, out_dim, w, xt[sl], t[sl], ut[sl], act=act)
        loss += rl.item() * n / B
        rg, sc = [g * (n / B) for g in rg], [s * (n / B) for s in sc]
        grads = rg if grads is None else [a + b for a, b in zip(grads, rg)]
        scales = sc if scales is None else [a + b for a, b in zip(scales, sc)]
    return loss, grads, scales


def _big_flow_case(dim, out_dim, w, act, B, seed):
    m = rc.make_model(dim, out_dim, w, act, seed=seed)
    xt, t, ut = rc.flow_batch(m, B, seed, act)
    m = m.to(DEV)
    m.zero_grad(set_to_none=True)
    loss = cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), ut.to(DEV))
    loss.backward()
    state = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    rl, rg, sc = chunked_flow_reference(state, dim, out_dim, w, xt, t, ut, act)
    lgap = abs(loss.item() - rl) / (rl + ut.double().pow(2).mean().item())
    gap = _entry_gap([p.grad for p in m.parameters()], rg, sc)
    rgap = max((p.grad.cpu().double() - r).abs().max().item() / r.abs().max().item()
               for p, r in zip(m.parameters(), rg))
    return lgap, gap, rgap


@pytest.mark.parametrize("w,act", [(32, "silu"), (64, "selu")])
def test_flow_matching_small_class_at_2_20_rows(w, act):
    """2^20 rows: each thread's register chain adds about 2^20 / (16 G) rows, 496 tiles on each of 132 CTAs."""
    lgap, gap, rgap = _big_flow_case(2, 2, w, act, 1 << 20, seed=340 + w)
    print(f"margins B=2^20 small w={w} {act}: loss {lgap:.2e} grad/abs-scale {gap:.2e} grad/max-abs {rgap:.2e}")
    assert lgap <= LOSS_REL and gap <= BIG_GATE and rgap <= GRAD_REL, (lgap, gap, rgap)


def test_flow_matching_tensor_core_class_at_2_18_rows():
    lgap, gap, rgap = _big_flow_case(64, 64, 256, "selu", 1 << 18, seed=350)
    print(f"margins B=2^18 tc: loss {lgap:.2e} grad/abs-scale {gap:.2e} grad/max-abs {rgap:.2e}")
    assert lgap <= LOSS_REL and gap <= BIG_GATE and rgap <= GRAD_REL, (lgap, gap, rgap)


def test_action_matching_at_2_20_rows():
    dim, w, act, B = 2, 64, "silu", 1 << 20
    m = rc.make_model(dim, 1, w, act, seed=360)
    xt, t, x0, x1 = rc.action_batch(m, B, seed=361, act=act)
    m = m.to(DEV)
    m.zero_grad(set_to_none=True)
    loss = cfm_b200.action_matching_loss(m, *(v.to(DEV) for v in (xt, t, x0, x1)))
    loss.backward()
    state = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    rl, grads, scales, lscale = 0.0, None, None, 0.0
    mc = ao.make_action(state, dim, w, act)
    for lo in range(0, B, CHUNK):
        sl = slice(lo, min(B, lo + CHUNK))
        f = (sl.stop - lo) / B
        cl, cg = ao.action_matching_loss_and_grads(state, dim, w, xt[sl], t[sl], x0[sl], x1[sl], act)
        cs = so.action_grad_scales(state, xt[sl], t[sl], x0[sl], x1[sl], act)
        rl += cl.item() * f
        lscale += ao.loss_scale(mc, xt[sl], t[sl], x0[sl], x1[sl]) * f
        cg, cs = [g * f for g in cg], [s * f for s in cs]
        grads = cg if grads is None else [a + b for a, b in zip(grads, cg)]
        scales = cs if scales is None else [a + b for a, b in zip(scales, cs)]
    lgap = abs(loss.item() - rl) / lscale
    gap = _entry_gap([p.grad for p in m.parameters()], grads, scales)
    rgap = max((p.grad.cpu().double() - r).abs().max().item() / r.abs().max().item()
               for p, r in zip(list(m.parameters())[:7], grads[:7]))  # b3's gradient and scale are exactly 0
    print(f"margins B=2^20 action: loss {lgap:.2e} grad/abs-scale {gap:.2e} grad/max-abs {rgap:.2e}")
    assert lgap <= LOSS_REL and gap <= BIG_GATE and rgap <= GRAD_REL, (lgap, gap, rgap)
