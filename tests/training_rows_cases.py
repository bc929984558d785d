"""TEST INFRASTRUCTURE ONLY -- the cases of tests/test_gpu_training_rows.py without a device: the launch rules of the
four training kernels restated from their sources, the row positions they give, the models and inputs of every case
(built on the CPU from seeds), the float64 one-row references and the gates.  tests/test_train_scale_host.py checks
on these same inputs that the gates can see one row lost or counted twice.

Launch rules: mlp_train_kernel and mlp_action_train_kernel (train_small.cuh: ctas_for, launch_folded's co-residency
clamp; 16-row tiles, one row pair per warp, CTA c takes tiles c, c + G, ...), cnf_euler_backward_kernel (cnf_train.cu:
cnf_back_rows, back_ctas) and the split-K weight gradients of train_tc.cu (slicing, 64-row K-chunks)."""
import torch

import action_oracle as ao
import cnf_train_oracle as cto
import train_scale_oracle as so
import wide_train_oracle as wo
from oracle import train as ot

import cfm_b200
from cfm_b200 import _ffi

ROW_GATE = 1e-6     # one-row gradients, of each entry's absolute scale (flow matching, both classes, and CNF)
SWAP_GATE = 5e-8    # action matching: the change of the gradient, of the sum of both calls' scales
_KINK_REL = 1e-5

# ---- the launch rules, restated --------------------------------------------------------------------------------------
MAX_CTAS = 132      # kMaxCtas, train_small.cuh
TILE = 16           # kTile: 8 warps x one row pair
SMEM_BUDGET = 227 * 1024  # kSmemBudget, cnf_train.cu
HK, TM, TN = 64, 128, 128  # K-chunk and output tile of the tensor-core GEMM core (gemm_h3.cuh, gemm_tc.cuh)
SLICE_MAX_CHUNKS, SLICE_TARGET = 8, 132  # kSliceMaxChunks, kSliceTargetItems, train_tc.cu
# 256-thread CTAs of the folded kernels that one SM can hold: every instantiation uses 94 to 167 registers per thread
# (ptxas -v), so the 64 K registers of an SM take at most two, and their shared-memory plans allow at least one
MAX_CTAS_PER_SM = 2


def co_resident_grids(B, R, sms):
    """The grids a folded launch of R-row tiles can get: one CTA per tile, at most MAX_CTAS, clamped to the CTAs the
    device holds at once, per_sm * sms with per_sm = 1 or 2 as the occupancy query finds.  With 132 SMs or more the
    clamp cannot bind and there is one grid."""
    return sorted({min(-(-B // R), MAX_CTAS, k * sms) for k in range(1, MAX_CTAS_PER_SM + 1)})


def tile_positions(B, R, G):
    """{name: row} of the row-loop positions that exist at batch B for R-row tiles on G CTAs."""
    ntiles = -(-B // R)
    pos = {"first row of a warp pair": 0, "batch's last row": B - 1}
    if B > 1:
        pos["second row of a warp pair"] = 1
    if B >= R:
        pos["last row of a tile"] = R - 1
    if G > 1:
        pos["first row of CTA G-1"] = R * (G - 1)
    if ntiles > G:
        pos["first row of CTA 0's second pass"] = R * G
    tail = B - R * (ntiles - 1)
    if tail < R and tail % 2 == 1:
        pos["lone valid row of an odd partial tile"] = B - 1
    return pos


def positions_on(B, R, sms):
    """tile_positions for every grid the device may give (named with G where there is more than one)."""
    grids = co_resident_grids(B, R, sms)
    if len(grids) == 1:
        return tile_positions(B, R, grids[0])
    return {f"{name} (G={G})": r for G in grids for name, r in tile_positions(B, R, G).items()}


def small_batches(sms):
    """A batch of 3 tiles ending in an odd partial tile, and one where CTA 0 takes a second, full tile and CTA 1 a
    second, partial one of 5 rows."""
    G = min(MAX_CTAS, sms)
    return [2 * TILE + 5, (G + 1) * TILE + 5]


def cnf_plan_bytes(dim, w, R):
    """cnf_back_plan(dim, w, R).total: weights and the tile's stash, every block rounded up to 4 floats."""
    vrows = (1 + dim) * R
    blocks = [(dim + 1) * w, w, w, w, w * w, w * w, w * w, w * w, dim * w, vrows * 16] + [vrows * w] * 6 + [R * 16] * 2
    return 4 * sum(-(-n // 4) * 4 for n in blocks)


def cnf_back_rows(B, dim, w):
    r = 2
    while r < TILE and r * MAX_CTAS < B:
        r *= 2
    while r >= 2:
        if cnf_plan_bytes(dim, w, r) <= SMEM_BUDGET:
            return r
        r //= 2
    return 0


def cnf_batches(dim, w):
    """[(R, B)]: for R = 2, 4, 8 the most rows that still give R, with a last tile of odd length, and a batch past 133
    tiles of 16 rows, where R = 16 or, if that stash does not fit, its cap; CTA 0 then takes a second tile."""
    return [(cnf_back_rows(B, dim, w), B)
            for B in (2 * MAX_CTAS - 1, 4 * MAX_CTAS - 1, 8 * MAX_CTAS - 3, (MAX_CTAS + 1) * TILE + 5)]


def slicing(B, n0, n1):
    """(slices, chunks per slice) of a split-K weight-gradient GEMM with K = B."""
    nk = -(-B // HK)
    tiles = -(-n0 // TM) * -(-n1 // TN)
    s = max(-(-nk // SLICE_MAX_CHUNKS), min(nk, -(-SLICE_TARGET // tiles)))
    chunks = -(-nk // s)
    return -(-nk // chunks), chunks


def tc_positions(B, dim, w, out_dim):
    """{name: row}: the first rows of GEMM M-tiles and K-chunks, and each layer's slice edges."""
    pos = {f"row {r}": r for r in (0, 63, 64, 127, 128) if r < B}
    pos["batch's last row"] = B - 1
    for l, (n0, n1) in enumerate(((w, dim + 2), (w, w + 1), (w, w + 1), (out_dim, w + 1))):
        slices, chunks = slicing(B, n0, n1)
        for k in (1, slices - 1):
            if 0 < k < slices:
                edge = k * chunks * HK
                pos[f"dW{l} slice {k - 1} last row"] = edge - 1
                pos[f"dW{l} slice {k} first row"] = edge
    return pos


def swap_partner(B, r):
    return (r + B // 2) % B if B > 1 else r


# ---- the cases' models and inputs, on the CPU ------------------------------------------------------------------------
TC_SHAPE, TC_BATCHES = (64, 256, 64), ((5001, "occupancy"), (40003, "cap"))
CNF_SPAN = 4  # t_span = linspace(1, 0, CNF_SPAN)


def make_model(dim, out_dim, w, act, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m


def flow_small_model(w, act):
    return make_model(2, 2, w, act, seed=300 + w)


def flow_tc_model(act):
    dim, w, out_dim = TC_SHAPE
    return make_model(dim, out_dim, w, act, seed=310)


def action_model(w, act):
    return make_model(2, 1, w, act, seed=320 + w)


def cnf_model(dim, w, act):
    return make_model(dim, dim, w, act, seed=330 + dim + w)


def state_of(m):
    return {k: v.detach().cpu() for k, v in m.state_dict().items()}


def away_from_kink(state, dim, out_dim, w, z):
    """Rows of z (B, dim + 1) whose float64 hidden pre-activations all stay further than _KINK_REL of their magnitude
    sum from SELU's kink."""
    mc = ot.make_model(state, dim, out_dim, w)
    with torch.no_grad():
        h = z.double()
        keep = torch.ones(h.shape[0], dtype=torch.bool)
        for li in (0, 2, 4):
            W, b = mc.net[li].weight, mc.net[li].bias
            p = h @ W.T + b
            keep &= (p.abs() > _KINK_REL * (h.abs() @ W.abs().T + b.abs())).all(1)
            h = mc.net[li + 1](p)
    return keep


def flow_batch(m, B, seed, act):
    g = torch.Generator().manual_seed(seed)
    n = B + max(64, B // 5)
    xt, t, ut = torch.randn(n, m.dim, generator=g) * 1.5, torch.rand(n, generator=g), torch.randn(n, m.out_dim,
                                                                                                   generator=g)
    if act == "selu":
        keep = away_from_kink(state_of(m), m.dim, m.out_dim, m.w, torch.cat([xt, t[:, None]], 1))
        assert int(keep.sum()) >= B
        xt, t, ut = xt[keep], t[keep], ut[keep]
    return xt[:B].clone(), t[:B].clone(), ut[:B].clone()


def action_batch(m, B, seed, act):
    g = torch.Generator().manual_seed(seed)
    n = B + max(64, B // 10)
    x0, x1 = torch.randn(n, m.dim, generator=g) * 1.5, torch.randn(n, m.dim, generator=g) * 1.5 + 1.0
    t = torch.rand(n, 1, generator=g)
    xt = t * x1 + (1 - t) * x0
    if act == "selu":
        s = state_of(m)
        keep = (away_from_kink(s, m.dim, 1, m.w, torch.cat([xt, t], 1))
                & away_from_kink(s, m.dim, 1, m.w, torch.cat([x0, torch.zeros(n, 1)], 1))
                & away_from_kink(s, m.dim, 1, m.w, torch.cat([x1, torch.ones(n, 1)], 1)))
        assert int(keep.sum()) >= B
        xt, t, x0, x1 = xt[keep], t[keep], x0[keep], x1[keep]
    return tuple(v[:B].clone() for v in (xt, t, x0, x1))


def cnf_span():
    return torch.linspace(1, 0, CNF_SPAN)


def cnf_inputs(state, dim, w, act, B, positions):
    """(z (B, dim + 1), the cotangent draw (CNF_SPAN, B, dim + 1)) of a CNF case; each call gives G = this draw on
    one row and 0 elsewhere.  With SELU, a tested row whose float64 Euler path passes near the kink takes the initial
    state of a row that does not."""
    g = torch.Generator().manual_seed(B)
    z, Gdraw = torch.randn(B, dim + 1, generator=g), torch.randn(CNF_SPAN, B, dim + 1, generator=g)
    if act == "selu":
        near = cto.kink_rows(state, euler_states(state, dim, w, act, z, cnf_span()), cnf_span())
        z = donate_away_from_kink(z, near, positions)
    return z, Gdraw


def donate_away_from_kink(z, near, positions):
    """z with every tested row that is ``near`` ((B,) bool) given the initial state of a row that is not and lies
    further than 2 rows from every tested row."""
    z = z.clone()
    donor = ~near
    for r in positions.values():
        donor[max(0, r - 2):r + 3] = False
    donors = iter(torch.nonzero(donor)[:, 0].tolist())
    for r in positions.values():
        if near[r]:
            z[r] = z[next(donors)]
    return z


def euler_states(state, dim, w, act, z, span):
    """(n_span, B, dim + 1) float64 Euler states of x; the likelihood column is left 0 (the adjoint does not read
    it).  The device's fp32 states are within rounding of these."""
    mc = ot.make_model(state, dim, dim, w, act)
    x = z[:, :dim].double()
    out = [x]
    span = span.double()
    with torch.no_grad():
        for a, b in zip(span[:-1], span[1:]):
            x = x + (b - a) * mc(torch.cat([x, torch.full_like(x[:, :1], float(a))], 1))
            out.append(x)
    return torch.cat([torch.stack(out), torch.zeros(len(out), z.shape[0], 1, dtype=torch.float64)], 2)


# ---- float64 one-row references --------------------------------------------------------------------------------------
def one_row_flow_reference(state, dim, out_dim, w, xt, t, ut, r, act):
    """(loss, gradients, scales) in float64 of the B-row loss with row_scale = 1 on row r and 0 elsewhere: the
    gradients and scales of row r alone times 1 / B, and the loss with the other rows' ut^2."""
    B = xt.shape[0]
    one = slice(r, r + 1)
    rl, rg = ot.loss_and_grads(state, dim, out_dim, w, xt[one], t[one], ut[one], act=act)
    sc = wo.grad_scales(state, dim, out_dim, w, xt[one], t[one], ut[one], act=act)
    rest = ut.double().pow(2).sum().item() - ut[r].double().pow(2).sum().item()
    loss = (rl.item() + rest / out_dim) / B
    return loss, [g / B for g in rg], [s / B for s in sc]


def action_row_terms(state, dim, w, xt, t, x0, x1, act):
    """Per-row float64 gradients and scales as functions of a row index: the B-row loss is the mean of one-row
    losses, so a row adds (its one-row gradient) / B."""
    def grads(i):
        one = slice(i, i + 1)
        return ao.action_matching_loss_and_grads(state, dim, w, xt[one], t[one], x0[one], x1[one], act)[1]

    def scales(i):
        one = slice(i, i + 1)
        return so.action_grad_scales(state, xt[one], t[one], x0[one], x1[one], act)
    return grads, scales


def swap_reference(S, grads, scales, B, r, q):
    """(float64 change of the gradient when row r takes row q's values, the sum of both calls' scales)"""
    gq, gr, sq, sr = grads(q), grads(r), scales(q), scales(r)
    return [(a - b) / B for a, b in zip(gq, gr)], [2 * s + (a - b) / B for s, a, b in zip(S, sq, sr)]


def one_row_cnf_reference(state, traj, span, Gdraw, r, act):
    """(gradients + [z's gradient of row r], scales) in float64 for the cotangent Gdraw on row r alone."""
    one = slice(r, r + 1)
    t1, G1 = traj[:, one].detach().cpu(), Gdraw[:, one].detach().cpu()
    ref_p, ref_z = cto.restated_backward(state, t1, span, G1, act, h32=True)
    sc_p, sc_z = so.cnf_grad_scales(state, t1, span, G1, act)
    return list(ref_p) + [ref_z], list(sc_p) + [sc_z]
