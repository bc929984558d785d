"""cfm_b200.flow_matching_loss for wide MLPs on the device (csrc/train_tc.cu: fp16x3 tensor-core GEMMs, split-K weight
gradients) against oracle/train.py, the loss in float64 on the CPU with torch autograd.

Gates (DESIGN.md section 3.15): the loss within LOSS_REL of loss + mean(ut^2) (the residual is a difference, so its
rounding is relative to its terms), and every gradient entry within GRAD_ABS of its own absolute scale from
tests/wide_train_oracle.py.  As in test_gpu_train.py, SELU batches leave out rows whose float64 pre-activations lie
within _KINK_REL of SELU's kink, where the gradient is discontinuous in the weights."""
import subprocess
import re

import pytest
import torch

import cfm_b200
import wide_train_oracle as wo
from cfm_b200 import _ffi
from oracle import train as ot

DEV = "cuda:0"
gpu = pytest.mark.gpu

SHAPES = [(32, 32, 4), (40, 200, 12), (64, 256, 64), (784, 256, 784), (1024, 128, 8)]  # (dim, w, out_dim)
BATCHES = [1, 127, 128, 129, 1000, 8192]
LOSS_REL, GRAD_ABS = 2e-6, 1e-5
_KINK_REL = 1e-5
LAUNCHES_WITH_GRAD, LAUNCHES_LOSS_ONLY = 19, 8


def _model(dim, w, out_dim, act, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m.to(DEV)


def _away_from_kink(m, xt, t):
    mc = ot.make_model(m.state_dict(), m.dim, m.out_dim, m.w)
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
    g = torch.Generator().manual_seed(seed)
    n = B + max(64, B // 10)
    xt, t = torch.randn(n, m.dim, generator=g), torch.rand(n, generator=g)
    ut, s = torch.randn(n, m.out_dim, generator=g), torch.rand(n, generator=g) * 2.0
    if act == "selu":
        keep = _away_from_kink(m, xt, t)
        assert int(keep.sum()) >= B
        xt, t, ut, s = xt[keep], t[keep], ut[keep], s[keep]
    return xt[:B].clone(), t[:B].clone(), ut[:B].clone(), (s[:B].clone() if row_scale else None)


def _device(m, xt, t, ut, s=None):
    m.zero_grad(set_to_none=True)
    loss = cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), ut.to(DEV), None if s is None else s.to(DEV))
    loss.backward()
    return loss.detach(), [p.grad.detach().clone() for p in m.parameters()]


def _gaps(m, act, xt, t, ut, s=None):
    """(loss error over its scale, worst gradient error over its entry's absolute scale, worst max-abs-relative
    gradient error) against the float64 oracle."""
    loss, grads = _device(m, xt, t, ut, s)
    assert loss.shape == () and loss.dtype == torch.float32 and loss.is_cuda
    args = (m.state_dict(), m.dim, m.out_dim, m.w, xt, t, ut)
    rl, rg = ot.loss_and_grads(*args, row_scale=s, act=act)
    scales = wo.grad_scales(*args, row_scale=s, act=act)
    lgap = abs(loss.item() - rl.item()) / (rl.item() + ut.double().pow(2).mean().item())
    ggap = rgap = 0.0
    for p, g, r, sc in zip(m.parameters(), grads, rg, scales):
        assert g.shape == p.shape and torch.isfinite(g).all()
        err = (g.cpu().double() - r).abs()
        ggap = max(ggap, (err / sc.clamp_min(1e-300)).max().item())
        rgap = max(rgap, err.max().item() / r.abs().max().item())
    return lgap, ggap, rgap


# ---- every shape, both activations, every batch-size class -------------------------------------------------------
@gpu
@pytest.mark.parametrize("dim,w,out_dim", SHAPES)
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_loss_and_gradients_match_the_float64_oracle(act, dim, w, out_dim):
    m = _model(dim, w, out_dim, act, seed=100 + dim + w)
    worst = [0.0, 0.0, 0.0]
    for B in BATCHES:
        lgap, ggap, rgap = _gaps(m, act, *_batch(m, B, seed=B, act=act))
        assert lgap <= LOSS_REL and ggap <= GRAD_ABS, (B, lgap, ggap)
        worst = [max(a, b) for a, b in zip(worst, (lgap, ggap, rgap))]
    print(f"margins {act} dim={dim} w={w} out={out_dim}: loss {worst[0]:.2e} grad/abs-scale {worst[1]:.2e} "
          f"grad/max-abs {worst[2]:.2e}")


# batches one either side of split-K boundaries: for w = 32 every weight gradient is one output tile, so the slice
# count is min(chunks of 64 rows, 132) up to 132 chunks (8448 rows) and ceil(chunks / 2) slices of 2 chunks above;
# 1024 * 8 rows is where the accuracy cap of 8 chunks per slice starts to bind at 256-wide layers (6 tiles -> 22
# slices by occupancy, 8 chunks x 22 = 176 chunks = 11264 rows)
@gpu
@pytest.mark.parametrize("B", [63, 64, 65, 8447, 8448, 8449, 11263, 11264, 11265])
def test_batches_around_slice_boundaries(B):
    for dim, w, out_dim in ((32, 32, 4), (64, 256, 64)):
        m = _model(dim, w, out_dim, "selu", seed=B)
        lgap, ggap, _ = _gaps(m, "selu", *_batch(m, B, seed=B + 1, row_scale=True))
        assert lgap <= LOSS_REL and ggap <= GRAD_ABS, (dim, w, B, lgap, ggap)


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_large_batch(act):
    """65 536 rows: 128 slices of 8 chunks per weight gradient, every forward and delta GEMM on 512 row tiles."""
    m = _model(64, 256, 64, act, seed=8)
    lgap, ggap, rgap = _gaps(m, act, *_batch(m, 65536, seed=10, act=act, row_scale=True))
    assert lgap <= LOSS_REL and ggap <= GRAD_ABS, (lgap, ggap)
    print(f"margins B=65536 {act}: loss {lgap:.2e} grad/abs-scale {ggap:.2e} grad/max-abs {rgap:.2e}")


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_row_scale_with_zero_rows_and_the_score_loss(act):
    m = _model(40, 200, 12, act, seed=7)
    for B in (5, 300):
        xt, t, ut, s = _batch(m, B, seed=B, act=act, row_scale=True)
        s[::3] = 0.0  # a zero row adds ut^2 to the loss and nothing to any gradient
        lgap, ggap, _ = _gaps(m, act, xt, t, ut, s)
        assert lgap <= LOSS_REL and ggap <= GRAD_ABS, (B, lgap, ggap)
    eps = -ut
    mc = ot.make_model(m.state_dict(), 40, 12, 200, act)
    st = mc(torch.cat([xt, t[:, None]], -1).double())
    ref = torch.mean((s.double()[:, None] * st + eps.double()) ** 2)
    with torch.no_grad():
        got = cfm_b200.flow_matching_loss(m, xt.to(DEV), t.to(DEV), (-eps).to(DEV), row_scale=s.to(DEV))
    assert abs(got.item() - ref.item()) <= LOSS_REL * (ref.item() + eps.pow(2).mean().item())


@gpu
def test_every_row_uses_its_own_time():
    m = _model(32, 64, 8, "selu", seed=3)
    xt, _, ut, _ = _batch(m, 600, seed=1)
    t = torch.linspace(0.0, 1.0, 600)[torch.randperm(600, generator=torch.Generator().manual_seed(2))]
    keep = _away_from_kink(m, xt, t)
    xt, t, ut = xt[keep], t[keep], ut[keep]
    _, grads = _device(m, xt, t, ut)
    args = (m.state_dict(), 32, 8, 64, xt)
    _, rg = ot.loss_and_grads(*args, t, ut)
    sc = wo.grad_scales(*args, t, ut)[0][:, -1]
    col, ref = grads[0][:, -1].cpu().double(), rg[0][:, -1]
    assert ((col - ref).abs() / sc).max().item() <= GRAD_ABS
    _, shared = ot.loss_and_grads(*args, torch.full_like(t, t.mean().item()), ut)
    assert (col - shared[0][:, -1]).abs().max().item() > 1e-2 * ref.abs().max().item()


# ---- determinism, launches, stale workspaces ------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("B", [129, 8192])
def test_repeated_calls_give_the_same_bits_and_no_grad_gives_the_same_loss(B):
    m = _model(784, 256, 784, "selu", seed=5)
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
def test_fixed_launch_count_per_call_and_none_in_backward():
    m = _model(784, 256, 784, "selu", seed=5)
    xt, t, ut, _ = (None if v is None else v.to(DEV) for v in _batch(m, 1000, seed=9))
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()  # loads the kernels
    L = _ffi.lib()
    before = L.cfm_launch_count()
    loss = cfm_b200.flow_matching_loss(m, xt, t, ut)
    assert L.cfm_launch_count() - before == LAUNCHES_WITH_GRAD
    loss.backward()
    assert L.cfm_launch_count() - before == LAUNCHES_WITH_GRAD
    with torch.no_grad():
        cfm_b200.flow_matching_loss(m, xt, t, ut)
    assert L.cfm_launch_count() - before == LAUNCHES_WITH_GRAD + LAUNCHES_LOSS_ONLY


def _direct(m, xt, t, ut, ws, with_grad):
    L = _ffi.lib()
    params = [p.detach() for p in m.parameters()]
    loss = torch.full((), float("nan"), device=DEV)
    grads = torch.full((sum(p.numel() for p in params),), float("nan"), device=DEV)
    _ffi.check(L.cfm_mlp_tc_mse_grad_f32(
        *[_ffi.ptr(p) for p in params], m.dim, m.w, m.out_dim, m.act, _ffi.ptr(xt), _ffi.ptr(t), _ffi.ptr(ut), None,
        xt.shape[0], with_grad, _ffi.ptr(loss), _ffi.ptr(grads) if with_grad else None, _ffi.ptr(ws), ws.numel(),
        _ffi.stream_ptr()), "cfm_mlp_tc_mse_grad_f32")
    return loss, grads


@gpu
@pytest.mark.parametrize("B", [127, 1000])
def test_nan_filled_stale_workspace_gives_the_same_bits(B):
    m = _model(40, 200, 12, "silu", seed=11)
    xt, t, ut, _ = (None if v is None else v.to(DEV) for v in _batch(m, B, seed=12, act="silu"))
    nbytes = _ffi.lib().cfm_mlp_tc_train_workspace_bytes(B, 40, 200, 12)
    zero = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    stale = torch.full((nbytes // 4,), float("nan"), device=DEV).view(torch.uint8)
    for with_grad in (1, 0):
        a = _direct(m, xt, t, ut, zero, with_grad)
        b = _direct(m, xt, t, ut, stale, with_grad)
        assert torch.equal(a[0], b[0]) and torch.isfinite(a[0])
        if with_grad:
            assert torch.equal(a[1], b[1]) and torch.isfinite(a[1]).all()


# ---- the autograd contract ------------------------------------------------------------------------------------------
@gpu
def test_gradients_accumulate_scale_and_follow_in_place_updates():
    m = _model(64, 256, 64, "selu", seed=6)
    xt, t, ut, _ = (None if v is None else v.to(DEV) for v in _batch(m, 512, seed=4))
    _, g1 = _device(m, xt, t, ut)
    m.zero_grad(set_to_none=True)
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
    for p, g in zip(m.parameters(), g1):
        assert torch.equal(p.grad, g + g)
    m.zero_grad(set_to_none=True)
    (0.5 * cfm_b200.flow_matching_loss(m, xt, t, ut)).backward()
    for p, g in zip(m.parameters(), g1):
        assert torch.equal(p.grad, 0.5 * g)
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    before = cfm_b200.flow_matching_loss(m, xt, t, ut)
    opt.zero_grad()
    before.backward()
    torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
    opt.step()  # in place: the next call must split the new weights
    lgap, ggap, _ = _gaps(m, "selu", xt.cpu(), t.cpu(), ut.cpu())
    assert lgap <= LOSS_REL and ggap <= GRAD_ABS, (lgap, ggap)
    with torch.no_grad():
        after = cfm_b200.flow_matching_loss(m, xt, t, ut)
    assert after.item() < before.item()
    m.zero_grad(set_to_none=True)
    m.net[0].bias.requires_grad_(False)
    cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
    assert m.net[0].bias.grad is None and m.net[0].weight.grad is not None


# ---- training ---------------------------------------------------------------------------------------------------------
@gpu
def test_twenty_adam_steps_of_ot_cfm_track_float64_training_and_the_model_samples():
    """OT-CFM on MNIST-shaped synthetic batches (784 pixels in [-1, 1], B = 256): 20 Adam steps through
    flow_matching_loss against the same steps in float64 on the same pairs; the trained model then samples through
    NeuralODE(torch_wrapper(model)) on the fused tensor-core forward."""
    g = torch.Generator().manual_seed(0)
    m = _model(784, 256, 784, "selu", seed=1)
    mc = ot.make_model(m.state_dict(), 784, 784, 256)
    opt, optc = torch.optim.Adam(m.parameters(), lr=1e-4), torch.optim.Adam(mc.parameters(), lr=1e-4)
    fm = cfm_b200.ExactOptimalTransportConditionalFlowMatcher(sigma=0.0)
    protos = torch.rand(10, 784, generator=g) * 2 - 1
    for _ in range(20):
        x1 = (protos[torch.randint(0, 10, (256,), generator=g)] + 0.1 * torch.randn(256, 784, generator=g)).clamp(-1, 1)
        x0 = torch.randn(256, 784, generator=g)
        t, xt, ut = fm.sample_location_and_conditional_flow(x0.to(DEV), x1.to(DEV))
        opt.zero_grad()
        cfm_b200.flow_matching_loss(m, xt, t, ut).backward()
        opt.step()
        optc.zero_grad()
        ot.loss_of(mc, xt, t, ut).backward()
        optc.step()
    for p, r in zip(m.parameters(), mc.parameters()):
        # Adam normalises each step to ~lr per entry: compare the parameter change against 20 steps of lr
        assert (p.detach().cpu().double() - r.detach()).abs().max().item() <= 1e-2 * 20 * 1e-4
    node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(m), solver="dopri5", atol=1e-4, rtol=1e-4)
    with torch.no_grad():
        traj = node.trajectory(torch.randn(256, 784, generator=g).to(DEV), torch.linspace(0, 1, 2, device=DEV))
    assert m.tc_path(256) and torch.isfinite(traj).all() and traj.shape == (2, 256, 784)


# ---- the compiled instantiations -----------------------------------------------------------------------------------
def test_compiled_training_gemm_instantiations(lib_built):
    """The training GEMMs take the split-K-capable entry with their own epilogues; the cost-matrix and per-layer MLP
    instantiations keep gemm_wg_kernel (test_gpu_tensor_core_gemms.py guards those).  No device needed."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    epis = {re.search(r"(Tc\w+?Epi)E", s).group(1) for s in set(re.findall(r"\w*gemm_wg_splitk_kernel\w*", out))}
    assert epis == {"TcHiddenEpi", "TcOutEpi", "TcDeltaEpi", "TcGradEpi"}
