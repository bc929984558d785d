"""cfm_b200.action_matching_loss without a device: the float64 oracle (tests/action_oracle.py) against the notebook's
lines verbatim, a NumPy float64 restatement of the kernel's per-row algorithm (csrc/action_train.cu) against the
oracle, the Python wrapper's refusals (raised before any device call) and the library's argument errors (returned
before any CUDA call)."""
import ctypes
import re

import action_oracle as ao
import numpy as np
import pytest
import torch

import cfm_b200
from cfm_b200 import _ffi

ERR_ARG = -1  # CFM_ERR_ARG
_SELU_L, _SELU_A = 1.0507009873554804934193349852946, 1.6732632423543772848170429916717


def _state(dim, w, seed):
    torch.manual_seed(seed)
    return cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True).state_dict()


def _inputs(B, dim, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(B, dim, generator=g), torch.rand(B, 1, generator=g), torch.randn(B, dim, generator=g) * 2,
            torch.randn(B, dim, generator=g))


# ---- the oracle ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_oracle_is_the_notebook_lines(act):
    """The notebook's cell, verbatim, with float64 as the default dtype."""
    dim, w, batch_size = 2, 32, 7
    state = _state(dim, w, 0)
    xt0, t0, x0, x1 = _inputs(batch_size, dim, 1)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        action = ao.make_action(state, dim, w, act)
        x0, x1 = x0.double(), x1.double()
        t = t0.double().requires_grad_(True)
        xt = xt0.double().detach().requires_grad_(True)
        st = torch.sum(action(torch.cat([xt, t], dim=-1)))
        dsdx, dsdt = torch.autograd.grad(st, (xt, t), create_graph=True, retain_graph=True)
        xt.requires_grad, t.requires_grad = False, False
        a0 = action(torch.cat([x0, torch.zeros(batch_size, 1)], dim=-1))
        a1 = action(torch.cat([x1, torch.ones(batch_size, 1)], dim=-1))
        loss = (a0 - a1 + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt).mean()
        loss.backward()
    finally:
        torch.set_default_dtype(prev)
    rl, rg = ao.action_matching_loss_and_grads(state, dim, w, xt0, t0[:, 0], x0, x1, act)
    assert abs(loss.item() - rl.item()) <= 1e-14 * ao.loss_scale(action, xt0, t0, x0, x1)
    for p, r in zip(action.parameters(), rg):
        assert torch.allclose(p.grad, r, rtol=1e-13, atol=1e-15 * max(1.0, r.abs().max().item()))
    assert rg[7].item() == 0.0  # b3 cancels in a0 - a1 and does not enter ds


# ---- the kernel's algorithm, restated row by row in float64 ---------------------------------------------------------
def _act(x, act):
    """(act(x), act'(x), act''(x))"""
    if act == "selu":
        e = np.exp(np.minimum(x, 0.0))
        neg = x <= 0
        return (np.where(neg, _SELU_L * _SELU_A * (e - 1), _SELU_L * x), np.where(neg, _SELU_L * _SELU_A * e, _SELU_L),
                np.where(neg, _SELU_L * _SELU_A * e, 0.0))
    s = 1.0 / (1.0 + np.exp(-x))
    return x * s, s + x * s * (1 - s), s * (1 - s) * (2 + x * (1 - 2 * s))


def _restated(state, xt, t, x0, x1, act):
    """Loss and gradients by the kernel's steps: endpoints with cotangent +-1/B; at the middle point the forward, the
    reverse pass for g = grad s, the tangent forward along c = [g_x, 1] and its reverse pass; four (delta, a) pairs per
    layer and row, the tangent pair without a bias term."""
    Ws = [state[f"net.{k}.weight"].double().numpy() for k in (0, 2, 4, 6)]
    bs = [state[f"net.{k}.bias"].double().numpy() for k in (0, 2, 4)]
    xt, t, x0, x1 = (v.double().numpy() for v in (xt, t, x0, x1))
    B, dim = xt.shape
    gW = [np.zeros_like(W) for W in Ws]
    gb = [np.zeros_like(b) for b in bs]
    w3 = Ws[3][0]
    loss = 0.0

    def forward(z):
        h, d1, d2, a = z, [], [], [z]
        for W, b in zip(Ws[:3], bs):
            h, da, dda = _act(W @ h + b, act)
            d1.append(da), d2.append(dda), a.append(h)
        return a, d1, d2  # a = [z, h0, h1, h2]

    def accumulate(deltas, a, bias):
        for l in range(3):
            gW[l] += np.outer(deltas[l], a[l])
            if bias:
                gb[l] += deltas[l]

    for r in range(B):
        for z, cot in ((np.append(x0[r], 0.0), 1.0 / B), (np.append(x1[r], 1.0), -1.0 / B)):
            a, d1, _ = forward(z)
            loss += cot * B * (w3 @ a[3])
            delta = [None, None, d1[2] * w3 * cot]
            delta[1] = d1[1] * (Ws[2].T @ delta[2])
            delta[0] = d1[0] * (Ws[1].T @ delta[1])
            accumulate(delta, a, True)
            gW[3][0] += cot * a[3]
        a, d1, d2 = forward(np.append(xt[r], t[r]))
        g = [None, None, d1[2] * w3]
        m = [None, Ws[2].T @ g[2], None]
        g[1] = d1[1] * m[1]
        m[0] = Ws[1].T @ g[1]
        g[0] = d1[0] * m[0]
        gz = Ws[0].T @ g[0]
        loss += 0.5 * gz[:dim] @ gz[:dim] + gz[dim]
        c = np.append(gz[:dim], 1.0)
        hd, pd = [c], []
        for l in range(3):
            pd.append(Ws[l] @ hd[-1])
            hd.append(d1[l] * pd[-1])
        Q = [None, None, d2[2] * pd[2] * w3 / B]
        Q[1] = d1[1] * (Ws[2].T @ Q[2]) + d2[1] * pd[1] * m[1] / B
        Q[0] = d1[0] * (Ws[1].T @ Q[1]) + d2[0] * pd[0] * m[0] / B
        accumulate(Q, a, True)
        accumulate([gl / B for gl in g], hd, False)
        gW[3][0] += hd[3] / B
    return loss / B, [gW[0], gb[0], gW[1], gb[1], gW[2], gb[2], gW[3], np.zeros(1)]


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", [1, 3])
def test_restated_kernel_algorithm_matches_the_oracle(act, dim):
    w, B = 16, 5
    state = _state(dim, w, 2)
    xt, t, x0, x1 = _inputs(B, dim, 3)
    loss, grads = _restated(state, xt, t[:, 0], x0, x1, act)
    rl, rg = ao.action_matching_loss_and_grads(state, dim, w, xt, t, x0, x1, act)
    assert abs(loss - rl.item()) <= 1e-12 * ao.loss_scale(ao.make_action(state, dim, w, act), xt, t, x0, x1)
    for g, r in zip(grads, rg):
        assert g.shape == tuple(r.shape)
        assert np.abs(g - r.numpy()).max() <= 1e-12 * max(r.abs().max().item(), 1e-300), (g, r)


# ---- the Python wrapper: every refusal fires on the host ----------------------------------------------------------
def _args(B=4, dim=2):
    return torch.randn(B, dim), torch.rand(B), torch.randn(B, dim), torch.randn(B, dim)


@pytest.mark.parametrize("model", [
    torch.nn.Linear(3, 1),
    cfm_b200.MLP(dim=2, out_dim=1, w=64, time_varying=False),
    cfm_b200.MLP(dim=2, out_dim=1, w=128, time_varying=True),
    cfm_b200.MLP(dim=2, out_dim=1, w=16, time_varying=True),
    cfm_b200.MLP(dim=9, out_dim=1, w=64, time_varying=True),
    cfm_b200.MLP(dim=2, out_dim=2, w=64, time_varying=True),
], ids=["linear", "not_time_varying", "w128", "w16", "dim9", "out_dim2"])
def test_actions_outside_the_kernel_class_are_not_implemented(model):
    with pytest.raises(NotImplementedError, match=re.escape("w in {32, 64}, dim <= 8, out_dim = 1")):
        cfm_b200.action_matching_loss(model, *_args())


def test_shape_and_requires_grad_errors_are_value_errors():
    m = cfm_b200.MLP(dim=2, out_dim=1, w=64, time_varying=True)
    xt, t, x0, x1 = _args()
    for args in ((xt[:, :1], t, x0, x1), (xt, t[:3], x0, x1), (xt, torch.rand(4, 2), x0, x1), (xt, t, x0[:, :1], x1),
                 (xt, t, x0, x1[:3]), (xt.reshape(-1), t, x0, x1), (xt[:0], t[:0], x0[:0], x1[:0])):
        with pytest.raises(ValueError, match="action_matching_loss"):
            cfm_b200.action_matching_loss(m, *args)
    for k in range(4):
        args = list(_args())
        args[k] = args[k].requires_grad_(True)
        with pytest.raises(ValueError, match="requires grad"):
            cfm_b200.action_matching_loss(m, *args)


def test_cpu_tensors_and_non_fp32_parameters_raise_with_no_fallback():
    m = cfm_b200.MLP(dim=2, out_dim=1, w=64, time_varying=True)
    xt, t, x0, x1 = _args()
    with pytest.raises(_ffi.CfmLibraryError, match="no CPU fallback"):
        cfm_b200.action_matching_loss(m, xt, t, x0, x1)
    with pytest.raises(_ffi.CfmLibraryError):  # t as the notebook draws it, (B, 1), passes the shape checks
        cfm_b200.action_matching_loss(m, xt, t[:, None], x0, x1)
    with pytest.raises(_ffi.CfmLibraryError), torch.no_grad():
        cfm_b200.action_matching_loss(m, xt, t, x0, x1)
    with pytest.raises(_ffi.CfmLibraryError):
        cfm_b200.action_matching_loss(m.double(), *(v.double() for v in _args()))


# ---- the library: argument errors before any CUDA call ------------------------------------------------------------
def _call(lib, p, *, w=64, batch=256, ws_bytes=None, with_grad=1, grads=True, act=0, dim=2):
    if ws_bytes is None:
        ws_bytes = max(lib.cfm_mlp_small_train_workspace_bytes(batch, dim, w, 1), 1 << 20)
    return lib.cfm_mlp_small_action_grad_f32(p, p, p, p, p, p, p, p, dim, w, act, p, p, p, p, batch, with_grad, p,
                                             p if grads else None, p, ws_bytes, None)


def test_bad_arguments_are_refused_before_any_launch(lib_built):
    """Every case is an argument error found on the host.  The pointers are dummies that are never dereferenced."""
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    for kw, text in (({"w": 128}, b"unsupported shape"), ({"w": 16}, b"unsupported shape"),
                     ({"dim": 9}, b"unsupported shape"), ({"dim": 0}, b"unsupported shape"),
                     ({"batch": 0}, b"unsupported shape"), ({"ws_bytes": 16}, b"workspace too small"),
                     ({"grads": False}, b"with_grad needs a grads buffer"), ({"act": 7}, b"unknown activation")):
        assert _call(lib, p, **kw) == ERR_ARG, kw
        assert text in lib.cfm_last_error(), (kw, lib.cfm_last_error())
    for slot in list(range(8)) + [11, 12, 13, 14, 17, 19]:  # parameters, xt, t, x0, x1, loss, workspace
        args = [p] * 8 + [2, 64, 0] + [p] * 4 + [256, 1, p, p, p, 1 << 20, None]
        args[slot] = None
        assert lib.cfm_mlp_small_action_grad_f32(*args) == ERR_ARG, slot
        assert b"null pointer" in lib.cfm_last_error()
