"""Gradients through the exact-likelihood Euler trajectory without a device: the float64 restatement of the discrete
adjoint (tests/cnf_train_oracle.py) against torch's autograd through the float64 Euler loop, the library's backward
planner and argument errors (returned before any CUDA call), the header against the binding, and the wrapper's
refusals."""
import ctypes
import os
import re

import pytest
import torch

import cnf_oracle as co
import cnf_train_oracle as cto
from conftest import ROOT
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

ERR_ARG = -1  # CFM_ERR_ARG
NAMES = ["net.0.weight", "net.0.bias", "net.2.weight", "net.2.bias", "net.4.weight", "net.4.bias", "net.6.weight",
         "net.6.bias"]


def _state(dim, w, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
    return {k: v.double().requires_grad_(True) for k, v in m.state_dict().items()}


def _span(n, direction):
    s = torch.linspace(0, 1, n, dtype=torch.float64)
    return s.flip(0) if direction == "reverse" else s


def _autograd(state, z, span, G, act):
    f = co.cnf_field(lambda inp: vf.mlp_forward_from_state(state, inp, act=act))
    traj = cto.euler_loop(f, z, span)
    grads = torch.autograd.grad((traj * G).sum(), [state[k] for k in NAMES] + [z])
    return traj, grads[:-1], grads[-1]


@pytest.mark.parametrize("direction", ["forward", "reverse"])
def test_euler_loop_is_the_oracle_trajectory(direction):
    state = _state(2, 16, 0)
    f = co.cnf_field(lambda inp: vf.mlp_forward_from_state(state, inp))
    z = torch.randn(7, 3, dtype=torch.float64)
    span = _span(6, direction)
    with torch.no_grad():
        assert torch.equal(cto.euler_loop(f, z, span), co.euler_any_direction(f, z, span))


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", [1, 2, 5, 8])
@pytest.mark.parametrize("direction", ["forward", "reverse"])
def test_restated_adjoint_matches_autograd_through_the_euler_loop(act, dim, direction):
    """Cotangents on the last state, on two inner checkpoints (one with the x columns only, one with the log-density
    column only) and none on the others."""
    state = _state(dim, 16, dim)
    g = torch.Generator().manual_seed(10 + dim)
    z = torch.randn(6, dim + 1, dtype=torch.float64, generator=g).requires_grad_(True)
    span = _span(5, direction)
    G = torch.randn(5, 6, dim + 1, dtype=torch.float64, generator=g)
    G[0] = 0.0
    G[1, :, dim] = 0.0
    G[2, :, :dim] = 0.0
    G[3] = 0.0
    traj, ref_p, ref_z = _autograd(state, z, span, G, act)
    got_p, got_z = cto.restated_backward({k: v.detach() for k, v in state.items()}, traj.detach(), span, G, act)
    for name, a, b in zip(NAMES + ["z"], list(got_p) + [got_z], list(ref_p) + [ref_z]):
        assert a.shape == b.shape, name
        scale = max(b.abs().max().item(), 1e-300)
        assert (a - b).abs().max().item() <= 1e-12 * scale, (name, (a - b).abs().max().item(), scale)


def test_gradcheck_of_the_float64_oracle():
    dim, w = 2, 4
    state = _state(dim, w, 3)
    z = torch.randn(3, dim + 1, dtype=torch.float64).requires_grad_(True)
    span = _span(3, "reverse")

    def fn(z, *params):
        st = dict(zip(NAMES, params))
        f = co.cnf_field(lambda inp: vf.mlp_forward_from_state(st, inp, act="silu"))
        return cto.euler_loop(f, z, span)

    assert torch.autograd.gradcheck(fn, (z, *[state[k] for k in NAMES]))


# ---- the library: planner, workspace and argument errors, all on the host -----------------------------------------
def test_backward_supported_table(lib_built):
    lib = _ffi.load_library(lib_built)
    for w in (16, 32, 64, 128):
        for dim in range(0, 10):
            for B in (0, 1, 2, 17, 256, 4096, 1 << 20):
                want = (w in (32, 64) and 1 <= dim <= 8 and B >= 1
                        and bool(lib.cfm_ode_small_cnf_supported(B, dim, w)))
                assert bool(lib.cfm_ode_small_cnf_backward_supported(B, dim, w)) == want, (w, dim, B)
    assert lib.cfm_ode_small_cnf_backward_supported(256, 2, 64)  # the tutorial's shape
    assert lib.cfm_ode_small_cnf_backward_supported(4096, 8, 64)
    assert not lib.cfm_ode_small_cnf_backward_supported(1 << 40, 2, 64)  # past the forward's planner


def test_backward_workspace_is_monotone(lib_built):
    lib = _ffi.load_library(lib_built)
    prev = 0
    for w in (32, 64):
        for dim in range(1, 9):
            for B in (1, 256, 4096):
                for n in (2, 101):
                    nb = lib.cfm_ode_small_cnf_backward_workspace_bytes(B, n, dim, w)
                    assert nb >= prev, (w, dim, B, n)
                    prev = nb
    n_params = 64 * 9 + 64 + 2 * (64 * 64 + 64) + 8 * 64 + 8
    assert prev >= 132 * n_params * 4  # one partial gradient vector per CTA


def _call(lib, p, *, w=64, dim=2, batch=256, n_span=101, ws_bytes=None, act=0, grads=True):
    if ws_bytes is None:
        ws_bytes = lib.cfm_ode_small_cnf_backward_workspace_bytes(batch, n_span, dim, w)
    return lib.cfm_ode_small_cnf_euler_backward_f32(p, p, p, p, p, p, p, p, dim, w, act, p, batch, p, n_span, p, p,
                                                    p if grads else None, p, ws_bytes, None)


def test_bad_arguments_are_refused_before_any_launch(lib_built):
    """Every case is an argument error found on the host.  The pointers are dummies that are never dereferenced."""
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    for kw, text in (({"w": 128}, b"unsupported shape"), ({"w": 16}, b"unsupported shape"),
                     ({"dim": 9}, b"unsupported shape"), ({"dim": 0}, b"unsupported shape"),
                     ({"batch": 0}, b"unsupported shape"), ({"batch": 1 << 40}, b"unsupported shape"),
                     ({"n_span": 1}, b"n_span"), ({"ws_bytes": 16}, b"workspace too small"),
                     ({"act": 7}, b"unknown activation"), ({"grads": False}, b"null pointer")):
        assert _call(lib, p, **kw) == ERR_ARG, kw
        assert text in lib.cfm_last_error(), (kw, lib.cfm_last_error())
    for slot in list(range(8)) + [11, 13, 15, 18]:  # parameters, traj, t_span, grad_traj, workspace
        args = [p] * 8 + [2, 64, 0, p, 256, p, 101, p, p, p, p, 1 << 22, None]
        args[slot] = None
        assert lib.cfm_ode_small_cnf_euler_backward_f32(*args) == ERR_ARG, slot
        assert b"null pointer" in lib.cfm_last_error()


def test_header_declares_what_the_binding_binds():
    with open(os.path.join(ROOT, "include", "cfm_b200.h")) as f:
        header = f.read()
    for name in ("cfm_ode_small_cnf_backward_supported", "cfm_ode_small_cnf_backward_workspace_bytes",
                 "cfm_ode_small_cnf_euler_backward_f32"):
        m = re.search(r"\b(int|size_t)\s+" + name + r"\(([^)]*)\)", header)
        assert m, name
        res, args = _ffi.SIGNATURES[name]
        assert (res is _ffi._sz) == (m.group(1) == "size_t"), name
        assert len([a for a in m.group(2).split(",") if a.strip()]) == len(args), name
    assert _ffi.SIGNATURES["cfm_ode_small_cnf_backward_supported"][1] == [_ffi._i64, _ffi._i, _ffi._i]
    assert "#define CFM_ABI_VERSION 2" in header


# ---- the wrapper's refusals without a device ------------------------------------------------------------------------
def _node(solver="euler", w=64, dim=2):
    torch.manual_seed(0)
    m = cfm_b200.MLP(dim=dim, w=w, time_varying=True)
    return cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, "exact"), solver=solver, sensitivity="adjoint"), m


def test_t_span_requiring_grad_is_a_value_error():
    node, _ = _node()
    with pytest.raises(ValueError, match="t_span requires grad"):
        node.trajectory(torch.zeros(4, 3), torch.linspace(1, 0, 5).requires_grad_(True))


@pytest.mark.parametrize("solver,w,B,text", [
    ("dopri5", 64, 4, "adaptive dopri5 solve are not implemented; use solver='euler'"),
    ("euler", 128, 4, "w=128"),
    ("euler", 64, 1 << 40, "B=1099511627776"),
])
def test_the_node_outside_the_class_names_its_reason(solver, w, B, text):
    node, m = _node(solver, w)
    x = torch.empty(B, 3, device="meta") if B > 4096 else torch.zeros(B, 3)
    assert text in node._cnf_backward_gap(m, x)
    euler, m = _node()
    assert euler._cnf_backward_gap(m, torch.zeros(256, 3)) is None


def test_no_fallback_on_the_cpu_under_autograd():
    node, _ = _node()
    with pytest.raises(_ffi.CfmLibraryError, match="needs CUDA inputs"):
        node.trajectory(torch.zeros(4, 3), torch.linspace(1, 0, 5))
    node.vf = cfm_b200.cnf_wrapper(node.vf.model, "hutch_gaussian")
    with pytest.raises(NotImplementedError, match="Hutchinson"):
        node.trajectory(torch.zeros(4, 3), torch.linspace(1, 0, 5))
