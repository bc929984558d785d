"""cfm_b200.flow_matching_loss without a device: which shapes the training kernel takes, the library's argument
errors (returned before any CUDA call), the Python wrapper's refusals (raised before any device call), and the float64
oracle against a hand-computed case and against torch.autograd.gradcheck."""
import ctypes
import re

import pytest
import torch

import cfm_b200
from cfm_b200 import _ffi
from oracle import train as ot

ERR_ARG = -1  # CFM_ERR_ARG


@pytest.mark.parametrize("w", [16, 32, 64, 128])
@pytest.mark.parametrize("dim", [1, 8, 9])
@pytest.mark.parametrize("out_dim", [1, 8, 9])
def test_supported_truth_table(lib_built, w, dim, out_dim):
    lib = _ffi.load_library(lib_built)
    want = w in (32, 64) and dim <= 8 and out_dim <= 8
    for batch in (1, 255, 1 << 20):  # rows stream from device memory: the batch does not enter
        assert bool(lib.cfm_mlp_small_train_supported(batch, dim, w, out_dim)) == want
    assert not lib.cfm_mlp_small_train_supported(0, dim, w, out_dim)
    assert (lib.cfm_mlp_small_train_workspace_bytes(256, dim, w, out_dim) > 0) == want


def test_workspace_is_positive_and_non_decreasing_in_batch(lib_built):
    lib = _ffi.load_library(lib_built)
    for w, dim, out_dim in ((32, 1, 1), (64, 2, 2), (64, 8, 8)):
        sizes = [lib.cfm_mlp_small_train_workspace_bytes(b, dim, w, out_dim)
                 for b in (1, 2, 16, 17, 255, 256, 257, 4096, 65536, 1 << 24)]
        assert sizes[0] > 0 and sizes == sorted(sizes)
        n_params = w * (dim + 1) + w + 2 * (w * w + w) + out_dim * w + out_dim
        assert sizes[0] >= 4 * n_params + 8  # one CTA's partial gradients and its float64 loss partial


def _call(lib, p, *, w=64, batch=256, ws_bytes=None, with_grad=1, grads=True, act=0, dim=2, out_dim=2):
    if ws_bytes is None:
        ws_bytes = max(lib.cfm_mlp_small_train_workspace_bytes(batch, dim, w, out_dim), 1 << 20)
    return lib.cfm_mlp_small_mse_grad_f32(p, p, p, p, p, p, p, p, dim, w, out_dim, act, p, p, p, None, batch, with_grad,
                                          p, p if grads else None, p, ws_bytes, None)


def test_bad_arguments_are_refused_before_any_launch(lib_built):
    """Every case is an argument error found on the host.  The pointers are dummies that are never dereferenced."""
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    for kw, text in (({"w": 128}, b"unsupported shape"), ({"w": 16}, b"unsupported shape"),
                     ({"dim": 9}, b"unsupported shape"), ({"out_dim": 9}, b"unsupported shape"),
                     ({"batch": 0}, b"unsupported shape"), ({"ws_bytes": 16}, b"workspace too small"),
                     ({"grads": False}, b"with_grad needs a grads buffer"), ({"act": 7}, b"unknown activation")):
        assert _call(lib, p, **kw) == ERR_ARG, kw
        assert text in lib.cfm_last_error(), (kw, lib.cfm_last_error())
    assert lib.cfm_mlp_small_mse_grad_f32(None, p, p, p, p, p, p, p, 2, 64, 2, 0, p, p, p, None, 256, 1, p, p, p,
                                          1 << 20, None) == ERR_ARG
    assert b"null pointer" in lib.cfm_last_error()


# ---- the Python wrapper: every refusal fires on the host ----------------------------------------------------------
def _inputs(B=4, dim=2, out_dim=2):
    return torch.randn(B, dim), torch.rand(B), torch.randn(B, out_dim)


@pytest.mark.parametrize("model", [
    torch.nn.Linear(3, 2),
    cfm_b200.MLP(dim=2, w=64, time_varying=False),
    cfm_b200.MLP(dim=2, w=128, time_varying=True),
    cfm_b200.MLP(dim=2, w=16, time_varying=True),
    cfm_b200.MLP(dim=9, w=64, time_varying=True),
    cfm_b200.MLP(dim=2, out_dim=9, w=64, time_varying=True),
], ids=["linear", "not_time_varying", "w128", "w16", "dim9", "out_dim9"])
def test_models_outside_the_kernel_class_are_not_implemented(model):
    with pytest.raises(NotImplementedError, match=re.escape("w in {32, 64}, dim <= 8")):
        cfm_b200.flow_matching_loss(model, *_inputs())


def test_shape_and_requires_grad_errors_are_value_errors():
    m = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    xt, t, ut = _inputs()
    for args in ((xt[:, :1], t, ut), (xt, t[:, None], ut), (xt, t[:3], ut), (xt, t, ut[:, :1]), (xt, t, ut[:3]),
                 (xt.reshape(-1), t, ut), (xt[:0], t[:0], ut[:0])):
        with pytest.raises(ValueError):
            cfm_b200.flow_matching_loss(m, *args)
    with pytest.raises(ValueError, match="row_scale"):
        cfm_b200.flow_matching_loss(m, xt, t, ut, row_scale=torch.ones(3))
    with pytest.raises(ValueError, match="requires grad"):
        cfm_b200.flow_matching_loss(m, xt.clone().requires_grad_(True), t, ut)
    with pytest.raises(ValueError, match="requires grad"):
        cfm_b200.flow_matching_loss(m, xt, t, ut, row_scale=torch.ones(4, requires_grad=True))


def test_cpu_tensors_and_non_fp32_parameters_raise_with_no_fallback():
    m = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    with pytest.raises(_ffi.CfmLibraryError, match="no CPU fallback"):
        cfm_b200.flow_matching_loss(m, *_inputs())
    with pytest.raises(_ffi.CfmLibraryError), torch.no_grad():
        cfm_b200.flow_matching_loss(m, *_inputs())
    with pytest.raises(_ffi.CfmLibraryError):
        cfm_b200.flow_matching_loss(m.double(), *(v.double() for v in _inputs()))


def test_mlp_forward_under_autograd_is_still_plain_pytorch():
    m = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    x = torch.randn(5, 3)
    assert torch.equal(m(x), m.net(x)) and m(x).requires_grad


# ---- the oracle -----------------------------------------------------------------------------------------------------
def test_oracle_on_a_hand_computed_row():
    """All weights zero except the output layer's: vt = b3, loss = mean((s * b3 - ut)^2), d loss / d b3 =
    2 s (s b3 - ut) / out_dim, and every other gradient but W3's is zero (SELU(0) = 0, so W3's is too)."""
    m = cfm_b200.MLP(dim=2, w=32, time_varying=True)
    state = {k: torch.zeros_like(v) for k, v in m.state_dict().items()}
    state["net.6.bias"] = torch.tensor([0.5, -1.0])
    xt, t, ut = torch.tensor([[0.3, -0.7]]), torch.tensor([0.25]), torch.tensor([[1.5, 1.0]])
    loss, grads = ot.loss_and_grads(state, 2, 2, 32, xt, t, ut)
    assert loss.item() == pytest.approx((1.0 + 4.0) / 2)
    assert torch.allclose(grads[7], torch.tensor([-1.0, -2.0], dtype=torch.float64))
    assert all(not g.any() for g in grads[:7])
    s = torch.tensor([2.0])
    loss, grads = ot.loss_and_grads(state, 2, 2, 32, xt, t, ut, row_scale=s)
    assert loss.item() == pytest.approx((0.25 + 9.0) / 2)
    assert torch.allclose(grads[7], torch.tensor([2 * 2 * -0.5 / 2, 2 * 2 * -3.0 / 2], dtype=torch.float64))


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_oracle_gradients_pass_gradcheck(act):
    torch.manual_seed(0)
    m = ot.make_model(cfm_b200.MLP(dim=2, out_dim=3, w=32, time_varying=True).state_dict(), 2, 3, 32, act)
    xt, t, ut, s = torch.randn(5, 2), torch.rand(5), torch.randn(5, 3), torch.rand(5) + 0.5
    names = [k for k, _ in m.named_parameters()]

    def f(*ps):
        return ot.loss_of(lambda z: torch.func.functional_call(m, dict(zip(names, ps)), (z,)), xt, t, ut, s)

    assert torch.autograd.gradcheck(f, tuple(p.detach().clone().requires_grad_(True) for p in m.parameters()))
    _, grads = ot.loss_and_grads(m.state_dict(), 2, 3, 32, xt, t, ut, row_scale=s, act=act)
    ps = [p.detach().clone().requires_grad_(True) for p in m.parameters()]
    for g, r in zip(grads, torch.autograd.grad(f(*ps), ps)):
        assert torch.equal(g, r)
