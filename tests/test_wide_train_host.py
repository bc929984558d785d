"""cfm_b200.flow_matching_loss for wide MLPs (the tensor-core class, csrc/train_tc.cu) without a device: which shapes
the library takes, its workspace, its argument errors (returned before any CUDA call), the Python wrapper's routing
and refusals, and the two float64 oracles the GPU tests use (gradcheck; the absolute-scale bound)."""
import ctypes
import re

import pytest
import torch

import cfm_b200
import wide_train_oracle as wo
from cfm_b200 import _ffi
from oracle import train as ot

ERR_ARG = -1  # CFM_ERR_ARG


@pytest.mark.parametrize("dim", [24, 32, 36, 40, 784])
@pytest.mark.parametrize("w", [24, 32, 36, 256])
@pytest.mark.parametrize("out_dim", [2, 4, 784])
def test_supported_truth_table(lib_built, dim, w, out_dim):
    lib = _ffi.load_library(lib_built)
    want = dim >= 32 and dim % 8 == 0 and w >= 32 and w % 8 == 0 and out_dim % 4 == 0
    assert bool(lib.cfm_mlp_tc_supported(128, dim, w, out_dim)) == want  # the forward's rule at its batch floor
    for batch in (1, 127, 128, 1 << 20):  # any batch: rows are GEMM rows or K
        assert bool(lib.cfm_mlp_tc_train_supported(batch, dim, w, out_dim)) == want
        assert (lib.cfm_mlp_tc_train_workspace_bytes(batch, dim, w, out_dim) > 0) == want
    assert not lib.cfm_mlp_tc_train_supported(0, dim, w, out_dim)
    assert lib.cfm_mlp_tc_train_workspace_bytes(0, dim, w, out_dim) == 0


def test_the_two_training_classes_do_not_overlap(lib_built):
    lib = _ffi.load_library(lib_built)
    for dim in range(1, 41):
        for w in (32, 64):
            for out_dim in (1, 4, 8):
                assert not (lib.cfm_mlp_small_train_supported(256, dim, w, out_dim)
                            and lib.cfm_mlp_tc_train_supported(256, dim, w, out_dim))


def test_workspace_is_positive_and_non_decreasing_in_batch(lib_built):
    lib = _ffi.load_library(lib_built)
    for dim, w, out_dim in ((32, 32, 4), (40, 200, 12), (784, 256, 784), (1024, 128, 8)):
        sizes = [lib.cfm_mlp_tc_train_workspace_bytes(b, dim, w, out_dim)
                 for b in (1, 2, 63, 64, 65, 127, 128, 129, 1000, 8192, 8449, 65536, 1 << 20)]
        assert sizes[0] > 0 and sizes == sorted(sizes), sizes
        # at least the fp32 pre-activations of the three hidden layers
        assert sizes[-1] >= 3 * 4 * w * (1 << 20)


def _call(lib, p, *, dim=32, w=32, out_dim=4, batch=256, ws_bytes=None, with_grad=1, grads=True, act=0, ws=None):
    if ws_bytes is None:
        ws_bytes = max(lib.cfm_mlp_tc_train_workspace_bytes(batch, dim, w, out_dim), 1 << 20)
    return lib.cfm_mlp_tc_mse_grad_f32(p, p, p, p, p, p, p, p, dim, w, out_dim, act, p, p, p, None, batch, with_grad,
                                       p, p if grads else None, p if ws is None else ws, ws_bytes, None)


def test_bad_arguments_are_refused_before_any_launch(lib_built):
    """Every case is an argument error found on the host.  The pointers are dummies that are never dereferenced; a
    launch would show in cfm_launch_count."""
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(256)
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    before = lib.cfm_launch_count()
    for kw, text in (({"w": 24}, b"unsupported shape"), ({"w": 36}, b"unsupported shape"),
                     ({"dim": 8}, b"unsupported shape"), ({"dim": 36}, b"unsupported shape"),
                     ({"out_dim": 2}, b"unsupported shape"), ({"batch": 0}, b"unsupported shape"),
                     ({"ws_bytes": 16}, b"workspace too small"), ({"ws": p + 4}, b"16-byte aligned"),
                     ({"grads": False}, b"with_grad needs a grads buffer"), ({"act": 7}, b"unknown activation")):
        assert _call(lib, p, **kw) == ERR_ARG, kw
        assert text in lib.cfm_last_error(), (kw, lib.cfm_last_error())
    assert lib.cfm_mlp_tc_mse_grad_f32(None, p, p, p, p, p, p, p, 32, 32, 4, 0, p, p, p, None, 256, 1, p, p, p,
                                       1 << 30, None) == ERR_ARG
    assert b"null pointer" in lib.cfm_last_error()
    assert lib.cfm_launch_count() == before


# ---- the Python wrapper ---------------------------------------------------------------------------------------------
def _inputs(B=4, dim=32, out_dim=4):
    return torch.randn(B, dim), torch.rand(B), torch.randn(B, out_dim)


@pytest.mark.parametrize("dim", [9, 16, 24, 31, 36])
def test_dims_between_the_classes_are_refused_naming_both(dim):
    m = cfm_b200.MLP(dim=dim, w=64, time_varying=True)
    with pytest.raises(NotImplementedError, match=re.escape("w in {32, 64}, dim <= 8")) as e:
        cfm_b200.flow_matching_loss(m, *_inputs(dim=dim, out_dim=dim))
    assert "tensor-core" in str(e.value) and "dim >= 32" in str(e.value)


@pytest.mark.parametrize("kw", [{"dim": 32, "w": 36}, {"dim": 32, "out_dim": 6}, {"dim": 32, "w": 24}])
def test_wide_shapes_outside_the_tensor_core_rule_are_refused(kw):
    m = cfm_b200.MLP(time_varying=True, **kw)
    with pytest.raises(NotImplementedError, match="tensor-core"):
        cfm_b200.flow_matching_loss(m, *_inputs(dim=m.dim, out_dim=m.out_dim))


def test_wide_model_that_is_not_time_varying_is_refused():
    with pytest.raises(NotImplementedError):
        cfm_b200.flow_matching_loss(cfm_b200.MLP(dim=32, w=64), *_inputs())


def test_tensor_core_class_with_cpu_tensors_raises_library_error_not_not_implemented():
    m = cfm_b200.MLP(dim=784, w=256, time_varying=True)
    with pytest.raises(_ffi.CfmLibraryError, match="no CPU fallback"):
        cfm_b200.flow_matching_loss(m, *_inputs(dim=784, out_dim=784))
    with pytest.raises(_ffi.CfmLibraryError), torch.no_grad():
        cfm_b200.flow_matching_loss(m, *_inputs(dim=784, out_dim=784))


def test_shape_errors_of_the_tensor_core_class_are_value_errors():
    m = cfm_b200.MLP(dim=32, w=64, time_varying=True)
    xt, t, ut = _inputs()
    for args in ((xt[:, :8], t, ut), (xt, t[:3], ut), (xt, t, ut[:, :2]), (xt[:0], t[:0], ut[:0])):
        with pytest.raises(ValueError):
            cfm_b200.flow_matching_loss(m, *args)


# ---- the oracles --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_oracle_gradients_pass_gradcheck_at_a_wide_shape(act):
    torch.manual_seed(0)
    dim, out_dim, w = 32, 4, 32
    m = ot.make_model(cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True).state_dict(), dim, out_dim, w,
                      act)
    xt, t, ut, s = torch.randn(3, dim), torch.rand(3), torch.randn(3, out_dim), torch.rand(3) + 0.5
    names = [k for k, _ in m.named_parameters()]

    def f(*ps):
        return ot.loss_of(lambda z: torch.func.functional_call(m, dict(zip(names, ps)), (z,)), xt, t, ut, s)

    assert torch.autograd.gradcheck(f, tuple(p.detach().clone().requires_grad_(True) for p in m.parameters()))
    _, grads = ot.loss_and_grads(m.state_dict(), dim, out_dim, w, xt, t, ut, row_scale=s, act=act)
    ps = [p.detach().clone().requires_grad_(True) for p in m.parameters()]
    for g, r in zip(grads, torch.autograd.grad(f(*ps), ps)):
        assert torch.equal(g, r)


@pytest.mark.parametrize("act", ["selu", "silu"])
def test_absolute_scales_bound_a_cpu_fp32_autograd_run(act):
    """fp32 autograd on the CPU errs by far less than 1e-5 of each entry's absolute scale (the GPU gate), and the
    scale is what it claims: at least |gradient|, and equal to it when every term is non-negative."""
    torch.manual_seed(1)
    dim, out_dim, w, B = 64, 12, 96, 300
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    if act == "silu":
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    xt, t, ut, s = torch.randn(B, dim), torch.rand(B), torch.randn(B, out_dim), torch.rand(B) * 2
    rl, rg = ot.loss_and_grads(m.state_dict(), dim, out_dim, w, xt, t, ut, row_scale=s, act=act)
    scales = wo.grad_scales(m.state_dict(), dim, out_dim, w, xt, t, ut, row_scale=s, act=act)
    loss = torch.mean((s[:, None] * m(torch.cat([xt, t[:, None]], 1)) - ut) ** 2)
    g32 = torch.autograd.grad(loss, list(m.parameters()))
    worst = 0.0
    for g, r, sc in zip(g32, rg, scales):
        assert sc.shape == r.shape and (r.abs() <= sc * (1 + 1e-12)).all()
        worst = max(worst, ((g.double() - r).abs() / sc).max().item())
    assert 0 < worst < 1e-6, worst
    # a one-layer check of the recursion: with |.| everywhere the scale is the gradient itself
    pos = {k: v.abs() for k, v in m.state_dict().items()}
    xp, up = xt.abs(), -ut.abs()
    _, rgp = ot.loss_and_grads(pos, dim, out_dim, w, xp, t, up, act=act)
    scp = wo.grad_scales(pos, dim, out_dim, w, xp, t, up, act=act)
    if act == "selu":  # positive inputs and weights: every pre-activation is positive, act' is the constant lambda
        for r, sc in zip(rgp, scp):
            assert torch.allclose(r, sc, rtol=1e-10, atol=0)
