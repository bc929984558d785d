"""The training step of the 2-D tutorials on the device: drop-in for the three lines every training cell repeats,

    vt = model(torch.cat([xt, t[:, None]], dim=-1))
    loss = torch.mean((vt - ut) ** 2)
    loss.backward()

(examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb raw lines 166-186, 310-330, 458-479, 602-623;
Flow_matching_tutorial.ipynb and SF2M_tutorial.ipynb likewise), as

    loss = cfm_b200.flow_matching_loss(model, xt, t, ut)
    loss.backward()

One library call computes the loss and the gradients of all eight parameters; ``loss`` is attached to the autograd
graph of the parameters, so ``backward()``, gradient accumulation, clipping, any ``torch.optim`` optimizer and DDP
hooks work as with the eager lines.  The SF2M score loss ``torch.mean((lambda_t[:, None] * score_model(...) + eps) **
2)`` is ``flow_matching_loss(score_model, xt, t, -eps, row_scale=lambda_t)``.

Two classes of ``cfm_b200.MLP(time_varying=True)`` (SELU or SiLU, fp32 on a CUDA device) are accelerated:

* small: ``w`` in {32, 64}, ``dim <= 8``, ``out_dim <= 8`` -- ONE kernel (csrc/train_small.cu);
* tensor-core: the shapes the tensor-core forward samples, ``dim >= 32`` and ``w >= 32`` multiples of 8, ``out_dim`` a
  multiple of 4, e.g. the MNIST model ``MLP(784, w=256, time_varying=True)`` -- fp16x3 wgmma GEMMs with split-K weight
  gradients, a fixed 19 launches (csrc/train_tc.cu).

Anything else raises -- there is no eager fallback (``MLP.forward`` under autograd is still plain PyTorch for whoever
wants it).  Gradients flow to the parameters only.

``action_matching_loss(action, xt, t, x0, x1)`` does the same for the action-matching cell of the same notebook, whose
loss needs a double backward: one kernel (csrc/action_train.cu) computes the loss, the input gradient of the action it
contains, and all eight parameter gradients of ``MLP(dim, out_dim=1, time_varying=True)``.
"""
import torch
from torch.autograd.function import once_differentiable

from . import _ffi
from .models import MLP


def _launch(model, params, xt, t, ut, row_scale, with_grad, kind="small"):
    """One library call of the class ``kind`` ("small" or "tc"): (loss 0-d, flat gradient buffer in parameters() order
    or None)."""
    L = _ffi.lib()
    name = f"cfm_mlp_{kind}_mse_grad_f32"
    dev = xt.device
    B = xt.shape[0]
    loss = torch.empty((), dtype=torch.float32, device=dev)
    grads = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev) if with_grad else None
    ws = _ffi.workspace(getattr(L, f"cfm_mlp_{kind}_train_workspace_bytes")(B, model.dim, model.w, model.out_dim), dev)
    with torch.cuda.device(dev):  # kernels launch on the current device: make it the tensors' one
        _ffi.check(getattr(L, name)(
            *[_ffi.ptr(p) for p in params], model.dim, model.w, model.out_dim, model.act, _ffi.ptr(xt), _ffi.ptr(t),
            _ffi.ptr(ut), _ffi.ptr(row_scale), B, 1 if with_grad else 0, _ffi.ptr(loss), _ffi.ptr(grads),
            _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(dev)), name)
    return loss, grads


class _FusedLossGrad(torch.autograd.Function):
    """loss(parameters) of one library call ``launch(params, with_grad) -> (loss, flat gradients)``: forward computes the
    loss and, in the same launch, its gradients for upstream gradient 1; backward scales that flat buffer by
    ``grad_output`` and hands out views of it."""

    @staticmethod
    def forward(ctx, launch, *params):
        loss, grads = launch([p.detach().contiguous() for p in params], True)
        ctx.grads = grads
        ctx.shapes = [p.shape for p in params]
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        flat = ctx.grads * grad_output
        out, o = [], 0
        for shape in ctx.shapes:
            n = shape.numel()
            out.append(flat[o:o + n].view(shape))
            o += n
        return (None, *out)


def _attach(launch, params):
    """The loss of ``launch`` on the parameters' autograd graph when autograd wants their gradients; else the loss only
    (the kernel skips the gradients)."""
    if torch.is_grad_enabled() and any(p.requires_grad for p in params):
        return _FusedLossGrad.apply(launch, *params)
    loss, _ = launch([p.detach().contiguous() for p in params], False)
    return loss


def _check_model(model, fn="flow_matching_loss", action=False):
    out = "out_dim = 1" if action else "out_dim <= 8"
    if not isinstance(model, MLP):
        raise NotImplementedError(
            f"{fn}: no training kernel for {type(model).__name__}; it takes "
            f"cfm_b200.MLP(time_varying=True) with w in {{32, 64}}, dim <= 8, {out}")
    if not (model.time_varying and model.w in (32, 64) and 1 <= model.dim <= 8
            and (model.out_dim == 1 if action else 1 <= model.out_dim <= 8)
            and model.act in (_ffi.ACT_SELU, _ffi.ACT_SILU)):
        raise NotImplementedError(
            f"{fn}: no training kernel for MLP(dim={model.dim}, out_dim={model.out_dim}, w={model.w}, "
            f"time_varying={model.time_varying}, act={model.act}); the kernel's class is w in {{32, 64}}, dim <= 8, "
            f"{out}, time_varying=True, SELU or SiLU")


def _flow_matching_class(model):
    """"small" or "tc": which kernel trains ``model``; raises NotImplementedError naming both classes otherwise."""
    if (isinstance(model, MLP) and model.time_varying and model.act in (_ffi.ACT_SELU, _ffi.ACT_SILU)):
        if model.w in (32, 64) and 1 <= model.dim <= 8 and 1 <= model.out_dim <= 8:
            return "small"
        if _ffi.lib().cfm_mlp_tc_train_supported(1, model.dim, model.w, model.out_dim):
            return "tc"
    what = (f"MLP(dim={model.dim}, out_dim={model.out_dim}, w={model.w}, time_varying={model.time_varying}, "
            f"act={model.act})" if isinstance(model, MLP) else type(model).__name__)
    raise NotImplementedError(
        f"flow_matching_loss: no training kernel for {what}; it takes cfm_b200.MLP(time_varying=True), SELU or SiLU, "
        "in one of two classes: small (w in {32, 64}, dim <= 8, out_dim <= 8) or tensor-core (dim >= 32 and w >= 32, "
        "both multiples of 8, out_dim a multiple of 4)")


def _check_tensors(fn, tensors):
    for name, v in tensors:
        if not torch.is_tensor(v):
            raise ValueError(f"{fn}: {name} must be a tensor; got {type(v).__name__}")
        if v.requires_grad:
            raise ValueError(f"{fn}: {name} requires grad, but gradients flow to the model's parameters "
                             "only; detach it")


def _check_devices(fn, model, tensors):
    """The model's eight parameters, after checking that they and ``tensors`` are fp32 on one CUDA device."""
    params = [p for lin in model._linears() for p in (lin.weight, lin.bias)]
    dev = params[0].device
    if dev.type != "cuda" or any(p.device != dev or p.dtype != torch.float32 for p in params):
        raise _ffi.CfmLibraryError(f"{fn}: the MLP's parameters must be fp32 on one CUDA device (there "
                                   "is no CPU fallback; the eager lines run anywhere)")
    for name, v in tensors:
        if v.device != dev or v.dtype != torch.float32:
            raise _ffi.CfmLibraryError(f"{fn}: {name} must be fp32 on the parameters' device {dev}; got "
                                       f"{v.dtype} on {v.device}")
    return params


def flow_matching_loss(model, xt, t, ut, row_scale=None):
    """``torch.mean((s[:, None] * model(torch.cat([xt, t[:, None]], -1)) - ut) ** 2)`` with ``s = row_scale`` (or 1),
    as a 0-d fp32 CUDA tensor.

    ``model`` is a ``cfm_b200.MLP(time_varying=True)`` with SELU or SiLU of the small class (``w`` in {32, 64},
    ``dim <= 8``, ``out_dim <= 8``: one kernel) or the tensor-core class (``dim >= 32`` and ``w >= 32`` multiples of 8,
    ``out_dim`` a multiple of 4: fp16x3 tensor-core GEMMs, 19 launches); anything else raises NotImplementedError.
    ``xt`` (B, dim), ``t`` (B,), ``ut`` (B, out_dim), ``row_scale`` (B,): fp32 on the parameters' CUDA device.  With
    autograd enabled the result carries the gradients of the model's eight parameters (computed in the same call as
    the loss); under ``torch.no_grad()`` the library computes the loss only, with the same bits."""
    kind = _flow_matching_class(model)
    tensors = [("xt", xt), ("t", t), ("ut", ut)] + ([("row_scale", row_scale)] if row_scale is not None else [])
    _check_tensors("flow_matching_loss", tensors)
    if xt.dim() != 2 or xt.shape[1] != model.dim or xt.shape[0] < 1:
        raise ValueError(f"flow_matching_loss: xt must be (B >= 1, {model.dim}); got {tuple(xt.shape)}")
    B = xt.shape[0]
    if tuple(t.shape) != (B,):
        raise ValueError(f"flow_matching_loss: t must be ({B},), one time per row; got {tuple(t.shape)}")
    if tuple(ut.shape) != (B, model.out_dim):
        raise ValueError(f"flow_matching_loss: ut must be ({B}, {model.out_dim}); got {tuple(ut.shape)}")
    if row_scale is not None and tuple(row_scale.shape) != (B,):
        raise ValueError(f"flow_matching_loss: row_scale must be ({B},); got {tuple(row_scale.shape)}")
    params = _check_devices("flow_matching_loss", model, tensors)
    xt, t, ut = xt.contiguous(), t.contiguous(), ut.contiguous()
    if row_scale is not None:
        row_scale = row_scale.contiguous()
    return _attach(lambda ps, with_grad: _launch(model, ps, xt, t, ut, row_scale, with_grad, kind), params)


def _launch_action(model, params, xt, t, x0, x1, with_grad):
    """One library call: (loss 0-d, flat gradient buffer in parameters() order or None)."""
    L = _ffi.lib()
    dev = xt.device
    B = xt.shape[0]
    loss = torch.empty((), dtype=torch.float32, device=dev)
    grads = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev) if with_grad else None
    ws = _ffi.workspace(L.cfm_mlp_small_train_workspace_bytes(B, model.dim, model.w, 1), dev)
    with torch.cuda.device(dev):  # kernels launch on the current device: make it the tensors' one
        _ffi.check(L.cfm_mlp_small_action_grad_f32(
            *[_ffi.ptr(p) for p in params], model.dim, model.w, model.act, _ffi.ptr(xt), _ffi.ptr(t), _ffi.ptr(x0),
            _ffi.ptr(x1), B, 1 if with_grad else 0, _ffi.ptr(loss), _ffi.ptr(grads), _ffi.ptr(ws), ws.numel(),
            _ffi.stream_ptr(dev)), "cfm_mlp_small_action_grad_f32")
    return loss, grads


def action_matching_loss(action, xt, t, x0, x1):
    """The action-matching loss of tutorial_training_8_gaussians_to_moons.ipynb (cell 11) as a 0-d fp32 CUDA tensor:

        mean_r [ s(x0_r, 0) - s(x1_r, 1) + 1/2 |d s / d x (xt_r, t_r)|^2 + d s / d t (xt_r, t_r) ]

    for the scalar action ``s = action``, a ``cfm_b200.MLP(dim, out_dim=1, w, time_varying=True)`` with ``w`` in
    {32, 64}, ``dim <= 8``, SELU or SiLU.  It replaces the notebook's double backward:

        st = torch.sum(action(torch.cat([xt, t], dim=-1)))
        dsdx, dsdt = torch.autograd.grad(st, (xt, t), create_graph=True, retain_graph=True)
        a0 = action(torch.cat([x0, torch.zeros(batch_size, 1)], dim=-1))
        a1 = action(torch.cat([x1, torch.ones(batch_size, 1)], dim=-1))
        loss = (a0 - a1 + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt).mean()

    ``xt``, ``x0``, ``x1`` (B, dim) and ``t`` (B,) or (B, 1): fp32 on the parameters' CUDA device, not requiring grad.
    With autograd enabled the result carries the gradients of the action's eight parameters, computed in the same
    launch as the loss (``b3``'s is exactly 0); under ``torch.no_grad()`` the kernel computes the loss only, with the
    same bits."""
    fn = "action_matching_loss"
    _check_model(action, fn, action=True)
    tensors = [("xt", xt), ("t", t), ("x0", x0), ("x1", x1)]
    _check_tensors(fn, tensors)
    if xt.dim() != 2 or xt.shape[1] != action.dim or xt.shape[0] < 1:
        raise ValueError(f"{fn}: xt must be (B >= 1, {action.dim}); got {tuple(xt.shape)}")
    B = xt.shape[0]
    if tuple(t.shape) not in ((B,), (B, 1)):
        raise ValueError(f"{fn}: t must be ({B},) or ({B}, 1), one time per row; got {tuple(t.shape)}")
    for name, v in (("x0", x0), ("x1", x1)):
        if tuple(v.shape) != (B, action.dim):
            raise ValueError(f"{fn}: {name} must be ({B}, {action.dim}); got {tuple(v.shape)}")
    params = _check_devices(fn, action, tensors)
    xt, t, x0, x1 = xt.contiguous(), t.reshape(B).contiguous(), x0.contiguous(), x1.contiguous()
    return _attach(lambda ps, with_grad: _launch_action(action, ps, xt, t, x0, x1, with_grad), params)
