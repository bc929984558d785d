"""TEST INFRASTRUCTURE ONLY -- the action-matching training lines of the 2-D tutorial in float64 on the CPU, with torch
autograd and its double backward (examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb, cell 11):

    st = torch.sum(action(torch.cat([xt, t], dim=-1)))
    dsdx, dsdt = torch.autograd.grad(st, (xt, t), create_graph=True, retain_graph=True)
    a0 = action(torch.cat([x0, torch.zeros(batch_size, 1)], dim=-1))
    a1 = action(torch.cat([x1, torch.ones(batch_size, 1)], dim=-1))
    loss = (a0 - a1 + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt).mean()

The parity gate of cfm_b200.action_matching_loss."""
import torch

from oracle import train as otr


def make_action(state, dim, w, act="selu"):
    """The reference MLP(dim, out_dim=1, w, time_varying=True) in float64 holding ``state``."""
    return otr.make_model(state, dim, 1, w, act)


def terms(action, xt, t, x0, x1):
    """Per row (s(x0, 0), s(x1, 1), d s / d x (xt, t), d s / d t (xt, t)), the last two attached to the graph of the
    action's parameters; inputs are cast to float64 on the CPU and ``t`` may be (B,) or (B, 1)."""
    xt, t, x0, x1 = (v.detach().cpu().double() for v in (xt, t, x0, x1))
    B = xt.shape[0]
    xt, t = xt.clone().requires_grad_(True), t.reshape(B, 1).clone().requires_grad_(True)
    st = torch.sum(action(torch.cat([xt, t], dim=-1)))
    dsdx, dsdt = torch.autograd.grad(st, (xt, t), create_graph=True, retain_graph=True)
    a0 = action(torch.cat([x0, torch.zeros(B, 1, dtype=torch.float64)], dim=-1))
    a1 = action(torch.cat([x1, torch.ones(B, 1, dtype=torch.float64)], dim=-1))
    return a0, a1, dsdx, dsdt


def loss_of(action, xt, t, x0, x1):
    a0, a1, dsdx, dsdt = terms(action, xt, t, x0, x1)
    return (a0 - a1 + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt).mean()


def loss_scale(action, xt, t, x0, x1):
    """mean(|s0| + |s1| + 1/2 |d s / d x|^2 + |d s / d t|): the loss is a difference of terms of this size, so its fp32
    rounding error is relative to this, not to the loss."""
    with torch.enable_grad():
        a0, a1, dsdx, dsdt = terms(action, xt, t, x0, x1)
    return (a0.abs() + a1.abs() + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt.abs()).mean().item()


def action_matching_loss_and_grads(state, dim, w, xt, t, x0, x1, act="selu"):
    """(loss, [d loss / d p for p in parameters()]) in float64: net.0.weight, net.0.bias, ..., net.6.bias."""
    m = make_action(state, dim, w, act)
    loss = loss_of(m, xt, t, x0, x1)
    grads = torch.autograd.grad(loss, list(m.parameters()))
    return loss.detach(), [g.detach() for g in grads]
