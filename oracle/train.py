"""TEST INFRASTRUCTURE ONLY -- the training lines of the 2-D tutorials in float64 on the CPU, with torch autograd.

    vt = model(torch.cat([xt, t[:, None]], dim=-1))
    loss = torch.mean((vt - ut) ** 2)
    loss.backward()

(examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb raw lines 166-186; the SF2M score loss
``torch.mean((lambda_t[:, None] * st + eps) ** 2)`` of SF2M_tutorial.ipynb is the same expression with a per-row
scale and ``ut = -eps``).  Pure torch: the parity gate of cfm_b200.flow_matching_loss.
"""
import torch

from . import vector_field as vf

_ACTS = {"selu": torch.nn.SELU, "silu": torch.nn.SiLU}


def make_model(state, dim, out_dim, w, act="selu"):
    """The reference MLP(dim, out_dim, w, time_varying=True) in float64 holding ``state`` (a state_dict of any float
    dtype and device), with SELU or SiLU between the layers."""
    m = vf.make_mlp(dim, out_dim=out_dim, w=w, time_varying=True, dtype=torch.float64)
    m.load_state_dict({k: v.detach().cpu().double() for k, v in state.items()})
    for k in (1, 3, 5):
        m.net[k] = _ACTS[act]()
    return m


def loss_of(model, xt, t, ut, row_scale=None):
    """The notebook's loss for a float64 model; inputs are cast to float64 on the CPU."""
    xt, t, ut = (v.detach().cpu().double() for v in (xt, t, ut))
    vt = model(torch.cat([xt, t[:, None]], dim=-1))
    if row_scale is not None:
        vt = row_scale.detach().cpu().double()[:, None] * vt
    return torch.mean((vt - ut) ** 2)


def loss_and_grads(state, dim, out_dim, w, xt, t, ut, row_scale=None, act="selu"):
    """(loss, [d loss / d p for p in parameters()]) in float64: net.0.weight, net.0.bias, ..., net.6.bias."""
    m = make_model(state, dim, out_dim, w, act)
    loss = loss_of(m, xt, t, ut, row_scale)
    grads = torch.autograd.grad(loss, list(m.parameters()))
    return loss.detach(), [g.detach() for g in grads]
