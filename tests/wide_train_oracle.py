"""Absolute scales of the flow-matching loss gradients of an MLP(dim, out_dim, w, time_varying=True), in float64 on the
CPU: the backward pass of oracle/train.py with every term replaced by its magnitude, on the magnitudes of the forward
terms,

    P_l = |W_l| A_{l-1} + |b_l|,   A_l = max(|a_l|, |act'(pre_l)| P_l),   A_{-1} = |[x, t]|
    |delta_3| = L |s| (|s| P_3 + |target|),   L = 2 / (B out_dim)
    |delta_{l-1}| = |act'(pre_{l-1})| * (|delta_l| |W_l|)
    scale(dW_l) = |delta_l|^T A_{l-1},   scale(b_l) = sum_r |delta_l|

so every gradient entry gets the size of the sums it is made of, not of the largest entry of its tensor: a computed
activation errs by a multiple of act' times the size of its pre-activation's terms, which cancellation can make far
larger than the activation itself.  Any fp32-grade evaluation of the gradient (fp32 autograd on the CPU, the fp16x3
tensor-core kernels) errs by a small multiple of that scale; tests/test_wide_train_host.py checks the bound on a CPU
fp32 autograd run."""
import torch

from oracle import train as ot


def _act_deriv(p, act):
    if act == "selu":
        lam, alpha = 1.0507009873554804934193349852946, 1.6732632423543772848170429916717
        return torch.where(p > 0, torch.full_like(p, lam), lam * alpha * torch.exp(p))
    s = torch.sigmoid(p)
    return s + p * s * (1 - s)


def grad_scales(state, dim, out_dim, w, xt, t, ut, row_scale=None, act="selu"):
    """[scale of d loss / d p for p in parameters()] in float64, shapes as the parameters."""
    m = ot.make_model(state, dim, out_dim, w, act)
    Ws = [m.net[k].weight.detach() for k in (0, 2, 4, 6)]
    bs = [m.net[k].bias.detach() for k in (0, 2, 4, 6)]
    h = torch.cat([xt, t[:, None]], 1).detach().cpu().double()
    mag = h.abs()
    ins, pres = [mag], []
    for k in range(3):
        p = h @ Ws[k].T + bs[k]
        pres.append(p)
        h = m.net[2 * k + 1](p)
        mag = torch.maximum(h.abs(), _act_deriv(p, act).abs() * (mag @ Ws[k].abs().T + bs[k].abs()))
        ins.append(mag)
    P3 = mag @ Ws[3].abs().T + bs[3].abs()
    B = h.shape[0]
    s = torch.ones(B, dtype=torch.float64) if row_scale is None else row_scale.detach().cpu().double()
    L = 2.0 / (B * out_dim)
    d = L * s.abs()[:, None] * (s.abs()[:, None] * P3 + ut.detach().cpu().double().abs())
    out = [None] * 8
    for k in (3, 2, 1, 0):
        out[2 * k] = d.T @ ins[k]
        out[2 * k + 1] = d.sum(0)
        if k:
            d = _act_deriv(pres[k - 1], act).abs() * (d @ Ws[k].abs())
    return out
