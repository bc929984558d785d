"""TEST INFRASTRUCTURE ONLY -- float64 references for gradients through the exact-likelihood Euler trajectory
(cfm_b200.NeuralODE(cnf_wrapper(mlp, "exact"), solver="euler"), csrc/cnf_train.cu).

* ``euler_loop``: torchdyn's fixed-step Euler over ``t_span`` with autograd enabled (oracle/vector_field.py's
  ``euler_trajectory`` is ``no_grad``); in values it is bit-equal to ``cnf_oracle.euler_any_direction``.
* ``restated_backward``: the discrete adjoint the kernel computes, restated in float64 from the stored states:
  a_N = G_N and, for n = N-1 .. 0, with phi_n = a_{x,n+1} . f(t_n, x_n) + a_{l,n+1} tr(df/dx)(t_n, x_n),
  a_{x,n} = G_{x,n} + a_{x,n+1} + h_n grad_x phi_n, a_{l,n} = G_{l,n} + a_{l,n+1}, theta_bar += h_n grad_theta phi_n.
  grad phi is the reverse pass of the primal chain and of the dim forward-mode tangent chains of the trace.
"""
import torch

_SELU_L, _SELU_A = 1.0507009873554804934193349852946, 1.6732632423543772848170429916717


def euler_loop(f, z, t_span):
    """(n_span, B, dim + 1): x_{n+1} = x_n + (t_{n+1} - t_n) f(t_n, x_n), on the autograd graph."""
    t_span = t_span.to(z)
    sol = [z]
    for a, b in zip(t_span[:-1], t_span[1:]):
        z = z + (b - a) * f(a, z)
        sol.append(z)
    return torch.stack(sol)


def _act(x, act):
    """(act(x), act'(x), act''(x))"""
    if act == "selu":
        e = torch.exp(torch.clamp(x, max=0.0))
        neg = x <= 0
        return (torch.where(neg, _SELU_L * _SELU_A * (e - 1), _SELU_L * x),
                torch.where(neg, _SELU_L * _SELU_A * e, torch.full_like(x, _SELU_L)),
                torch.where(neg, _SELU_L * _SELU_A * e, torch.zeros_like(x)))
    s = torch.sigmoid(x)
    return x * s, s + x * s * (1 - s), s * (1 - s) * (2 + x * (1 - 2 * s))


def _params(state):
    Ws = [state[f"net.{k}.weight"].detach().double() for k in (0, 2, 4, 6)]
    bs = [state[f"net.{k}.bias"].detach().double() for k in (0, 2, 4, 6)]
    return Ws, bs


def phi_grads(Ws, bs, x, t, a, c, act):
    """grad_x and grad_theta of sum_rows [a . f(t, x) + c tr(df/dx)], theta in parameters() order, for rows x
    (B, dim), the scalar time t, a (B, dim) and c (B,)."""
    W0, W1, W2, W3 = Ws
    b0, b1, b2, _ = bs
    B, dim = x.shape
    z = torch.cat([x, torch.full((B, 1), float(t), dtype=x.dtype, device=x.device)], 1)
    s0, d0, dd0 = _act(z @ W0.T + b0, act)
    P0 = W0[:, :dim].T                       # (dim, w): p_{0,k} = W0[:, k]
    T0 = d0[:, None, :] * P0[None]           # (B, dim, w)
    s1, d1, dd1 = _act(s0 @ W1.T + b1, act)
    P1 = T0 @ W1.T
    T1 = d1[:, None, :] * P1
    s2, d2, dd2 = _act(s1 @ W2.T + b2, act)
    P2 = T1 @ W2.T
    T2 = d2[:, None, :] * P2
    tau2 = c[:, None, None] * W3[None]       # adjoint of T_{2,k}
    e2 = tau2 * d2[:, None, :]               # adjoint of p_{2,k}
    delta2 = d2 * (a @ W3) + dd2 * (tau2 * P2).sum(1)
    tau1 = e2 @ W2
    e1 = tau1 * d1[:, None, :]
    delta1 = d1 * (delta2 @ W2) + dd1 * (tau1 * P1).sum(1)
    tau0 = e1 @ W1
    e0 = tau0 * d0[:, None, :]
    delta0 = d0 * (delta1 @ W1) + dd0 * (tau0 * P0[None]).sum(1)
    gx = delta0 @ W0[:, :dim]
    gW0 = delta0.T @ z
    gW0[:, :dim] += e0.sum(0).T
    g = [gW0, delta0.sum(0),
         delta1.T @ s0 + torch.einsum("bkw,bkv->wv", e1, T0), delta1.sum(0),
         delta2.T @ s1 + torch.einsum("bkw,bkv->wv", e2, T1), delta2.sum(0),
         a.T @ s2 + torch.einsum("b,bkw->kw", c, T2), a.sum(0)]
    return gx, g


def kink_rows(state, traj, t_span, rel=1e-5):
    """(B,) bool: rows whose path passes within ``rel`` (relative to the sum of the magnitudes that form it) of
    SELU's kink at a hidden pre-activation at some Euler step.  There act' and act'' jump, so an fp32 path and a
    float64 one may take different branches; rows are independent, so a zero cotangent takes such a row out of
    both sides exactly."""
    Ws, bs = _params(state)
    Ws, bs = [W.to(traj.device) for W in Ws], [b.to(traj.device) for b in bs]
    dim = traj.shape[2] - 1
    near = torch.zeros(traj.shape[1], dtype=torch.bool, device=traj.device)
    for n in range(traj.shape[0] - 1):
        x = traj[n][:, :dim].double()
        h = torch.cat([x, torch.full_like(x[:, :1], float(t_span[n]))], 1)
        for W, b in zip(Ws[:3], bs[:3]):
            pre = h @ W.T + b
            mag = h.abs() @ W.abs().T + b.abs()
            near |= (pre.abs() <= rel * mag).any(1)
            h = torch.nn.functional.selu(pre)
    return near


def restated_backward(state, traj, t_span, G, act="selu", h32=False):
    """(parameter gradients in parameters() order, input gradient) of L with dL/dtraj = G, by the discrete adjoint
    over the states ``traj`` (n_span, B, dim + 1).  ``h32``: form h_n = t_{n+1} - t_n in fp32, as the kernel does."""
    Ws, bs = _params(state)
    Ws, bs = [W.to(traj.device) for W in Ws], [b.to(traj.device) for b in bs]
    traj, G = traj.double(), G.double()
    dim = traj.shape[2] - 1
    if h32:
        ts = t_span.float()
        hs = [float(ts[n + 1] - ts[n]) for n in range(len(ts) - 1)]
        ts = ts.double()
    else:
        ts = t_span.double()
        hs = [float(ts[n + 1] - ts[n]) for n in range(len(ts) - 1)]
    grads = [torch.zeros_like(p) for pair in zip(Ws, bs) for p in pair]
    adj = G[-1].clone()
    for n in range(traj.shape[0] - 2, -1, -1):
        h = hs[n]
        gx, g = phi_grads(Ws, bs, traj[n][:, :dim], ts[n], h * adj[:, :dim], h * adj[:, dim], act)
        for acc, v in zip(grads, g):
            acc += v
        adj = G[n] + adj + torch.cat([gx, torch.zeros_like(gx[:, :1])], 1)
    return grads, adj
