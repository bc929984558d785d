"""TEST INFRASTRUCTURE ONLY -- absolute scales of the action-matching loss gradients (csrc/action_train.cu) and of the
gradients through the exact-likelihood Euler trajectory (csrc/cnf_train.cu), in float64, rows vectorised.

Each is the kernel's own recursion with every term replaced by its magnitude, on the magnitudes of the forward terms,
as tests/wide_train_oracle.py does for the flow-matching loss:

    P_l = |W_l| A_{l-1} + |b_l|,   A_l = max(|a_l|, |act'(pre_l)| P_l),   A_{-1} = |input|

and the same bound along every forward-mode tangent chain (Pd_l = |W_l| Hd_{l-1}, Hd_l = |act'(pre_l)| Pd_l).  A
gradient entry's scale is the sum over rows of |delta| (x) A of every (delta, a) pair that enters it, so it is the size
of the sums the entry is made of, not of the largest entry of its tensor.  An fp32-grade evaluation errs by a small
multiple of it; tests/test_train_scale_host.py checks the bound against fp32 runs on the CPU.

``action_grad_scales``: the four (delta, a) pairs per layer and row of tests/test_action_train_host.py's ``_restated``
(end 0 and end 1 with cotangent +-1/B, the middle point's primal pair Q with its act'' terms, and the tangent pair
g / B against the tangent activations along c = [g_x, 1]).

``cnf_grad_scales``: tests/cnf_train_oracle.py's ``phi_grads`` in magnitudes, and the adjoint carried step by step as
|a_n| <= |G_n| + |a_{n+1}| + |h_n| |grad_x phi_n|."""
import torch

from cnf_train_oracle import _act


# ---- action matching -------------------------------------------------------------------------------------------------
def action_grad_scales(state, xt, t, x0, x1, act="selu"):
    """[scale of d loss / d p for p in parameters()] in float64, shapes as the parameters; b3's is 0 (its gradient is
    exactly 0).  ``t`` may be (B,) or (B, 1)."""
    Ws = [state[f"net.{k}.weight"].detach().cpu().double() for k in (0, 2, 4, 6)]
    bs = [state[f"net.{k}.bias"].detach().cpu().double() for k in (0, 2, 4)]
    aW = [W.abs() for W in Ws]
    ab = [b.abs() for b in bs]
    xt, x0, x1 = (v.detach().cpu().double() for v in (xt, x0, x1))
    B, dim = xt.shape
    t = t.detach().cpu().double().reshape(B, 1)
    w3 = aW[3][0]
    gW = [torch.zeros_like(W) for W in Ws]
    gb = [torch.zeros_like(b) for b in bs] + [torch.zeros(1, dtype=torch.float64)]

    def forward(z):
        """activations' bounds A_{-1..2}, |act'|, |act''| per hidden layer"""
        h, A, D1, D2 = z, [z.abs()], [], []
        for W, b, Wa, ba in zip(Ws[:3], bs, aW[:3], ab):
            p = h @ W.T + b
            h, d1, d2 = _act(p, act)
            D1.append(d1.abs()), D2.append(d2.abs())
            A.append(torch.maximum(h.abs(), d1.abs() * (A[-1] @ Wa.T + ba)))
        return A, D1, D2

    def accumulate(deltas, A, bias):
        for l in range(3):
            gW[l] += deltas[l].T @ A[l]
            if bias:
                gb[l] += deltas[l].sum(0)

    for z in (torch.cat([x0, torch.zeros(B, 1, dtype=torch.float64)], 1),
              torch.cat([x1, torch.ones(B, 1, dtype=torch.float64)], 1)):
        A, D1, _ = forward(z)
        d = [None, None, D1[2] * w3 / B]
        d[1] = D1[1] * (d[2] @ aW[2])
        d[0] = D1[0] * (d[1] @ aW[1])
        accumulate(d, A, True)
        gW[3][0] += A[3].sum(0) / B
    # the middle point: g = grad s by the reverse pass, then the tangent forward along c = [g_x, 1] and its reverse
    A, D1, D2 = forward(torch.cat([xt, t], 1))
    g = [None, None, D1[2] * w3]
    M = [None, g[2] @ aW[2], None]
    g[1] = D1[1] * M[1]
    M[0] = g[1] @ aW[1]
    g[0] = D1[0] * M[0]
    gz = g[0] @ aW[0]
    Hd = [torch.cat([gz[:, :dim], torch.ones(B, 1, dtype=torch.float64)], 1)]
    Pd = []
    for l in range(3):
        Pd.append(Hd[-1] @ aW[l].T)
        Hd.append(D1[l] * Pd[-1])
    Q = [None, None, D2[2] * Pd[2] * w3 / B]
    Q[1] = D1[1] * (Q[2] @ aW[2]) + D2[1] * Pd[1] * M[1] / B
    Q[0] = D1[0] * (Q[1] @ aW[1]) + D2[0] * Pd[0] * M[0] / B
    accumulate(Q, A, True)
    accumulate([gl / B for gl in g], Hd, False)
    gW[3][0] += Hd[3].sum(0) / B
    return [gW[0], gb[0], gW[1], gb[1], gW[2], gb[2], gW[3], gb[3]]


# ---- the CNF Euler adjoint -------------------------------------------------------------------------------------------
def phi_scales(Ws, bs, x, t, a, c, act):
    """Magnitude version of cnf_train_oracle.phi_grads: (scale of grad_x phi, [scale of grad_theta phi]) for rows x
    (B, dim) at the scalar time t, cotangent bounds a >= 0 (B, dim) and c >= 0 (B,)."""
    aW = [W.abs() for W in Ws]
    ab = [b.abs() for b in bs]
    B, dim = x.shape
    z = torch.cat([x, torch.full((B, 1), float(t), dtype=x.dtype, device=x.device)], 1)
    P0 = aW[0][:, :dim].T                      # (dim, w): |p_{0,k}| = |W0[:, k]|, exact
    d, dd, S, T, Pt = [], [], [z.abs()], [], [P0[None].expand(B, dim, -1)]
    h = z
    for l in range(3):
        pre = h @ Ws[l].T + bs[l]
        h, d1, d2 = _act(pre, act)
        d.append(d1.abs()), dd.append(d2.abs())
        S.append(torch.maximum(h.abs(), d1.abs() * (S[-1] @ aW[l].T + ab[l])))
        T.append(d[l][:, None, :] * Pt[l])   # bound of T_{l,k}
        if l < 2:
            Pt.append(T[l] @ aW[l + 1].T)      # bound of p_{l+1,k}
    tau = [None, None, c[:, None, None] * aW[3][None]]
    e = [None, None, tau[2] * d[2][:, None, :]]
    delta = [None, None, d[2] * (a @ aW[3]) + dd[2] * (tau[2] * Pt[2]).sum(1)]
    for l in (1, 0):
        tau[l] = e[l + 1] @ aW[l + 1]
        e[l] = tau[l] * d[l][:, None, :]
        delta[l] = d[l] * (delta[l + 1] @ aW[l + 1]) + dd[l] * (tau[l] * Pt[l]).sum(1)
    gx = delta[0] @ aW[0][:, :dim]
    gW0 = delta[0].T @ S[0]
    gW0[:, :dim] += e[0].sum(0).T
    g = [gW0, delta[0].sum(0),
         delta[1].T @ S[1] + torch.einsum("bkw,bkv->wv", e[1], T[0]), delta[1].sum(0),
         delta[2].T @ S[2] + torch.einsum("bkw,bkv->wv", e[2], T[1]), delta[2].sum(0),
         a.T @ S[3] + torch.einsum("b,bkw->kw", c, T[2]), a.sum(0)]
    return gx, g


def cnf_grad_scales(state, traj, t_span, G, act="selu"):
    """(scales of the parameter gradients in parameters() order, scale of the input gradient) of L with dL/dtraj = G,
    over the states ``traj`` (n_span, B, dim + 1), with h_n formed in fp32 as the kernel forms it; on traj's device."""
    dev = traj.device
    Ws = [state[f"net.{k}.weight"].detach().to(dev).double() for k in (0, 2, 4, 6)]
    bs = [state[f"net.{k}.bias"].detach().to(dev).double() for k in (0, 2, 4, 6)]
    traj, G = traj.detach().double(), G.detach().to(dev).double().abs()
    dim = traj.shape[2] - 1
    ts = t_span.detach().cpu().float()
    hs = [abs(float(ts[n + 1] - ts[n])) for n in range(len(ts) - 1)]
    ts = ts.double()
    scales = [torch.zeros_like(p) for pair in zip(Ws, bs) for p in pair]
    adj = G[-1].clone()
    for n in range(traj.shape[0] - 2, -1, -1):
        gx, g = phi_scales(Ws, bs, traj[n][:, :dim], ts[n], hs[n] * adj[:, :dim], hs[n] * adj[:, dim], act)
        for acc, v in zip(scales, g):
            acc += v
        adj = G[n] + adj + torch.cat([gx, torch.zeros_like(gx[:, :1])], 1)
    return scales, adj
