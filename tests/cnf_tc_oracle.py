"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the Hutchinson likelihood path of the tensor-core class
(csrc/cnf_tc.cu driven by cfm_b200/ode.py), built on oracle/sde.py and oracle/vector_field.py (used unchanged).

* ``device_rademacher`` / ``device_probes``: the probes the kernel draws, entry (r, c) of probe n.  Gaussian: the SDE
  noise stream (``oracle.sde.device_normals``).  Rademacher: -1 where the top bit of Philox word c % 4 of the counter
  (c // 4, r mod 2^32, r >> 32, n) is set, +1 otherwise.
* ``hutch_field``: the reference's ``cnf_wrapper(model, "hutch_*")`` field, d/dt [x, ll] = [f, eps . (J eps)], with
  the probe of each evaluation supplied by ``Probes`` in evaluation order, i.e. with torchdyn's count as ordinal
  (``stats["nfe"]``).  J eps is a forward-mode tangent (``torch.func.jvp``); the reference writes the same number as
  ``(vjp(eps)[0] * eps).sum()`` per row (tests/test_cnf_tc_host.py checks the two agree).
* ``magnitudes``: per-row float64 magnitude chains of one evaluation, the scales the error bounds of
  tests/test_gpu_cnf_tc.py are stated in; ``EPS_GEMM``, ``DIV_K`` and ``F_K``: those bounds (derived there), shared
  by every test of the tensor-core samplers; ``lipschitz``: the growth rate the trajectory bounds carry.
"""
import math

import numpy as np
import torch

from oracle import sde as osde

_MASK = np.uint64(0xFFFFFFFF)
EPS_GEMM = 1e-6
DIV_K, F_K = 10 * EPS_GEMM, 16 * EPS_GEMM


def device_rademacher(seed, n, rows, cols):
    """(len(rows), cols) float64 of +-1: the Rademacher probe entries of ordinal n."""
    rows = np.asarray(rows, dtype=np.uint64)[:, None]
    c = np.arange(cols, dtype=np.uint64)[None, :]
    ctr = np.stack(np.broadcast_arrays(c >> np.uint64(2), rows & _MASK, rows >> np.uint64(32),
                                       np.full_like(c, n)), axis=-1)
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64)
    x = osde.philox4x32_10(ctr, key)
    idx = np.broadcast_to((c & np.uint64(3)).astype(np.int64), x.shape[:2])
    word = np.take_along_axis(x, idx[..., None], -1)[..., 0]
    return np.where(word >> np.uint32(31), -1.0, 1.0)


def device_probes(est, seed, n, rows, cols):
    if est == "hutch_gaussian":
        return osde.device_normals(seed, n, rows, cols)
    if est == "hutch_rademacher":
        return device_rademacher(seed, n, rows, cols)
    raise ValueError(est)


class Probes:
    """The probe of every field evaluation in order: evaluation k (k = 0, 1, ...) gets ordinal k."""

    def __init__(self, est, seed, B, D, rows=None, device="cpu"):
        self.est, self.seed, self.B, self.D, self.device = est, seed, B, D, device
        self.rows = np.arange(B) if rows is None else np.asarray(rows)
        self.n = 0

    def next(self):
        eps = device_probes(self.est, self.seed, self.n, self.rows, self.D)
        self.n += 1
        return torch.from_numpy(eps).to(self.device)


def hutch_div(model, t, x, eps):
    """eps . (J eps) per row, J = d model([x, t]) / dx, as one forward-mode tangent of the batch (rows are
    independent, so the batch's tangent is the per-row one)."""
    tt = t.reshape(()).to(x).expand(x.shape[0])[:, None]
    f, jv = torch.func.jvp(lambda y: model(torch.cat([y, tt], 1)), (x,), (eps,))
    return f, (eps * jv).sum(1)


def hutch_field(model, probes):
    def field(t, z):
        x = z[:, :-1]
        f, div = hutch_div(model, t, x, probes.next().to(x))
        return torch.cat([f, div[:, None]], 1)
    return field


def reference_div(model, t, x, eps):
    """The reference's formulation (models.py div_fn_hutch_trace under torch.vmap): (vjp(eps)[0] * eps).sum()."""
    t = t.reshape(())

    def u(y):
        return model(torch.cat([y, t[None].to(y)]))

    def div(y, e):
        _, pullback = torch.func.vjp(u, y)
        return (pullback(e)[0] * e).sum()

    return torch.vmap(div)(x, eps)


def _acts(act):
    if act == "selu":
        lam, alpha = 1.0507009873554805, 1.6732632423543772
        d1 = lambda p: torch.where(p > 0, torch.full_like(p, lam), lam * alpha * torch.exp(p))  # noqa: E731
        d2max = lam * alpha
        return torch.nn.functional.selu, d1, d2max
    s = torch.sigmoid
    d1 = lambda p: s(p) * (1 + p * (1 - s(p)))  # noqa: E731
    return torch.nn.functional.silu, d1, 0.5


def magnitudes(state, t, x, eps, act, eps_gemm):
    """Per-row float64 scales of one evaluation of the net ``state`` (a state_dict) at (t, x) with probe ``eps``:
    (F [B][D], S [B]).  F = |W3| |a_3| + |b3|: the magnitude of f, the scale of the fp16x3 error of every output
    entry.  S = sum_c |eps_c| (|W3| D_2 |W2| D_1 |W1| D_0 |W0x| |eps|)_c: the magnitude chain of eps . (J eps), with
    D_l = |act'(pre_l)| + max|act''| eps_gemm P_l, where P_l = |W_l| |a_l| + |b_l| (+ |t W0[:, dim]|) bounds the
    pre-activation's own error by eps_gemm P_l (so D_l covers act' evaluated at the perturbed pre-activation)."""
    f_act, d1, d2max = _acts(act)
    W = [state[f"net.{li}.weight"].double().to(x.device) for li in (0, 2, 4, 6)]
    b = [state[f"net.{li}.bias"].double().to(x.device) for li in (0, 2, 4, 6)]
    dim = x.shape[1]
    t = float(t)
    a, u = x, eps.abs()
    for li in range(3):
        Wx = W[li][:, :dim] if li == 0 else W[li]
        pre = a @ Wx.T + b[li]
        P = a.abs() @ Wx.abs().T + b[li].abs()
        if li == 0:
            pre = pre + t * W[0][:, dim]
            P = P + abs(t) * W[0][:, dim].abs()
        D = d1(pre).abs() + d2max * eps_gemm * P
        u = D * (u @ Wx.abs().T)
        a = f_act(pre)
    F = a.abs() @ W[3].abs().T + b[3].abs()
    S = (eps.abs() * (u @ W[3].abs().T)).sum(1)
    return F, S


def lipschitz(mc, act):
    """A Lipschitz bound of the MLP ``mc`` in x: the product of its layers' spectral norms times max|act'|^3."""
    slope = 1.0507009873554805 * 1.6732632423543772 if act == "selu" else 1.1
    norms = [torch.linalg.matrix_norm(mc.net[li].weight.double(), ord=2).item() for li in (0, 2, 4, 6)]
    return math.prod(norms) * slope ** 3
