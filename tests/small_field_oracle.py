"""TEST INFRASTRUCTURE ONLY -- float64 per-entry error bounds of the small-MLP fields of csrc/ode_small.cu: the MLP
forward of the SDE nets (mlp_eval, sde_small_kernel) and the action-matching gradient field (grad_eval,
ode_grad_kernel); and the step-by-step trajectory bound of both SDE classes (``Bounded``).

Magnitudes follow tests/train_scale_oracle.py: P_l = |W_l| A_{l-1} + |b_l| (+ |t w_time| at layer 0), A_{-1} = |x|,
A_l = max(|a_l|, D_l P_l), with D_l = |act'(pre_l)| widened for the error of the pre-activation the kernel feeds to the
activation.  ``mlp_bounds`` returns one scale F = |W3| A_2 + |b3| per output entry and ``grad_bounds`` one scale
G = |W0x|^T (D0 (.) |W1|^T (D1 (.) |W2|^T (|W3| (.) D2))) per field entry; both bound their entry (|f| <= F, |grad| <= G).

The gate of each entry is the kernel's own arithmetic carried through those magnitudes, u = 2^-24, to first order:
  * a sum of n fmaf terms (every one rounds once) errs by at most n u times the sum of the magnitudes of its terms.
    The chains: layer 0, the time fma and one per input (n_0 = dim + 1, from the staged bias); layers 1 and 2, one per
    hidden unit (w); layer 3 on the dim <= 8 branch, U = w / 32 lane fmas, 5 butterfly adds and the bias add
    (n_3 = U + 6), on the lane-strided branch w fmas from the bias (n_3 = w); the reverse products W^T g, w fmas from 0;
    the gradient's last sum, U lane fmas and 5 butterfly adds (U + 5); and one rounding per product g = w3 act',
    act' (W^T g).  So the pre-activation's error is delta_l = |W_l| E_{l-1} + n_l u P_l, E_{l-1} the error of the
    layer's input.
  * act_apply_fast (mlp_common.cuh): SELU's negative branch is fma(ex2(x log2e), lambda alpha, -lambda alpha); the
    rounded argument moves e^x by |x| u relative, ex2.approx errs by at most 2^-22 = 4 u relative, the fma and the
    rounded constant by u |a| each: act'(x) (|x| + 4) u + 2 u |a|.  SiLU is x / (1 + ex2(-x log2e)) with __fdividef:
    ((|x| + 4)(1 - s) + 3) u relative.  With |x| <= P_l and D_l P_l <= A_l, both are within
    u ((|x| + 7) A_l + 4 D_l) (the last term: ex2's error next to the cancellation in e^x - 1 near 0-).
  * act_deriv_fast: SELU's ex2(x log2e) lambda alpha errs by (|x| + 6) u act'; SiLU's fma(x s, 1 - s, s) by
    (|x| + 8) u (s + |x| s (1 - s)) plus |x| s u from the rounding of 1 - s; within u ((|x| + 8) M_l + |x| s [SiLU]),
    M_l = |act'| (SELU) or s + |x| s (1 - s) (SiLU).
  * the activation at a perturbed pre-activation: |act(p + d) - act(p)| <= D_l d with D_l = |act'(p)| + c d, c the
    largest |act''| within d of p, and max|act'| where SELU's kink lies within d of p (the gradient field leaves such rows out: its act' jumps there).
The forward's error is E_l = D_l delta_l + u ((|pre_l| + 7) A_l + 4 D_l) and the output's |W3| E_2 + n_3 u F.  The
gradient's reverse chain carries D_l + (error of act') in place of D_l, which is where G takes its widened D_l.

tests/test_small_field_oracle_host.py checks that each scale bounds its entry and that an fp32 CPU evaluation errs by
far less than the gate; tests/test_gpu_small_field_edges.py prints the worst measured error over the gate."""
import numpy as np
import torch

import cnf_tc_oracle as ho
from oracle import sde as osde
from oracle import vector_field as vf

U = 2.0**-24
SELU_L, SELU_A = 1.0507009873554805, 1.6732632423543772


def _params(state):
    return ([state[f"net.{k}.weight"].detach().double().cpu() for k in (0, 2, 4, 6)],
            [state[f"net.{k}.bias"].detach().double().cpu() for k in (0, 2, 4, 6)])


def _act(p, act):
    """(act(p), act'(p), M) in float64; M bounds the magnitude act_deriv_fast's error is relative to."""
    if act == "selu":
        d = torch.where(p > 0, torch.full_like(p, SELU_L), SELU_L * SELU_A * torch.exp(p))
        return torch.nn.functional.selu(p), d, d.abs()
    s = torch.sigmoid(p)
    d = s * (1 + p * (1 - s))
    return torch.nn.functional.silu(p), d, s + p.abs() * s * (1 - s)


def _d2(pre, delta, act):
    """A bound of |act''| on [pre - delta, pre + delta] (SELU: on its negative branch; the kink is handled apart)."""
    if act == "selu":
        return torch.where(pre + delta <= 0, SELU_L * SELU_A * torch.exp(torch.clamp(pre + delta, max=0)),
                           torch.zeros_like(pre))
    xm = (pre.abs() - delta).clamp_min(0)  # |SiLU''| <= s (1 - s) (2 + |x|), decreasing in |x| past 3
    s = torch.sigmoid(xm)
    return torch.where(xm < 3, torch.full_like(pre, 0.5), s * (1 - s) * (2 + xm))


def _forward(state, t, x, act):
    """The three hidden layers in float64 with their magnitudes and error bounds: [(pre, a, P, delta, Dw, A, E, M)]."""
    Ws, bs = _params(state)
    x = x.detach().double().cpu()
    dim = x.shape[1]
    w = Ws[1].shape[0]
    slope = SELU_L * SELU_A if act == "selu" else 1.1
    a, A, E = x, x.abs(), torch.zeros_like(x)
    out = []
    for l in range(3):
        Wx = Ws[l][:, :dim] if l == 0 else Ws[l]
        pre = a @ Wx.T + bs[l]
        P = A @ Wx.abs().T + bs[l].abs()
        n = dim + 1 if l == 0 else w
        if l == 0:
            pre = pre + float(t) * Ws[0][:, dim]
            P = P + abs(float(t)) * Ws[0][:, dim].abs()
        delta = E @ Wx.abs().T + n * U * P
        h, d, M = _act(pre, act)
        Dw = d.abs() + _d2(pre, delta, act) * delta
        if act == "selu":
            Dw = torch.where(pre.abs() <= delta, torch.full_like(Dw, slope), Dw)
        A = torch.maximum(h.abs(), Dw * P)
        E = Dw * delta + U * ((pre.abs() + 7) * A + 4 * Dw)
        out.append((pre, h, P, delta, Dw, A, E, M))
        a = h
    return Ws, bs, out


def mlp_bounds(state, t, x, act):
    """(f, F, gate) [B][out] in float64 of mlp_eval at time t on rows x (exact fp32 values): the output, its scale and
    the bound of the kernel's error."""
    Ws, bs, layers = _forward(state, t, x, act)
    w, out_dim = Ws[1].shape[0], Ws[3].shape[0]
    _, a, _, _, _, A, E, _ = layers[2]
    f = a @ Ws[3].T + bs[3]
    F = A @ Ws[3].abs().T + bs[3].abs()
    n3 = w // 32 + 6 if out_dim <= 8 else w
    return f, F, E @ Ws[3].abs().T + n3 * U * F


def grad_bounds(state, t, x, act):
    """(f, G, gate, kink) [B][dim] in float64 of grad_eval at time t on rows x: the field grad_x s, its scale, the bound
    of the kernel's error, and [B] the rows where a SELU pre-activation lies within its own error of the kink (there
    act' may take either side's value, so those rows have no bound)."""
    Ws, bs, layers = _forward(state, t, x, act)
    dim, w = x.shape[1], Ws[1].shape[0]
    w3 = Ws[3][0]
    D, Dw, kink = [], [], torch.zeros(x.shape[0], dtype=torch.bool)
    for pre, _, P, delta, _, _, _, M in layers:
        d = _act(pre, act)[1]
        err_d = U * ((pre.abs() + 8) * M + (0 if act == "selu" else pre.abs() * torch.sigmoid(pre)))
        D.append(d.abs())
        Dw.append(d.abs() + _d2(pre, delta, act) * delta + err_d)
        if act == "selu":
            kink |= (pre.abs() <= delta).any(1)
    g = w3 * _act(layers[2][0], act)[1]
    G2 = w3.abs() * Dw[2]
    err = w3.abs() * (Dw[2] - D[2]) + U * G2
    Gl = G2
    for l in (1, 0):
        g = _act(layers[l][0], act)[1] * (g @ Ws[l + 1])
        M = Gl @ Ws[l + 1].abs()
        err = Dw[l] * (err @ Ws[l + 1].abs() + w * U * M) + (Dw[l] - D[l]) * M + U * Dw[l] * M
        Gl = Dw[l] * M
    W0x = Ws[0][:, :dim]
    f = g @ W0x
    G = Gl @ W0x.abs()
    return f, G, err @ W0x.abs() + (w // 32 + 5) * U * G, kink


def half_ulp(v):
    """Half an fp32 ulp of each entry of v: the rounding of the fp32 state a one-step field is read from."""
    return torch.from_numpy(np.spacing(np.abs(v.detach().cpu().numpy().astype(np.float32))).astype(np.float64) / 2)


# ---- the SDE trajectory bound ---------------------------------------------------------------------------------------
def tc_net_err(state, t, y, act):
    """The fp16x3 pair forward's per-entry error (tests/test_gpu_cnf_tc.py derives F_K)."""
    return ho.F_K * ho.magnitudes(state, t, y, torch.zeros_like(y), act, ho.EPS_GEMM)[0]


def small_net_err(state, t, y, act):
    """mlp_eval's per-entry error (``mlp_bounds``), on y's device."""
    return mlp_bounds(state, t, y, act)[2].to(y.device)


def radius_uniform(seed, n, rows, cols):
    """The float64 uniform under the square root of osde.device_normals' Box-Muller, per (row, column)."""
    rows = np.asarray(rows, dtype=np.uint64)[:, None]
    c = np.arange(cols, dtype=np.uint64)[None, :]
    ctr = np.stack(np.broadcast_arrays(c >> np.uint64(2), rows & np.uint64(0xFFFFFFFF), rows >> np.uint64(32),
                                       np.full_like(c, n)), axis=-1)
    x = osde.philox4x32_10(ctr, np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64))
    u = (x >> np.uint32(8)).astype(np.float64) * 2.0**-24 + 2.0**-25
    return np.where((c & np.uint64(2)).astype(bool), u[..., 2], u[..., 0])


def device_increments(seed, ts, dt, rows, dim):
    """(increments, their error bounds) (n_steps, len(rows), dim) float64 of the device's own noise on the grid of
    (ts, dt): dW_n = sqrt(h_n) z_n with z_n = osde.device_normals(seed, n).  The device increment errs by at most
    sqrt(h_n) (2^-23 / rad + 2^-20 rad + 2^-23 |z|) per entry, rad = sqrt(-2 log u) the Box-Muller radius: the fp32
    rounding of a radius uniform u >= 1/2 moves rad by up to 2^-24 / rad, logf, sqrtf, sincospif and the angle's
    rounding by a few units of 2^-24 of rad, the products by 2^-24 each."""
    grid, _ = osde.step_grid(ts, dt)
    incs, errs = [], []
    for n in range(len(grid) - 1):
        root = float(grid[n + 1] - grid[n]) ** 0.5
        z = osde.device_normals(seed, n, rows, dim)
        rad = np.sqrt(-2.0 * np.log(radius_uniform(seed, n, rows, dim)))
        incs.append(torch.from_numpy(z * root))
        errs.append(torch.from_numpy(root * (2.0**-23 / rad + 2.0**-20 * rad + 2.0**-23 * np.abs(z))))
    return torch.stack(incs), torch.stack(errs)


class Bounded:
    """The float64 drift + score that osde.euler_sdeint calls once per step, carrying the per-entry error bound of the
    device trajectory along.  Step n adds
      * h_n (e_d + e_s): both nets' forward errors, ``net_err`` of each net on the oracle's state (``tc_net_err`` for
        the tensor-core class, ``small_net_err`` for sde_small_kernel);
      * 4 units of 2^-24 of |y_n| + h_n |f_n| + sigma |dW_n|: the fp32 roundings of d + s, the fma, sigma dW and the sum;
      * sigma inc_err[n]: the error of the device's own increment (zero when the increments are supplied).
    Output k gets the sum up to the step that brackets it times exp(T Lip), plus 4 units of 2^-24 of the magnitudes of
    the two states it interpolates (the fp32 interpolation and its fp32 weights)."""

    def __init__(self, nets, act, ts, dt, sigma, incs, inc_err=None, net_err=tc_net_err):
        self.nets, self.act, self.sigma, self.incs, self.inc_err = nets, act, sigma, incs, inc_err
        self.net_err = net_err
        self.states = [{k: v.detach() for k, v in m.state_dict().items()} for m in nets]
        self.grid, bracket = osde.step_grid(ts, dt)
        self.outputs = {}  # step n -> the outputs k it brackets
        for k, n in enumerate(bracket, 1):
            self.outputs.setdefault(n, []).append(k)
        self.n, self.cum, self.at = 0, 0.0, {}

    def __call__(self, t, y):
        n = self.n
        tt = torch.tensor(t, dtype=torch.float64, device=y.device)
        f = sum(vf.wrapped_forward(m, tt, y) for m in self.nets)
        e = sum(self.net_err(st, t, y, self.act) for st in self.states)
        h = float(self.grid[n + 1] - self.grid[n])
        mag = y.abs() + h * f.abs() + self.sigma * self.incs[n].abs()
        self.cum = self.cum + h * e + 4 * 2.0**-24 * mag
        if self.inc_err is not None:
            self.cum = self.cum + self.sigma * self.inc_err[n]
        for k in self.outputs.get(n, []):
            self.at[k] = (self.cum, mag + y.abs())
        self.n += 1
        return f

    def bound(self, grow):
        first = torch.zeros_like(self.at[1][1])  # ys[0] is y0 itself
        return torch.stack([first] + [grow * self.at[k][0] + 4 * 2.0**-24 * self.at[k][1]
                                      for k in range(1, len(self.at) + 1)])
