"""TEST INFRASTRUCTURE ONLY -- float64 restatement of the action-matching gradient field of the tensor-core class
(csrc/grad_tc.cu driven by cfm_b200/ode.py) and the per-entry bound of its error.

* ``field``: v(t, x) = grad_x s(t, x) of the scalar action s = MLP(dim, out_dim=1, w, time_varying=True), written as
  the kernels compute it: a forward pass to layer 2, then g2 = D2 * w3, g1 = D1 * (g2 W2), g0 = D0 * (g1 W1),
  v = g0 W0x with D_l = act'(pre_l) (tests/test_grad_tc_host.py checks it against torch.autograd.grad).
* ``bounds``: the scale M [B][dim] of every entry of v and the rows whose SELU pre-activations lie within their own
  error of the kink at 0.  M = |W0x|^T (D~0 * |W1|^T (D~1 * |W2|^T (D~2 * |w3|))) in row form, where
  D~_l = |act'(pre_l)| + max|act''| EPS_GEMM P_l widens act' by its perturbation from the pre-activation's own error
  bound EPS_GEMM P_l, P_l = |W_l| |a_{l-1}| + |b_l| (+ |t W0[:, dim]|) (as tests/cnf_tc_oracle.magnitudes does for the
  Hutchinson tangent).
* ``GRAD_K``: the gate, GRAD_K M per entry.  An fp16x3 GEMM output errs by at most EPS_GEMM = 1e-6 of its magnitude
  sum |a| |b| (DESIGN 3.0-3.1).  The three reverse GEMMs each contribute EPS_GEMM of their stage of M; the primal
  GEMMs' errors reach v through act', which D~ carries; act_deriv_fast's own error is at most (|pre| + 6) 2^-24 of
  act' (DESIGN 3.11), about EPS_GEMM per layer for |pre| <= 10; the splits add 2^-22 relative per operand and the fp32
  products 2^-24 each: at most (3 + 3 + 1) EPS_GEMM M, gated at GRAD_K = 10 EPS_GEMM M.
* SELU's act' jumps from lambda alpha to lambda at 0: a row with a pre-activation within EPS_GEMM P of 0 may take either
  side, so it leaves the tight gate (the rule of DESIGN 3.11 for the one-launch gradient field).  ``bounds`` returns
  those rows; the tests count them and bound their share.
* ``lipschitz``: a Lipschitz bound of v in x for the trajectory bounds (the three terms of the product rule through
  D0, D1 and D2, with spectral norms).
* ``layer_scales``: the powers of two of both prepared blobs, restated in float32 from gemm_h3.cuh's h3_pow2_scale and
  grad_tc.cu's chain rule: s_0..s_3 and the chain factors {2^k, 2^-k / s_0}.  ``chain_peaks``: the largest |g_l 2^k|
  the three saturating splits of the reverse chain see, in float64.  ``grad_blob``: the prepared gradient blob, byte
  for byte.
"""
import math

import numpy as np
import torch

EPS_GEMM = 1e-6
GRAD_K = 10 * EPS_GEMM
SELU_L, SELU_A = 1.0507009873554805, 1.6732632423543772


def _acts(act):
    """(act, act', max|act'|, max|act''|) in float64."""
    if act == "selu":
        d1 = lambda p: torch.where(p > 0, torch.full_like(p, SELU_L), SELU_L * SELU_A * torch.exp(p))  # noqa: E731
        return torch.nn.functional.selu, d1, SELU_L * SELU_A, SELU_L * SELU_A
    s = torch.sigmoid
    d1 = lambda p: s(p) * (1 + p * (1 - s(p)))  # noqa: E731
    return torch.nn.functional.silu, d1, 1.1, 0.5


def _params(state, device):
    W = [state[f"net.{li}.weight"].double().to(device) for li in (0, 2, 4, 6)]
    b = [state[f"net.{li}.bias"].double().to(device) for li in (0, 2, 4, 6)]
    return W, b


def _forward(state, t, x, act):
    """(pre_l, P_l) for l = 0, 1, 2 in float64."""
    f_act = _acts(act)[0]
    W, b = _params(state, x.device)
    dim = x.shape[1]
    t = float(t)
    a, out = x, []
    for li in range(3):
        Wx = W[li][:, :dim] if li == 0 else W[li]
        pre = a @ Wx.T + b[li]
        P = a.abs() @ Wx.abs().T + b[li].abs()
        if li == 0:
            pre = pre + t * W[0][:, dim]
            P = P + abs(t) * W[0][:, dim].abs()
        out.append((pre, P))
        a = f_act(pre)
    return out


def field(state, t, x, act):
    """v = grad_x s(t, x) [B][dim] in float64 through the kernels' chain."""
    _, d1, _, _ = _acts(act)
    W, _ = _params(state, x.device)
    dim = x.shape[1]
    D = [d1(pre) for pre, _ in _forward(state, t, x, act)]
    g = D[2] * W[3][0]
    g = D[1] * (g @ W[2])
    g = D[0] * (g @ W[1])
    return g @ W[0][:, :dim]


def bounds(state, t, x, act, eps_gemm=EPS_GEMM):
    """(M [B][dim], kink [B] bool): the scale of every entry of v and the rows that leave the tight gate."""
    _, d1, _, d2max = _acts(act)
    W, _ = _params(state, x.device)
    dim = x.shape[1]
    kink = torch.zeros(x.shape[0], dtype=torch.bool, device=x.device)
    Dt = []
    for pre, P in _forward(state, t, x, act):
        Dt.append(d1(pre).abs() + d2max * eps_gemm * P)
        if act == "selu":
            kink |= (pre.abs() <= eps_gemm * P).any(1)
    m = Dt[2] * W[3][0].abs()
    m = Dt[1] * (m @ W[2].abs())
    m = Dt[0] * (m @ W[1].abs())
    return m @ W[0][:, :dim].abs(), kink


def lipschitz(state, act, dim):
    """A Lipschitz bound of v(t, .): sum over l of the chain with D_l replaced by max|act''| times the bound of
    pre_l's own Lipschitz constant."""
    _, _, slope, d2max = _acts(act)
    W, _ = _params(state, "cpu")
    N = [torch.linalg.matrix_norm(W[0][:, :dim], ord=2).item()] + \
        [torch.linalg.matrix_norm(W[li], ord=2).item() for li in (1, 2)]
    n3 = W[3][0].norm().item()
    lp = [N[0], N[0] * N[1] * slope, N[0] * N[1] * N[2] * slope ** 2]  # Lipschitz bounds of pre_0, pre_1, pre_2
    # the term of D_l: every weight norm, the two other D's at most slope each, and max|act''| Lip(pre_l)
    return n3 * math.prod(N) * slope ** 2 * d2max * sum(lp)


# ---- the scales of the prepared blobs (float32, as the kernels form them) ---------------------------------------------
FP16_MAX = 65504.0
ACT_PRIME_MAX = np.float32(1.7581)  # grad_tc.cu's kActPrimeMax: >= max|act'| of SELU (lambda alpha) and SiLU (1.0998)


def _ilogb(v):
    return int(np.frexp(np.float32(v))[1]) - 1


def pow2_scale(am):
    """gemm_h3.cuh's h3_pow2_scale: 2^(13 - ilogb(am)), the exponent clamped to [-100, 100]; 1 for a zero or non-finite
    am."""
    am = np.float32(am)
    if not (am > 0 and am < np.float32(3.0e38)):
        return np.float32(1.0)
    return np.float32(2.0 ** max(-100, min(100, 13 - _ilogb(am))))


def _weights32(state, dim):
    """W0x, W1, W2, W3 as float32 NumPy arrays (W0x = W0[:, :dim])."""
    W = [state[f"net.{li}.weight"].detach().float().cpu().numpy() for li in (0, 2, 4, 6)]
    return [np.ascontiguousarray(W[0][:, :dim])] + W[1:]


def col_abs_sum_max(W):
    """max_i sum_j |W[j, i]| in float32, rows added in order (one thread per column, as grad_chain_scale)."""
    acc = np.zeros(W.shape[1], np.float32)
    for j in range(W.shape[0]):
        acc += np.abs(W[j])
    return np.float32(acc.max())


def layer_scales(state, dim, chain_bound=True):
    """(s_0..s_3, {2^k, 2^-k / s_0}) as cfm_mlp_prepare and cfm_grad_tc_prepare form them.  2^k is the largest power of
    two with max|W3| 2^k < 2^7 (2^k = s_3 2^-7) and, with ``chain_bound``, with every split of the reverse chain bounded
    by 65504: max|act'| max|W3| 2^k max(1, max|act'| C2, max|act'|^2 C2 C1) <= 65504, C_l the largest column
    abs-sum of W_l.  ``chain_bound=False`` is the W3-only rule."""
    W = _weights32(state, dim)
    s = [pow2_scale(np.abs(Wl).max()) for Wl in W]
    k = np.float32(2.0 ** -7) / (np.float32(1) / s[3])
    if chain_bound:
        A = ACT_PRIME_MAX
        m3 = np.float32(np.abs(W[3]).max())
        c1, c2 = col_abs_sum_max(W[1]), col_abs_sum_max(W[2])
        b2 = A * m3
        b1 = b2 * (A * c2)
        b0 = b1 * (A * c1)
        peak = max(b2, b1, b0)
        if peak > 0 and peak <= np.float32(3.0e38):
            with np.errstate(over="ignore"):
                q = np.float32(FP16_MAX) / peak
                lim = np.float32(np.inf) if np.isinf(q) else np.ldexp(np.float32(1), _ilogb(q)).astype(np.float32)
            k = min(k, lim)
    return s, (np.float32(k), (np.float32(1) / s[0]) / np.float32(k))


def chain_peaks(state, t, x, act, sk=None):
    """(max|g2 2^k|, max|g1 2^k|, max|g0 2^k|) in float64: the values the three saturating splits of the reverse chain
    see; 2^k from ``layer_scales`` unless given."""
    _, d1, _, _ = _acts(act)
    W, _ = _params(state, x.device)
    if sk is None:
        sk = float(layer_scales(state, x.shape[1])[1][0])
    D = [d1(pre) for pre, _ in _forward(state, t, x, act)]
    g2 = D[2] * W[3][0] * sk
    g1 = D[1] * (g2 @ W[2])
    g0 = D[0] * (g1 @ W[1])
    return float(g2.abs().max()), float(g1.abs().max()), float(g0.abs().max())


def activation_peak(state, t, x, act):
    """max|a_l| over the two activations the forward splits (layers 0 and 1) and x itself."""
    f_act = _acts(act)[0]
    pre = _forward(state, t, x, act)
    return max(float(x.abs().max()), *(float(f_act(p).abs().max()) for p, _ in pre[:2]))


def grad_blob(state, dim, w):
    """(bytes, regions): the prepared gradient blob of cfm_grad_tc_prepare as a uint8 array, and its defined regions
    [(name, offset, nbytes)] (the 1024-byte alignment gaps between them are not written).  GradBlob's layout: the chain
    factors {2^k, 2^-k / s_0} first, then per layer l = 0, 1, 2 the K-major (W_l s_l)^T [cols][w] split as hi =
    fp16_rn(v), lo = fp16_rn((v - hi) 2^11) (split_h3; NumPy's float16 cast rounds to nearest even like
    __float2half_rn)."""
    W = _weights32(state, dim)
    s, sc = layer_scales(state, dim)

    def align(n):
        return (n + 1023) // 1024 * 1024
    regions, o = [], 0
    parts = [("sc", np.array(sc, np.float32).view(np.uint8))]
    for li in range(3):
        v = np.ascontiguousarray((W[li] * s[li]).T.astype(np.float32))
        hi = v.astype(np.float16)
        lo = ((v - hi.astype(np.float32)) * np.float32(2048)).astype(np.float16)
        parts += [(f"wth{li}", hi.view(np.uint8).ravel()), (f"wtl{li}", lo.view(np.uint8).ravel())]
    for name, p in parts:
        regions.append((name, o, p.size))
        o += align(p.size)
    out = np.zeros(o, np.uint8)
    for (name, off, n), (_, p) in zip(regions, parts):
        out[off:off + n] = p
    return out, regions
