"""The SIMT fp32 GEMM core (gemm_nt_simt_kernel, csrc/gemm_simt.cuh) bit for bit against its NumPy emulation
(tests/simt_oracle.py), in both of its users:

* the cost matrix (cfm_sqdist_f32, csrc/sqdist.cu) with algo 1, and with auto where it routes to SIMT: output tile
  edges on both sides, every K from 1 to 36 (the 16-wide K tile, the float4 quad tail) and a few large ones, the
  float4 and scalar load paths, the float4 and scalar store paths with padding columns, both squared flags, exact
  zeros, the clamp of a negative d2, NaN locality, cost_max across many CTAs, NaN-filled workspaces and 8,388,481 rows
  (more 128-row tiles than gridDim.y's 65535);
* the MLP layers (cfm_mlp_forward_f32 with algo 1, csrc/mlp.cu): the last layer bit for bit from the device's own h2,
  layer 2's activation from the device's own h1 within the documented ulp bounds of expm1f and __expf, and the whole
  network against float64, over a covering sample of batch, input, hidden and output widths, and at 8,388,481 rows.

Every entry of the cost matrix is also held to a float64 gate, so that the emulation is checked as the right
operation and not only as a copy of the kernel.  Its bound is rigorous for the kernel's operation order, with u = 2^-24
and S = |x0_i|^2 + |x1_j|^2: the dot product and the two row norms each carry at most d u (1 + d u) of S (2 |dot| <= S);
adding the norms costs u S; d2 <= 2 S, so the subtraction costs 2 u S, and the square root followed by the square
3 u (2 S).  That sums to (2d + 9) u S plus 2 d^2 u^2 S, under (2d + 10) u S for d <= 4096.

The plan read-out (plan_materialize_kernel, csrc/sinkhorn.cu) had the same grid limit on its rows and is checked here
at 65,536 rows and at 20,000 columns (its 8-block column stride)."""
import re
import subprocess

import numpy as np
import pytest
import torch

import cfm_b200
from cfm_b200 import _ffi
import simt_oracle as so

DEV = "cuda:0"
gpu = pytest.mark.gpu
SENTINEL = -1234.5  # never a cost (costs are >= 0) and never an output of these MLPs
U = 2.0 ** -24
BIG_ROWS = 65535 * 128 + 1  # one row more than 65535 tiles of 128 rows hold


def _offset1(t):
    """A contiguous copy of ``t`` whose data pointer is 4 bytes past a 16-byte boundary (storage offset 1)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4
    return v


def _same_bits(got, ref):
    """Bit equality of two fp32 arrays, any NaN standing for any NaN (the device's and NumPy's NaN payloads differ)."""
    got, ref = np.asarray(got, dtype=np.float32), np.asarray(ref, dtype=np.float32)
    nan = np.isnan(ref)
    if not np.array_equal(np.isnan(got), nan):
        return False
    return np.array_equal(got[~nan].view(np.uint32), ref[~nan].view(np.uint32))


def _first_diff(got, ref):
    bad = np.argwhere(~((got == ref) | (np.isnan(got) & np.isnan(ref))))
    return None if bad.size == 0 else (tuple(bad[0]), got[tuple(bad[0])], ref[tuple(bad[0])], len(bad))


# ===================================================================================== cost matrix
def _sqdist(x0, x1, algo=1, squared=1, ldm=None, m_offset=False):
    """cfm_sqdist_f32 on caller-owned buffers: (M (n0, ldm), cost_max).  M is sentinel-filled (``m_offset``: 4 bytes
    past a 16-byte boundary), the workspace 0xFF-filled (NaN norms until the kernel writes them), cost_max starts at a
    negative sentinel."""
    L = _ffi.lib()
    n0, d = x0.shape
    n1 = x1.shape[0]
    ldm = n1 if ldm is None else ldm
    M = torch.full((n0, ldm), SENTINEL, device=DEV)
    if m_offset:
        M = _offset1(M)
    ws = torch.full((L.cfm_sqdist_workspace_bytes(n0, n1, d, algo),), 0xFF, dtype=torch.uint8, device=DEV)
    cmax = torch.full((1,), SENTINEL, device=DEV)
    _ffi.check(L.cfm_sqdist_f32(_ffi.ptr(x0), _ffi.ptr(x1), _ffi.ptr(M), n0, n1, d, ldm, squared, _ffi.ptr(cmax), algo,
                                _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(torch.device(DEV))), "cfm_sqdist_f32")
    return M, cmax


def _routes_to_simt(x0, x1, ldm, M_ptr):
    """Auto mode's choice (cfm_sqdist_f32): the tensor-core path only for aligned d % 4 == 0 shapes with d >= 32 and
    n0 n1 >= 256^2."""
    n0, d = x0.shape
    aligned = (x0.data_ptr() | x1.data_ptr() | M_ptr) % 16 == 0
    return not (d % 4 == 0 and aligned and ldm % 4 == 0 and n0 * x1.shape[0] >= 256 * 256 and d >= 32)


def _inputs(n0, n1, d, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x0 = torch.randn(n0, d, device=DEV, generator=g)
    x1 = torch.randn(n1, d, device=DEV, generator=g) + 0.25
    return x0, x1


def _f64_ratio(M, a, b):
    """max over entries of |M - exact| / ((2d + 10) u S) (see the module docstring); a, b are the fp32 inputs."""
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    na, nb = (a64 ** 2).sum(1)[:, None], (b64 ** 2).sum(1)[None, :]
    exact = np.maximum(na + nb - 2.0 * a64 @ b64.T, 0.0)
    bound = (2 * a.shape[1] + 10) * U * (na + nb)
    ok = ~np.isnan(M)
    return float((np.abs(M.astype(np.float64) - exact) / np.maximum(bound, 1e-300))[ok].max())


def _check_cost(M, cmax, x0, x1, squared=1, record=None):
    """Every entry and cost_max bit for bit against the emulation, padding columns untouched, and (squared) the
    float64 gate.  Returns the emulated matrix."""
    n1 = x1.shape[0]
    Mh = M.cpu().numpy()
    assert (Mh[:, n1:] == SENTINEL).all()
    a, b = x0.cpu().numpy(), x1.cpu().numpy()
    ref = so.sqdist(a, b, squared)
    got = Mh[:, :n1]
    assert _same_bits(got, ref), _first_diff(got, ref)
    assert _same_bits(cmax.cpu().numpy(), np.array([so.cost_max(ref)])), (cmax.item(), so.cost_max(ref))
    if squared:
        r = _f64_ratio(got, a, b)
        assert r <= 1.0, r
        if record is not None:
            record("f64_error_over_bound", r)
    return ref


_EDGES = [1, 2, 3, 4, 5, 63, 64, 65, 127, 128, 129, 255, 256, 257]
_TILE_EDGES = ([(a, _EDGES[(i + k) % len(_EDGES)]) for k in (0, 5, 9) for i, a in enumerate(_EDGES)]
               + [(1, 257), (257, 1), (1000, 65), (65, 1000)])


@gpu
@pytest.mark.parametrize("n0,n1", _TILE_EDGES)
def test_cost_tile_edges(n0, n1, record_property):
    """Partial 128-row and 128-column tiles and partial float4 column groups on both sides, 1 x N and N x 1, several
    tile rows in one tile column and the reverse.  squared and d alternate; auto mode gives the same bits."""
    squared = (n0 + n1) % 2
    d = 7 if n0 % 2 else 36
    x0, x1 = _inputs(n0, n1, d, seed=n0 * 1000 + n1)
    M, cmax = _sqdist(x0, x1, squared=squared)
    _check_cost(M, cmax, x0, x1, squared, record_property)
    if _routes_to_simt(x0, x1, n1, M.data_ptr()):
        M0, c0 = _sqdist(x0, x1, algo=0, squared=squared)
        assert torch.equal(M0, M) and torch.equal(c0, cmax)


_KS = list(range(1, 37)) + [47, 48, 49, 100, 784, 3072]


@gpu
@pytest.mark.parametrize("d", _KS)
def test_cost_k(d, record_property):
    """Every K tail of the 16-wide K tile and of the float4 quad (d % 4 != 0 takes scalar loads), on 130 x 70 (a
    partial second tile row); auto mode (SIMT: n0 n1 < 256^2) gives the same bits."""
    x0, x1 = _inputs(130, 70, d, seed=d)
    M, cmax = _sqdist(x0, x1)
    _check_cost(M, cmax, x0, x1, 1, record_property)
    M0, c0 = _sqdist(x0, x1, algo=0)
    assert torch.equal(M0, M) and torch.equal(c0, cmax)


@gpu
@pytest.mark.parametrize("d", [4, 36, 100])
def test_cost_load_paths_give_the_same_bits(d):
    """The float4 loads (d % 4 == 0, both operands 16-byte aligned), the scalar loads of one operand 4 bytes past a
    16-byte boundary, and the scalar loads of d - 1 columns: the same data with its last column zero, which the
    scalar path reads as K padding and the other paths as fmaf(0, 0, acc) = acc.  All of them give the same bits."""
    x0, x1 = _inputs(200, 150, d, seed=d + 7)
    x0[:, -1] = 0.0
    x1[:, -1] = 0.0
    M, cmax = _sqdist(x0, x1)
    _check_cost(M, cmax, x0, x1)
    for a, b in ((_offset1(x0), x1), (x0, _offset1(x1)), (x0[:, :-1].contiguous(), x1[:, :-1].contiguous())):
        Mo, co = _sqdist(a, b)
        assert torch.equal(Mo, M) and torch.equal(co, cmax)


_STORES = ["ldm_n1_unaligned_rows", "ldm_rounded_up", "ldm_n1_plus_5", "M_offset1"]


@gpu
@pytest.mark.parametrize("store", _STORES)
def test_cost_store_paths(store):
    """ldm = n1 with n1 % 4 != 0 (rows start off 16 bytes: scalar stores), ldm rounded up to 4 (float4 stores), ldm =
    n1 + 5, and M 4 bytes past a 16-byte boundary; padding columns keep the sentinel."""
    n0, n1, d = 131, 130, 5
    ldm = {"ldm_n1_unaligned_rows": n1, "ldm_rounded_up": 132, "ldm_n1_plus_5": n1 + 5, "M_offset1": 132}[store]
    x0, x1 = _inputs(n0, n1, d, seed=len(store))
    M, cmax = _sqdist(x0, x1, ldm=ldm, m_offset=store == "M_offset1")
    _check_cost(M, cmax, x0, x1)
    M0, c0 = _sqdist(x0, x1, algo=0, ldm=ldm, m_offset=store == "M_offset1")
    assert torch.equal(M0, M) and torch.equal(c0, cmax)


@gpu
@pytest.mark.parametrize("squared", [0, 1])
@pytest.mark.parametrize("d", [1, 3])
def test_cost_identical_rows_and_clamp(d, squared):
    """x1 holds every third row of x0, around a common offset of 1e3 where (a + b) - 2 dot of nearby points rounds
    below 0 and the clamp fires.  At d = 1 the norm and the dot product of a row with itself are the same rounded
    square, so its cost is exactly 0; at d = 3 they are summed in different orders."""
    g = torch.Generator(device=DEV).manual_seed(3)
    x0 = 1e3 + 0.01 * torch.randn(300, d, device=DEV, generator=g)
    x1 = torch.cat([x0[::3], 1e3 + 0.01 * torch.randn(40, d, device=DEV, generator=g)])
    M, cmax = _sqdist(x0, x1, squared=squared)
    ref = _check_cost(M, cmax, x0, x1, squared)
    if d == 1:
        assert (M[torch.arange(0, 300, 3), torch.arange(100)] == 0).all()
    a, b = x0.cpu().numpy(), x1.cpu().numpy()
    d2 = (so.row_sqnorm(a)[:, None] + so.row_sqnorm(b)[None, :]) - np.float32(2) * so.gemm_nt(a, b)
    assert (d2 < 0).sum() > 1000 and (ref == 0).sum() > 1000  # the clamp fires on many entries


@gpu
@pytest.mark.parametrize("d", [3, 36])
def test_cost_nan_stays_in_its_row_and_column(d):
    """A NaN in row i of x0 makes row i of M NaN and one in row j of x1 column j; every other entry keeps the bits of
    the clean run, and cost_max is the largest of them."""
    n0, n1 = 300, 390
    x0, x1 = _inputs(n0, n1, d, seed=d)
    M, _ = _sqdist(x0, x1)
    i, j = 129, 200
    y0, y1 = x0.clone(), x1.clone()
    y0[i, d // 2] = float("nan")
    y1[j, d - 1] = float("nan")
    N, cmax = _sqdist(y0, y1)
    _check_cost(N, cmax, y0, y1)
    assert N[i].isnan().all() and N[:, j].isnan().all()
    keep = torch.ones(n0, n1, dtype=torch.bool, device=DEV)
    keep[i], keep[:, j] = False, False
    assert torch.equal(N[keep], M[keep])
    assert cmax.item() == N[keep].max().item()


@gpu
def test_cost_max_across_many_ctas():
    """40 x 8 CTAs; the farthest pair sits in the last tile of the last tile row, and a second run moves it to the
    first tile.  cost_max is the matrix's maximum both times."""
    x0, x1 = _inputs(5000, 1000, 3, seed=11)
    for row, col in ((4999, 999), (0, 0)):
        y0, y1 = x0.clone(), x1.clone()
        y0[row] = 40.0
        y1[col] = -40.0
        M, cmax = _sqdist(y0, y1)
        assert M.argmax().item() == row * 1000 + col
        _check_cost(M, cmax, y0, y1)


def _emulate_rows(a, b, rows, squared=1):
    """Emulated cost rows ``rows`` of x0 = a against all of b (the row norms of b once)."""
    return so.sqdist_epilogue(so.gemm_nt(a[rows], b), so.row_sqnorm(a[rows])[:, None], so.row_sqnorm(b)[None, :],
                              squared)


@gpu
def test_cost_more_tile_rows_than_grid_dim_y(record_property):
    """8,388,481 rows (65,536 tiles of 128 rows, one more than gridDim.y holds), 3 columns, d = 2: every entry and
    cost_max bit for bit, chunk by chunk, and the float64 gate."""
    g = torch.Generator(device=DEV).manual_seed(12)
    x0 = torch.randn(BIG_ROWS, 2, device=DEV, generator=g)
    x1 = torch.randn(3, 2, device=DEV, generator=g)
    M, cmax = _sqdist(x0, x1)
    a, b, Mh = x0.cpu().numpy(), x1.cpu().numpy(), M.cpu().numpy()
    del M
    worst, top = 0.0, np.float32(0.0)
    for s in range(0, BIG_ROWS, 1 << 20):
        rows = slice(s, min(s + (1 << 20), BIG_ROWS))
        ref = _emulate_rows(a, b, rows)
        assert _same_bits(Mh[rows], ref), (s, _first_diff(Mh[rows], ref))
        top = max(top, so.cost_max(ref))
        worst = max(worst, _f64_ratio(Mh[rows], a[rows], b))
    assert cmax.item() == top
    assert worst <= 1.0
    record_property("f64_error_over_bound", worst)


# ===================================================================================== MLP layers
def _align256(n):
    return (n + 255) // 256 * 256


def _mlp(dim, w, out_dim, act, seed, tv=True, regime="normal"):
    """(device MLP, its fp32 parameters as NumPy arrays).  ``regime`` moves layer 2's pre-activations: "near_zero"
    scales W2 and b2 by 1e-4; "large_negative" shifts b2 by -95 (SiLU's __expf(-x) overflows below -88.7)."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=tv)
    with torch.no_grad():
        if regime == "near_zero":
            m.net[4].weight.mul_(1e-4)
            m.net[4].bias.mul_(1e-4)
        elif regime == "large_negative":
            m.net[4].bias.sub_(95.0)
    m.act = _ffi.ACT_SILU if act == "silu" else _ffi.ACT_SELU
    m = m.to(DEV)
    P = [p.detach().cpu().numpy() for lin in m._linears() for p in (lin.weight, lin.bias)]
    return m, P


def _forward(m, x, t=None, t_dev=None, y_offset=False):
    """cfm_mlp_forward_f32 with algo 1 on caller-owned buffers: (y, h1, h2).  The workspace starts 0xFF-filled.  mlp.cu
    writes layer 0 to hA at offset 0, layer 1 to hB at align_up(B w 4, 256), layer 2 to hA again and layer 3 to y, so
    afterwards the workspace holds h2 = layer 2's output at offset 0 and h1 = layer 1's at align_up(B w 4, 256)."""
    L = _ffi.lib()
    B, dim = x.shape
    tv = int(m.time_varying)
    blob = m._prepared(bool(tv), torch.device(DEV))
    nbytes = L.cfm_mlp_workspace_bytes(B, dim, m.w, m.out_dim, 1)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    y = torch.full((B, m.out_dim), SENTINEL, device=DEV)
    if y_offset:
        y = _offset1(y)
    _ffi.check(L.cfm_mlp_forward_f32(_ffi.ptr(blob), _ffi.ptr(x), B, dim, m.w, m.out_dim, tv, _ffi.ptr(t_dev),
                                     0.0 if t is None else float(t), m.act, _ffi.ptr(y), 1, _ffi.ptr(ws), nbytes,
                                     _ffi.stream_ptr(torch.device(DEV))), "cfm_mlp_forward_f32")
    n = B * m.w * 4
    h2 = ws[:n].view(torch.float32).view(B, m.w)
    h1 = ws[_align256(n):_align256(n) + n].view(torch.float32).view(B, m.w)
    return y, h1, h2


def _act64(v, act):
    v = v.astype(np.float64)
    if act == "selu":
        return 1.0507009873554804934193349852946 * np.where(v > 0, v, 1.6732632423543772848170429916717 * np.expm1(v))
    with np.errstate(over="ignore"):
        return v / (1.0 + np.exp(-v))


def _act_bound(pre, ref, act):
    """Per-entry bound on |fp32 activation - float64 activation| of the fp32 pre-activation ``pre``.
    SELU: expm1f is within 1 ulp (CUDA Math API), 2 u relative, and the product with the branch's coefficient and that
    constant's rounding add u each: 4 u to first order, 4.5 u with the higher-order terms and the float64 reference.
    SiLU, x / (1 + __expf(-x)): __expf(y) is within 2 + floor(|1.173 y|) ulp (CUDA Math API, intrinsics), an error
    that reaches the result scaled by e / (1 + e), plus the rounding of the sum and of the quotient; below x = -88.7
    __expf overflows and the device returns -0 where |silu(x)| < 2^-120."""
    r = np.abs(ref)
    if act == "selu":
        return 4.5 * U * r + 2.0 ** -140
    x = pre.astype(np.float64)
    with np.errstate(over="ignore"):
        e = np.exp(-x)
        frac = np.where(np.isinf(e), 1.0, e / (1.0 + e))
    return (frac * (2 + np.floor(np.abs(1.173 * x))) * 2 * U + 3 * U) * r + 2.0 ** -120


def _mlp64(P, x, t, act, tv=True):
    h = x.astype(np.float64)
    if tv:
        h = np.concatenate([h, np.full((h.shape[0], 1), float(np.float32(t)))], 1)
    for k in range(4):
        h = h @ P[2 * k].astype(np.float64).T + P[2 * k + 1]
        if k < 3:
            h = _act64(h, act)
    return h


def _check_layers(y, h1, h2, P, act, rows=slice(None)):
    """The last layer bit for bit from the device's h2; layer 2's activation from the device's h1 within
    _act_bound.  Returns the largest layer-2 error over its bound."""
    yh, h1h, h2h = (t[rows].cpu().numpy() for t in (y, h1, h2))
    ref_y = so.bias_act_pre(so.gemm_nt(h2h, P[6]), P[7])
    assert _same_bits(yh, ref_y), _first_diff(yh, ref_y)
    pre = so.bias_act_pre(so.gemm_nt(h1h, P[4]), P[5])
    ref2 = _act64(pre, act)
    ratio = np.abs(h2h.astype(np.float64) - ref2) / _act_bound(pre, ref2, act)
    assert ratio.max() <= 1.0, (ratio.max(), np.unravel_index(ratio.argmax(), ratio.shape))
    return float(ratio.max())


def _gate64(y, ref):
    err = np.abs(y.astype(np.float64) - ref).max()
    assert err <= 1e-5 * np.abs(ref).max(), (err, np.abs(ref).max())


_BS, _DIMS = [1, 2, 127, 128, 129, 257], [1, 2, 3, 4, 5, 15, 16, 17, 33]
_WS, _OUTS = [3, 4, 16, 50, 64, 127, 129, 256], [1, 2, 3, 4, 5, 129]
# a covering sample: every value of every list at least once, in 12 different combinations
_MLP_SHAPES = [(_BS[i % 6], _DIMS[i % 9], _WS[(5 * i) % 8], _OUTS[(i + i // 6) % 6]) for i in range(12)]


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("B,dim,w,out_dim", _MLP_SHAPES)
def test_mlp_layers(B, dim, w, out_dim, act, record_property):
    """The gates of _check_layers and float64 end to end; t as a host float and as a device scalar give the same bits
    in y and in the workspace."""
    m, P = _mlp(dim, w, out_dim, act, seed=B + 10 * dim + w)
    x = torch.randn(B, dim, device=DEV, generator=torch.Generator(device=DEV).manual_seed(dim))
    y, h1, h2 = _forward(m, x, t=0.37)
    assert y.shape == (B, out_dim)
    record_property("act_error_over_bound", _check_layers(y, h1, h2, P, act))
    _gate64(y.cpu().numpy(), _mlp64(P, x.cpu().numpy(), 0.37, act))
    yd, h1d, h2d = _forward(m, x, t_dev=torch.tensor([0.37], device=DEV))
    assert torch.equal(yd, y) and torch.equal(h1d, h1) and torch.equal(h2d, h2)


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("regime", ["near_zero", "large_negative"])
def test_mlp_activation_regimes(regime, act, record_property):
    """Layer 2's pre-activations within 1e-3 of 0 (expm1f's small arguments, SiLU's x / 2), and around -95 (SELU's
    saturation at -scale alpha, SiLU's __expf overflow)."""
    m, P = _mlp(5, 129, 3, act, seed=5, regime=regime)
    x = torch.randn(300, 5, device=DEV, generator=torch.Generator(device=DEV).manual_seed(6))
    y, h1, h2 = _forward(m, x, t=0.8)
    pre = so.bias_act_pre(so.gemm_nt(h1.cpu().numpy(), P[4]), P[5])
    if regime == "near_zero":
        assert np.abs(pre).max() < 1e-3 and (pre < 0).any() and (pre > 0).any()
    else:
        assert pre.max() < -88.8
    record_property("act_error_over_bound", _check_layers(y, h1, h2, P, act))
    _gate64(y.cpu().numpy(), _mlp64(P, x.cpu().numpy(), 0.8, act))


@gpu
@pytest.mark.parametrize("which", ["time_varying_false", "x_offset1", "y_offset1"])
def test_mlp_layout_cases(which):
    """time_varying=False (no time column in layer 0), and x or y 4 bytes past a 16-byte boundary: the misaligned runs
    give the aligned run's bits."""
    tv = which != "time_varying_false"
    m, P = _mlp(17, 50, 5, "selu", seed=21, tv=tv)
    x = torch.randn(257, 17, device=DEV, generator=torch.Generator(device=DEV).manual_seed(22))
    y, h1, h2 = _forward(m, x, t=0.25 if tv else None)
    _check_layers(y, h1, h2, P, "selu")
    _gate64(y.cpu().numpy(), _mlp64(P, x.cpu().numpy(), 0.25, "selu", tv=tv))
    if tv:
        ya, h1a, h2a = _forward(m, _offset1(x) if which == "x_offset1" else x, t=0.25, y_offset=which == "y_offset1")
        assert torch.equal(ya, y) and torch.equal(h1a, h1) and torch.equal(h2a, h2)


@gpu
def test_mlp_more_tile_rows_than_grid_dim_y(record_property):
    """B = 8,388,481 rows at dim 2, w 3, out_dim 2 (a shape only the SIMT path takes): the last layer bit for bit and
    layer 2's activation on every row, chunk by chunk; float64 end to end on 4096 sampled rows, the tiles around tile
    row 65535 and the last one."""
    m, P = _mlp(2, 3, 2, "selu", seed=31)
    x = torch.randn(BIG_ROWS, 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(32))
    assert not m.tc_path(BIG_ROWS)
    y, h1, h2 = _forward(m, x, t=0.6)
    worst = 0.0
    for s in range(0, BIG_ROWS, 1 << 21):
        worst = max(worst, _check_layers(y, h1, h2, P, "selu", slice(s, min(s + (1 << 21), BIG_ROWS))))
    record_property("act_error_over_bound", worst)
    g = torch.Generator().manual_seed(33)
    rows = torch.cat([torch.randint(0, BIG_ROWS, (4096,), generator=g), torch.arange(128),
                      torch.arange(BIG_ROWS - 257, BIG_ROWS)])
    _gate64(y[rows.to(DEV)].cpu().numpy(), _mlp64(P, x[rows.to(DEV)].cpu().numpy(), 0.6, "selu"))


# ===================================================================================== plan read-out
@gpu
@pytest.mark.parametrize("precision", ["fp32", "fp64"])
@pytest.mark.parametrize("n0,n1", [(65536, 16), (3, 20000)])
def test_get_map_plan_entries(n0, n1, precision):
    """get_map's float64 plan entry by entry against exp((double)(-fl32(fl32(M / cmax) / reg)) + log_u + log_v) from
    the device's own M, cost_max and potentials, within 2 ulp: 65,536 rows (one more than gridDim.y holds), and
    20,000 columns (8 blocks of 256 threads striding over them)."""
    g = torch.Generator(device=DEV).manual_seed(n0 + n1)
    x0 = torch.randn(n0, 2, device=DEV, generator=g)
    x1 = torch.randn(n1, 2, device=DEV, generator=g) + 0.5
    reg = 0.05
    s = cfm_b200.OTPlanSampler("sinkhorn", reg=reg, normalize_cost=True, warn=False, num_iter_max=30,
                               stop_thr=0.0, precision=precision)
    P = s.get_map(x0, x1)
    assert P.shape == (n0, n1)
    B = s._last_bufs
    M = B["M"][:, :n1].cpu().numpy()
    cmax = np.float32(B["cmax"].item())
    lu, lv = B["log_u"].cpu().numpy(), B["log_v"].cpu().numpy()
    q = (M.astype(np.float64) / np.float64(cmax)).astype(np.float32)  # correctly rounded fp32 divisions
    q = (q.astype(np.float64) / np.float64(np.float32(reg))).astype(np.float32)
    ref = np.exp((-q.astype(np.float64) + lu[:, None]) + lv[None, :])
    assert np.isfinite(ref).all() and ref.sum() > 0.5
    assert (np.abs(P - ref) <= 2 * np.spacing(ref)).all()


# ===================================================================================== instantiation guard
def test_compiled_simt_gemm_instantiations_are_the_tested_ones(lib_built):
    """Reads the kernels out of the library's cubin; no device needed.  A new user of the SIMT GEMM core needs cases
    in this file first."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    syms = set(re.findall(r"\w*gemm_nt_simt_kernel\w*", out))
    parsed = {s: re.search(r"gemm_nt_simt_kernelINS_\d+(\w+?)EEEv", s) for s in syms}
    assert syms and all(parsed.values()), syms
    assert {p.group(1) for p in parsed.values()} == {"SqDistEpilogue", "BiasActEpilogue"}
