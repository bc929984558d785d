"""The tensor-core samplers at their buffer and operand edges: one Hutchinson evaluation (csrc/cnf_tc.cu) with
per-layer weight scales, f and div at every 4-byte offset, the operand pair instead of x, rows past the batch and
stale workspaces; the SDE pair forward (mlp_pair_h3_kernel, csrc/mlp_h3.cu) with rows past the batch and stale
workspaces.  The shapes come from tests/tc_sampler_cases.py; the float64 gates are those of tests/test_gpu_cnf_tc.py
(DIV_K S, F_K F of cnf_tc_oracle)."""
import ctypes

import pytest
import torch

import tc_sampler_cases as tc
from test_gpu_cnf_tc import ESTS, _field, _pair, every_row_against_float64
from test_gpu_sde_tc import _nets, _split

from cfm_b200 import _ffi

DEV = "cuda:0"
pytestmark = pytest.mark.gpu
SENTINEL = -1234.5  # never an output of these nets
# (B, dim, w, act): partial hidden chunks, an 8-column hidden N tile, K tails and a one-row last M tile; a partial
# output chunk and 25 fold chunks at dim 784
EDGE_SHAPES = [(257, 72, 136, "selu"), (129, 784, 200, "silu")]


def _x(B, dim, seed):
    return torch.randn(B, dim, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _both(m, x, **kw):
    """f and div of both estimators at one (t, x)."""
    return [_field(m, x, 0.45, est, 77 + k, 5, **kw) for k, est in enumerate(ESTS)]


def _equal(a, b):
    return all(torch.equal(p, q) for u, v in zip(a, b) for p, q in zip(u, v))


# ---- one Hutchinson evaluation ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,dim,w,act", [(*s, a) for s, a in zip(tc.SCALE_SHAPES, ("selu", "silu"))])
def test_field_per_layer_weight_scales(B, dim, w, act):
    """Each primal and tangent GEMM divides by its own layer's power-of-two weight scale.  With nn.Linear's init the
    layers share one, so W0..W3 are multiplied by 1, 3, 0.2 and 11: four different scales, and an epilogue that used
    a neighbouring layer's would be off by a power of 2."""
    m, mc = _pair(dim, w, 61, act)
    with torch.no_grad():
        for li, k in zip((0, 2, 4, 6), tc.SCALE_FACTORS):
            m.net[li].weight.mul_(k)
            mc.net[li].weight.mul_(k)
    exps = {torch.frexp(m.net[li].weight.detach().abs().max())[1].item() for li in (0, 2, 4, 6)}
    assert len(exps) == 4, exps
    every_row_against_float64(m, mc, _x(B, dim, 62), act, f"scales {B}x{dim}x{w}")


@pytest.mark.parametrize("B,dim,w,act", EDGE_SHAPES)
def test_field_f_and_div_at_every_4_byte_offset(B, dim, w, act):
    """f at 1, 2 and 3 floats into a larger buffer (the per-element store of full chunks; dopri5's stage outputs
    lie there whenever B (D + 1) % 4 != 0), div likewise: the bits of the aligned call."""
    m, _ = _pair(dim, w, 63, act)
    x = _x(B, dim, 64)
    want = _both(m, x)
    for off in (1, 2, 3):
        fbuf = torch.full((B * dim + 4,), SENTINEL, device=DEV)
        dbuf = torch.full((B + 4,), SENTINEL, device=DEV)
        f, div = fbuf[off:off + B * dim].view(B, dim), dbuf[off:off + B]
        for k, est in enumerate(ESTS):
            _field(m, x, 0.45, est, 77 + k, 5, f=f, div=div)
            assert torch.equal(f, want[k][0]) and torch.equal(div, want[k][1]), (off, est)
        for buf, n in ((fbuf, B * dim), (dbuf, B)):
            assert bool((buf[:off] == SENTINEL).all()) and bool((buf[off + n:] == SENTINEL).all()), off


@pytest.mark.parametrize("B,dim,w,act", EDGE_SHAPES)
def test_field_on_the_operand_pair_of_either_split(B, dim, w, act):
    """(x_hi, x_lo) instead of x gives the same f and div bits, for the pair split4_store writes (the Euler init
    kernel) and the pair rk_split_h3 writes (a dopri5 stage input with dt = 0, i.e. x itself): on finite, in-range x
    the two splits and the plain fp16x3 split agree."""
    L = _ffi.lib()
    m, _ = _pair(dim, w, 65, act)
    x = _x(B, dim, 66)
    want = _both(m, x)
    sp = _ffi.stream_ptr(DEV)
    half = dict(dtype=torch.float16, device=DEV)
    # split4_store: the Hutchinson Euler init on z = [x, 0]
    z = torch.cat([x, torch.zeros(B, 1, device=DEV)], 1).contiguous()
    st = torch.zeros(ctypes.sizeof(_ffi.CnfTcState), dtype=torch.uint8, device=DEV)
    xs, ll = torch.empty(B, dim, device=DEV), torch.empty(B, device=DEV)
    traj = torch.empty(2, B, dim + 1, device=DEV)
    span = torch.tensor([0.0, 1.0], device=DEV)
    h4, l4 = torch.empty(B, dim, **half), torch.empty(B, dim, **half)
    _ffi.check(L.cfm_cnf_tc_euler_init(_ffi.ptr(st), _ffi.ptr(z), _ffi.ptr(xs), _ffi.ptr(ll), _ffi.ptr(h4),
                                       _ffi.ptr(l4), _ffi.ptr(traj), _ffi.ptr(span), 2, 1, B, dim, sp), "euler init")
    # rk_split_h3: stage 1 of a zeroed dopri5 state (dt = 0) writes the split of x + 0 k
    rk = torch.zeros(ctypes.sizeof(_ffi.RkState), dtype=torch.uint8, device=DEV)
    k0, t_stage = torch.zeros(B * dim, device=DEV), torch.zeros(1, device=DEV)
    hr, lr = torch.empty(B, dim, **half), torch.empty(B, dim, **half)
    _ffi.check(L.cfm_rk_stage_input(_ffi.ptr(rk), _ffi.ptr(x), _ffi.ptr(k0), None, _ffi.ptr(hr), _ffi.ptr(lr),
                                    _ffi.ptr(t_stage), None, B * dim, 1, sp), "stage input")
    hi, lo = _split(x)
    assert torch.equal(h4, hi) and torch.equal(l4, lo) and torch.equal(hr, hi) and torch.equal(lr, lo)
    for pair in ((h4, l4), (hr, lr)):
        assert _equal(_both(m, None, pair=pair), want)


@pytest.mark.parametrize("B,dim,w,act", EDGE_SHAPES)
def test_field_leaves_rows_past_the_batch_untouched(B, dim, w, act):
    m, _ = _pair(dim, w, 67, act)
    x = _x(B, dim, 68)
    want = _both(m, x)
    f = torch.full((B + 130, dim), SENTINEL, device=DEV)
    div = torch.full((B + 130,), SENTINEL, device=DEV)
    for k, est in enumerate(ESTS):
        _field(m, x, 0.45, est, 77 + k, 5, f=f, div=div)
        assert torch.equal(f[:B], want[k][0]) and torch.equal(div[:B], want[k][1]), est
        assert bool((f[B:] == SENTINEL).all()) and bool((div[B:] == SENTINEL).all()), est


@pytest.mark.parametrize("B,dim,w,act", EDGE_SHAPES)
def test_field_ignores_a_stale_workspace(B, dim, w, act):
    """The act' buffer, the tangent and primal ping-pong buffers and the div partials are reused across layers and
    calls: a workspace of NaN (every byte 0xFF) and one left over from a larger batch give the bits of a zeroed one."""
    L = _ffi.lib()
    m, _ = _pair(dim, w, 69, act)
    x = _x(B + 300, dim, 70)
    nbytes = L.cfm_cnf_tc_workspace_bytes(B + 300, dim, w)
    fresh = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    want = _both(m, x[:B], ws=fresh)
    nan = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    assert _equal(_both(m, x[:B], ws=nan), want)
    left = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    _both(m, x, ws=left)
    assert _equal(_both(m, x[:B], ws=left), want)


# ---- the SDE pair forward ---------------------------------------------------------------------------------------------
# (B, dim, w, act): the pair kernel with a ragged second slab; the per-layer path
PAIR_EDGES = [(129, 72, 256, "selu"), (200, 32, 128, "silu")]


def _pair_forward(blobs, hi, lo, B, dim, w, act, ya, yb, ws):
    L = _ffi.lib()
    t = torch.tensor([0.37], device=DEV)
    _ffi.check(L.cfm_mlp_pair_forward_split_f32(
        _ffi.ptr(blobs[0]), _ffi.ptr(blobs[1]), _ffi.ptr(hi), _ffi.ptr(lo), B, dim, w, dim, 1, _ffi.ptr(t), 0.0, act,
        _ffi.ptr(ya), _ffi.ptr(yb), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(DEV)), "pair")


def _pair_case(B, dim, w, act, seed):
    (d, _), (s, _) = _nets(dim, w, seed=seed, act=act)
    blobs = [n._prepared(True, torch.device(DEV)) for n in (d, s)]
    hi, lo = _split(_x(B + 300, dim, seed + 1))
    nbytes = 2 * _ffi.lib().cfm_mlp_workspace_bytes(B + 300, dim, w, dim, 2)
    return d.act, blobs, hi, lo, nbytes


@pytest.mark.parametrize("B,dim,w,act", PAIR_EDGES)
def test_pair_leaves_rows_past_the_batch_untouched(B, dim, w, act):
    code, blobs, hi, lo, nbytes = _pair_case(B, dim, w, act, 71)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    want = [torch.empty(B, dim, device=DEV) for _ in range(2)]
    _pair_forward(blobs, hi[:B], lo[:B], B, dim, w, code, *want, ws)
    got = [torch.full((B + 130, dim), SENTINEL, device=DEV) for _ in range(2)]
    _pair_forward(blobs, hi[:B], lo[:B], B, dim, w, code, *got, ws)
    for g, y in zip(got, want):
        assert torch.isfinite(y).all() and torch.equal(g[:B], y) and bool((g[B:] == SENTINEL).all())


@pytest.mark.parametrize("B,dim,w,act", PAIR_EDGES)
def test_pair_ignores_a_stale_workspace(B, dim, w, act):
    """The park buffers (fused) and the activation ping-pong (per-layer) of both nets: a NaN workspace and one left
    over from a larger batch give the bits of a zeroed one."""
    code, blobs, hi, lo, nbytes = _pair_case(B, dim, w, act, 73)

    def run(ws, rows=B):
        y = [torch.empty(rows, dim, device=DEV) for _ in range(2)]
        _pair_forward(blobs, hi[:rows], lo[:rows], rows, dim, w, code, *y, ws)
        return y
    want = run(torch.zeros(nbytes, dtype=torch.uint8, device=DEV))
    for a, b in zip(run(torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)), want):
        assert torch.equal(a, b)
    left = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    run(left, B + 300)
    for a, b in zip(run(left), want):
        assert torch.equal(a, b)
