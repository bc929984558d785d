"""The two fp16x3 tensor-core kernels behind the headline workloads, edge by edge against float64:

* the cost matrix on the persistent wgmma GEMM core (gemm_wg_kernel<H3Scheme, SqDistH3Epilogue>, csrc/gemm_tc.cuh,
  gemm_h3.cuh, sqdist_h3.cu) through cfm_sqdist_f32 with algo 3 and auto: every K tail from d = 4 up, output tile
  edges on both sides, several tiles per CTA with the 3-stage ring's parity wrapping inside a tile (nk = 1, 2, 3, 4),
  padding columns of M, stale workspaces, cost_max, squared = 0, the auto routing to SIMT and NaN locality;
* the fused four-layer MLP (mlp_fused_h3_kernel, csrc/mlp_h3.cu, w = 256): layer-1 K tails with odd and even chunk
  counts, partial output tiles, slab counts around the SM count, four different per-layer weight scales, both
  activations, t on the host and on the device, time_varying=False, the split-input entry and its skip flag, rows of
  y past the batch, stale workspaces and misaligned pointers (auto mode falls back to SIMT, algo 2 refuses).

Each cost entry is gated at 2.5e-6 of |x0_i|^2 + |x1_j|^2 (its own scale, not the matrix's); each MLP output at 1e-5
of max|ref|.  The oracles run in float64 on the device.  Batch and tile counts derive from the SM count, so every
case keeps its meaning on a part with a different one.  The per-layer tensor-core MLP has its own cases in
tests/test_gpu_small_fields.py.
"""
import re
import subprocess

import pytest
import torch

import cfm_b200
from cfm_b200 import _ffi
from oracle import vector_field as vf

DEV = "cuda:0"
gpu = pytest.mark.gpu
SENTINEL = -1234.5  # never a cost (costs are >= 0) and never an output of these MLPs


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _launches(fn):
    L = _ffi.lib()
    torch.cuda.synchronize()
    before = L.cfm_launch_count()
    out = fn()
    return out, L.cfm_launch_count() - before


def _offset1(t):
    """A contiguous copy of ``t`` whose data pointer is 4 bytes past a 16-byte boundary (storage offset 1)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    v = buf[1:].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4
    return v


# ===================================================================================== cost matrix
def _ws_bytes(n0, n1, d, algo):
    return _ffi.lib().cfm_sqdist_workspace_bytes(n0, n1, d, algo)


def _sqdist(x0, x1, algo=3, squared=1, ldm=None, M=None, ws=None):
    """cfm_sqdist_f32 on caller-owned buffers: (M (n0, ldm), cost_max).  ldm defaults to n1 rounded up to the 4 the
    tensor-core path needs, M to a sentinel-filled matrix and the workspace to a zeroed one of the size algo 3
    needs."""
    L = _ffi.lib()
    n0, d = x0.shape
    n1 = x1.shape[0]
    ldm = (n1 + 3) // 4 * 4 if ldm is None else ldm
    if M is None:
        M = torch.full((n0, ldm), SENTINEL, device=DEV)
    if ws is None:
        ws = torch.zeros(_ws_bytes(n0, n1, d, 3), dtype=torch.uint8, device=DEV)
    cmax = torch.full((1,), SENTINEL, device=DEV)
    _ffi.check(L.cfm_sqdist_f32(_ffi.ptr(x0), _ffi.ptr(x1), _ffi.ptr(M), n0, n1, d, ldm, squared, _ffi.ptr(cmax), algo,
                                _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(torch.device(DEV))), "cfm_sqdist_f32")
    return M, cmax


def _inputs(n0, n1, d, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x0 = torch.randn(n0, d, device=DEV, generator=g)
    x1 = torch.randn(n1, d, device=DEV, generator=g) + 0.25
    return x0, x1


def _ref64(x0, x1):
    """(float64 |x0_i - x1_j|^2, float64 |x0_i|^2 + |x1_j|^2): the exact cost and each entry's scale."""
    a, b = x0.double(), x1.double()
    na, nb = a.pow(2).sum(1)[:, None], b.pow(2).sum(1)[None, :]
    return (na + nb - 2.0 * a @ b.T).clamp_min(0.0), na + nb


def _rel_err(M, x0, x1):
    ref, scale = _ref64(x0, x1)
    return ((M[:, :x1.shape[0]].double() - ref).abs() / scale).max().item()


def _check_cost(M, cmax, x0, x1):
    n1 = x1.shape[0]
    Mv = M[:, :n1]
    assert (M[:, n1:] == SENTINEL).all()  # padding columns
    assert torch.isfinite(Mv).all() and (Mv >= 0).all()
    assert _rel_err(M, x0, x1) <= 2.5e-6
    assert cmax.item() == Mv.max().item()


_K_TAILS = list(range(4, 65, 4)) + [68, 124, 128, 132, 188, 192, 196, 252, 256, 260, 784, 1024]


@gpu
@pytest.mark.parametrize("d", _K_TAILS)
def test_cost_k_tail(d):
    """Every K tail of the 64-wide K-chunk (d % 64 from 4 to 60 and 0), on a ragged 300 x 257 output."""
    x0, x1 = _inputs(300, 257, d, seed=d)
    M, cmax = _sqdist(x0, x1)
    _check_cost(M, cmax, x0, x1)


_EDGES = [1, 31, 32, 33, 127, 128, 129, 255, 257]
_TILE_EDGES = [(a, _EDGES[(i + k) % len(_EDGES)]) for k in (0, 3) for i, a in enumerate(_EDGES)]


@gpu
@pytest.mark.parametrize("n0,n1", _TILE_EDGES)
def test_cost_tile_edges(n0, n1):
    """Partial 128-row and 128-column tiles and partial 32-column epilogue chunks, every edge on both sides."""
    d = 36 if n0 % 2 else 100
    x0, x1 = _inputs(n0, n1, d, seed=n0 * 1000 + n1)
    M, cmax = _sqdist(x0, x1)
    _check_cost(M, cmax, x0, x1)


@gpu
@pytest.mark.parametrize("shape", ["sm_rows_minus_5_x_545", "sm_rows_plus_1_x_384"])
@pytest.mark.parametrize("d", [32, 64, 128, 192, 256])
def test_cost_ring_parity_across_tiles(shape, d):
    """Three to five output tiles per CTA with nk = ceil(d / 64) in {1, 2, 3, 4}: the producer and the consumers carry
    the 3-stage ring's stage and parity from tile to tile, so tile k starts at ring position k nk.  For nk = 1, 2, 4
    successive tiles start at every stage and cross the ring's wrap (where the parity flips) at a different chunk each
    time; nk = 3 starts every tile at stage 0 with the other parity.  The first shape gives every CTA five tiles, the
    second gives three CTAs a fourth one."""
    s = _sms()
    n0, n1 = (128 * s - 5, 4 * 128 + 33) if shape.startswith("sm_rows_minus") else (128 * s + 1, 3 * 128)
    x0, x1 = _inputs(n0, n1, d, seed=d + n1)
    M, cmax = _sqdist(x0, x1)
    _check_cost(M, cmax, x0, x1)
    assert torch.equal(_sqdist(x0, x1, algo=0)[0], M)  # auto takes this path


@gpu
def test_cost_padding_columns_and_stale_workspace():
    """Columns of M past n1 (ldm > n1) keep their bits, and neither a 0xFF-filled workspace nor one left over from
    a call at another shape changes a bit of M or cost_max."""
    n0, n1, d, ldm = 300, 257, 196, 268
    x0, x1 = _inputs(n0, n1, d, seed=5)
    ws = torch.zeros(_ws_bytes(n0, n1, d, 3) + _ws_bytes(1000, 700, 260, 3), dtype=torch.uint8, device=DEV)
    outs = []
    for fill in ("zeros", "ones", "other_shape_first"):
        if fill == "zeros":
            ws.zero_()
        elif fill == "ones":
            ws.fill_(0xFF)
        else:
            ws.fill_(0xFF)
            y0, y1 = _inputs(1000, 700, 260, seed=6)
            _sqdist(y0 * 3.0, y1, ws=ws)
        M, cmax = _sqdist(x0, x1, ldm=ldm, ws=ws)
        assert (M[:, n1:] == SENTINEL).all()
        outs.append((M, cmax))
    _check_cost(outs[0][0], outs[0][1], x0, x1)
    for M, cmax in outs[1:]:
        assert torch.equal(M, outs[0][0]) and torch.equal(cmax, outs[0][1])


@gpu
def test_cost_max_is_reset_on_every_call():
    x0, x1 = _inputs(640, 520, 128, seed=7)
    ws = torch.zeros(_ws_bytes(640, 520, 128, 3), dtype=torch.uint8, device=DEV)
    cm, prev = torch.zeros(1, device=DEV), None
    for scale in (1.0, 0.5, 0.25):  # smaller data into the same cost_max buffer: the maximum must come down
        a0, a1, M = x0 * scale, x1 * scale, torch.empty(640, 520, device=DEV)
        _ffi.check(_ffi.lib().cfm_sqdist_f32(
            _ffi.ptr(a0), _ffi.ptr(a1), _ffi.ptr(M), 640, 520, 128, 520, 1, _ffi.ptr(cm), 3,
            _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(torch.device(DEV))), "cfm_sqdist_f32")
        assert cm.item() == M.max().item()
        assert prev is None or cm.item() < prev
        prev = cm.item()


@gpu
@pytest.mark.parametrize("n0,n1,d", [(300, 257, 64), (129, 1000, 784), (2048, 2048, 1024)])
def test_cost_unsquared(n0, n1, d):
    """squared = 0: the distance itself; its square is gated as the squared cost is (plus the rounding of the
    square root), and cost_max is the largest distance."""
    x0, x1 = _inputs(n0, n1, d, seed=n0 + d)
    D, cmax = _sqdist(x0, x1, squared=0)
    assert (D[:, n1:] == SENTINEL).all()
    D = D[:, :n1]
    ref = torch.cdist(x0.double(), x1.double())
    _, scale = _ref64(x0, x1)
    assert ((D.double().pow(2) - ref.pow(2)).abs() <= 2.5e-6 * scale + 2.0 ** -20 * ref.pow(2)).all()
    assert cmax.item() == D.max().item()


_ROUTES = ["x0_offset1", "x1_offset1", "M_offset1", "ldm_not_multiple_of_4", "d_below_32", "below_256x256"]


@gpu
@pytest.mark.parametrize("route", _ROUTES)
def test_cost_auto_routes_to_simt(route):
    """Auto mode sends what the tensor-core path cannot or should not take to SIMT: the result is the algo 1 result
    bit for bit, and a workspace sized for algo 1 suffices (algo 3's would be needed on the other path)."""
    n0, n1, d = (255, 256, 64) if route == "below_256x256" else (300, 260, 28 if route == "d_below_32" else 64)
    ldm = n1 + 2 if route == "ldm_not_multiple_of_4" else n1
    x0, x1 = _inputs(n0, n1, d, seed=len(route))
    if route == "x0_offset1":
        x0 = _offset1(x0)
    if route == "x1_offset1":
        x1 = _offset1(x1)

    def m_buf():
        if route == "M_offset1":
            return _offset1(torch.full((n0, ldm), SENTINEL, device=DEV))
        return torch.full((n0, ldm), SENTINEL, device=DEV)

    ws = torch.zeros(_ws_bytes(n0, n1, d, 1), dtype=torch.uint8, device=DEV)
    M_auto, c_auto = _sqdist(x0, x1, algo=0, ldm=ldm, M=m_buf(), ws=ws)
    M_simt, c_simt = _sqdist(x0, x1, algo=1, ldm=ldm, M=m_buf(), ws=ws)
    assert torch.equal(M_auto, M_simt) and torch.equal(c_auto, c_simt)
    assert _rel_err(M_auto, x0, x1) <= 2.5e-6
    if route in ("x0_offset1", "x1_offset1", "M_offset1", "ldm_not_multiple_of_4"):
        with pytest.raises(_ffi.CfmLibraryError, match="tensor-core path needs"):
            _sqdist(x0, x1, algo=3, ldm=ldm, M=m_buf())


@gpu
def test_cost_auto_takes_the_tensor_cores_when_it_can():
    """The control of the routing cases: aligned, d >= 32 and n0 n1 >= 256^2 is the algo 3 result, and a workspace
    sized for algo 1 is refused."""
    x0, x1 = _inputs(300, 260, 64, seed=9)
    assert torch.equal(_sqdist(x0, x1, algo=0)[0], _sqdist(x0, x1, algo=3)[0])
    ws = torch.zeros(_ws_bytes(300, 260, 64, 1), dtype=torch.uint8, device=DEV)
    with pytest.raises(_ffi.CfmLibraryError, match="workspace too small"):
        _sqdist(x0, x1, algo=0, ws=ws)


@gpu
@pytest.mark.parametrize("d", [64, 200])
def test_cost_nan_stays_in_its_row_and_column(d):
    """A NaN in row i of x0 makes row i of M NaN and one in row j of x1 column j; every other entry keeps the bits
    of the clean run (the row scales of the pre-pass ignore NaN)."""
    n0, n1 = 300, 390
    x0, x1 = _inputs(n0, n1, d, seed=d)
    M, _ = _sqdist(x0, x1)
    i, j = 127, 200
    y0, y1 = x0.clone(), x1.clone()
    y0[i, d // 2] = float("nan")
    y1[j, 3] = float("nan")
    N, cmax = _sqdist(y0, y1)
    assert (N[:, n1:] == SENTINEL).all()
    M, N = M[:, :n1], N[:, :n1]
    assert N[i].isnan().all() and N[:, j].isnan().all()
    keep = torch.ones(n0, n1, dtype=torch.bool, device=DEV)
    keep[i], keep[:, j] = False, False
    assert torch.equal(N[keep], M[keep])
    assert cmax.item() == N[keep].max().item()


# ===================================================================================== fused MLP
def _mlp(dim, out_dim=None, act="selu", seed=0, factors=None, time_varying=True):
    """(device MLP with w = 256, float64 device state) with the same weights; ``factors`` scale W0..W3."""
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=256, time_varying=time_varying)
    if factors is not None:
        with torch.no_grad():
            for lin, f in zip(m._linears(), factors):
                lin.weight.mul_(f)
    if act == "silu":
        m.act = _ffi.ACT_SILU
    m = m.to(DEV)
    state = {k: v.double() for k, v in m.state_dict().items()}
    return m, state


def _ref_vf(state, x, t, act):
    inp = torch.cat([x.double(), torch.full((x.shape[0], 1), t, dtype=torch.float64, device=x.device)], 1)
    return vf.mlp_forward_from_state(state, inp, act=act)


def _gate(y, ref):
    err = (y.double() - ref).abs().max().item()
    assert err <= 1e-5 * ref.abs().max().item(), (err, ref.abs().max().item())


def _fused_vf(m, t, x, **kw):
    """m.vector_field under no_grad, asserting that it ran as the input split plus ONE fused launch."""
    with torch.no_grad():
        m.vector_field(t, x, **kw)  # prepares the weights
        y, n = _launches(lambda: m.vector_field(t, x, **kw))
    assert n == 2, n  # the per-layer path takes 5 launches, SIMT 4
    return y


def _x(B, dim, seed):
    return torch.randn(B, dim, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed))


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", [64, 72, 120, 128, 136, 192, 200, 256, 264, 520, 784, 1024])
def test_mlp_fused_layer1_k_tails(dim, act):
    """Layer 1 over K = dim: a partial last chunk for dim % 64 != 0, an odd or even chunk count nk1 (the second
    128-column pass then starts in the other layer-1 stage); t given as a host float and as a CUDA scalar."""
    m, state = _mlp(dim, act=act, seed=dim)
    x = _x(1000, dim, seed=dim + 1)
    y = _fused_vf(m, 0.37, x)
    _gate(y, _ref_vf(state, x, 0.37, act))
    assert torch.equal(_fused_vf(m, torch.tensor([0.37], device=DEV), x), y)


@gpu
@pytest.mark.parametrize("out_dim", [4, 60, 124, 128, 132, 252, 256, 260, 784, 1028])
def test_mlp_fused_output_tiles(out_dim):
    """t4 = ceil(out_dim / 128) layer-4 tiles, the last one with a partial 32-column chunk or only 4 columns."""
    m, state = _mlp(128, out_dim=out_dim, seed=out_dim)
    x = _x(700, 128, seed=out_dim)
    y = _fused_vf(m, 0.8, x)
    assert y.shape == (700, out_dim)
    _gate(y, _ref_vf(state, x, 0.8, "selu"))


_SLABS = ["one_slab", "one_slab_plus_one_row", "one_slab_per_cta", "one_more_slab_than_ctas", "three_per_cta_ragged"]


@gpu
@pytest.mark.parametrize("slabs", _SLABS)
def test_mlp_fused_slab_counts(slabs):
    """128-row slabs: one, a one-row last slab, exactly one per CTA, one more than the CTAs (a CTA runs a second,
    one-row slab) and three per CTA with a ragged last one (barrier parities across slabs)."""
    s = _sms()
    B = {"one_slab": 128, "one_slab_plus_one_row": 129, "one_slab_per_cta": 128 * s,
         "one_more_slab_than_ctas": 128 * s + 1, "three_per_cta_ragged": 3 * 128 * s - 5}[slabs]
    m, state = _mlp(200, out_dim=132, act="silu", seed=B)
    x = _x(B, 200, seed=B)
    y = _fused_vf(m, 0.1, x)
    _gate(y, _ref_vf(state, x, 0.1, "silu"))


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim", [784, 128])
def test_mlp_fused_per_layer_weight_scales(dim, act):
    """Each layer's epilogue divides by its own power-of-two weight scale.  With nn.Linear's init every layer gets
    the same one, so W0..W3 are multiplied by 1, 3, 0.2 and 11: four different scales (2^-5, 2^-3, 2^-7, 2^-1 of
    max|W| at dim 784), and an epilogue that used another layer's scale would be off by a power of 2."""
    m, state = _mlp(dim, act=act, seed=11, factors=(1.0, 3.0, 0.2, 11.0))
    exps = {torch.frexp(lin.weight.detach().abs().max())[1].item() for lin in m._linears()}
    assert len(exps) == 4, exps
    x = _x(3000, dim, seed=12)
    y = _fused_vf(m, 0.6, x)
    _gate(y, _ref_vf(state, x, 0.6, act))


@gpu
def test_mlp_fused_forward_without_time_column():
    """MLP.forward runs the kernel with time_varying = 0 (no t column in the first-layer bias): on a time_varying=False
    model, and on a time_varying=True one whose input already carries t as its last column."""
    for tv, dim in ((False, 200), (True, 199)):
        m, state = _mlp(dim, out_dim=72, seed=13, time_varying=tv)
        x = _x(1500, 200, seed=14)
        if tv:
            x[:, -1] = 0.45
        with torch.no_grad():
            m(x)
            y, n = _launches(lambda: m(x))
        assert n == 2, n
        _gate(y, vf.mlp_forward_from_state(state, x))


@gpu
def test_mlp_fused_image_like_inputs():
    """Integers 0..255 at dim 784, as raw pixel data: large, exactly representable inputs."""
    m, state = _mlp(784, seed=15)
    g = torch.Generator(device=DEV).manual_seed(16)
    x = torch.randint(0, 256, (2000, 784), device=DEV, generator=g).float()
    y = _fused_vf(m, 0.5, x)
    _gate(y, _ref_vf(state, x, 0.5, "selu"))


def _split(x):
    """The fp16x3 operand pair of an in-range fp32 x, checked in float64: hi + lo 2^-11 is x to 2^-22 relative, or to
    2^-36 absolute where lo is an fp16 subnormal (half its spacing 2^-24, times 2^-11; the unscaled activation-side
    operands have no row scale that keeps them normal)."""
    hi = x.half()
    lo = ((x - hi.float()) * 2048.0).half()
    rec = hi.double() + lo.double() / 2048.0
    assert ((rec - x.double()).abs() <= 2.0 ** -22 * x.double().abs() + 2.0 ** -36).all()
    return hi, lo


@gpu
@pytest.mark.parametrize("act", ["selu", "silu"])
def test_mlp_fused_split_input_and_skip_flag(act):
    """vector_field_split on the (hi, lo) pair of x gives vector_field's bits on x; with a non-zero skip flag the
    kernel returns at once and out keeps its sentinel."""
    B, dim = 1300, 136
    m, _ = _mlp(dim, out_dim=260, act=act, seed=17)
    x = _x(B, dim, seed=18)
    t = torch.tensor([0.3], device=DEV)
    y = _fused_vf(m, t, x)
    hi, lo = _split(x)
    out = torch.full((B, 260), SENTINEL, device=DEV)
    skip = torch.zeros(1, dtype=torch.int32, device=DEV)
    with torch.no_grad():
        _, n = _launches(lambda: m.vector_field_split(t, hi, lo, out, skip))
    assert n == 1 and torch.equal(out, y)
    out.fill_(SENTINEL)
    skip.fill_(7)
    with torch.no_grad():
        m.vector_field_split(t, hi, lo, out, skip)
    assert (out == SENTINEL).all()


@gpu
def test_mlp_fused_rows_past_the_batch_are_untouched():
    B, out_dim = 1000, 132
    m, state = _mlp(128, out_dim=out_dim, seed=19)
    x = _x(B, 128, seed=20)
    big = torch.full((B + 130, out_dim), SENTINEL, device=DEV)
    y = _fused_vf(m, 0.25, x, out=big[:B])
    assert y.data_ptr() == big.data_ptr()
    assert (big[B:] == SENTINEL).all()
    assert torch.equal(big[:B], _fused_vf(m, 0.25, x))
    _gate(big[:B], _ref_vf(state, x, 0.25, "selu"))


@gpu
@pytest.mark.parametrize("batch", ["ragged", "two_slabs_per_cta"])
def test_mlp_fused_stale_workspace(batch):
    """Through the C ABI: a workspace full of 0xFF (NaN as fp16, in the input split and the park buffers) gives the
    bits of a zeroed one."""
    L = _ffi.lib()
    B = 1000 if batch == "ragged" else 2 * 128 * _sms() - 77
    dim, out_dim = 200, 260
    m, state = _mlp(dim, out_dim=out_dim, seed=21)
    x = _x(B, dim, seed=22)
    blob = m._prepared(True, torch.device(DEV))
    nbytes = L.cfm_mlp_workspace_bytes(B, dim, 256, out_dim, 2)
    outs = []
    for fill in (0x00, 0xFF):
        ws = torch.full((nbytes,), fill, dtype=torch.uint8, device=DEV)
        y = torch.full((B, out_dim), SENTINEL, device=DEV)

        def run():
            _ffi.check(L.cfm_mlp_forward_f32(_ffi.ptr(blob), _ffi.ptr(x), B, dim, 256, out_dim, 1, None, 0.7,
                                             _ffi.ACT_SELU, _ffi.ptr(y), 2, _ffi.ptr(ws), nbytes,
                                             _ffi.stream_ptr(torch.device(DEV))), "cfm_mlp_forward_f32")
        _, n = _launches(run)
        assert n == 2
        outs.append(y)
    assert torch.equal(outs[0], outs[1])
    _gate(outs[0], _ref_vf(state, x, 0.7, "selu"))


@gpu
@pytest.mark.parametrize("which", ["x", "out"])
def test_mlp_misaligned_pointer_in_auto_mode_takes_simt(which):
    """A contiguous x or out 4 bytes past a 16-byte boundary: auto mode returns the SIMT result (4 launches) instead of
    failing on the tensor-core path's alignment check; algo 2 refuses a misaligned x."""
    B, dim = 1000, 784
    m, state = _mlp(dim, seed=23)
    x = _x(B, dim, seed=24)
    with torch.no_grad():
        m.mlp_algo = 1
        y_simt = m.vector_field(0.5, x)
        m.mlp_algo = 0
        xa = _offset1(x) if which == "x" else x
        out = _offset1(torch.full((B, dim), SENTINEL, device=DEV)) if which == "out" else None
        y, n = _launches(lambda: m.vector_field(0.5, xa, out=out))
    assert n == 4, n
    assert torch.equal(y, y_simt)
    _gate(y, _ref_vf(state, x, 0.5, "selu"))
    if which == "x":
        m.mlp_algo = 2
        with torch.no_grad(), pytest.raises(_ffi.CfmLibraryError, match="16-byte aligned"):
            m.vector_field(0.5, xa)


# ===================================================================================== instantiation guard
def test_compiled_tensor_core_gemm_instantiations_are_the_tested_ones(lib_built):
    """Reads the kernels out of the library's cubin; no device needed.  A new gemm_wg_kernel or mlp_fused_h3_kernel
    instantiation needs cases in this file first."""
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout

    def args(kernel, pattern):
        syms = set(re.findall(r"\w*%s\w*" % kernel, out))
        parsed = {s: re.search(kernel + pattern, s) for s in syms}
        assert syms and all(parsed.values()), syms  # every instantiation has template arguments of the known form
        return {p.groups() for p in parsed.values()}

    assert args("gemm_wg_kernel", r"INS_\d+(\w+?)ENS_\d+(\w+?)EEEv") == {("H3Scheme", "SqDistH3Epilogue"),
                                                                        ("H3Scheme", "MlpH3Epilogue")}
    assert args("mlp_fused_h3_kernel", r"ILi(\d+)EEEv") == {(str(_ffi.ACT_SELU),), (str(_ffi.ACT_SILU),)}
