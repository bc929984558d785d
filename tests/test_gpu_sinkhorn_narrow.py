"""22-bit chunks of the Sinkhorn cost copy (sinkhorn_v2.cu, KG = 4, n1 > 7509): a chunk whose smallest cost encodes
below 2^22 is streamed at 44 bytes per thread and row instead of 48, with the same codes.  Every case here runs in
two fresh interpreters, one with CFM_SK_Q24=1 (every chunk at 3 bytes), and the potentials, status word and drawn
pairs must be the same bits (the marginal error too, up to the order of its float64 atomic sum).  The count of
narrow chunks (workspace control region, byte 288) must match the width rule evaluated on the host from the same
costs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from test_host_compact import _constants  # noqa: E402
from test_host_narrow import LIMIT, _q, cost_with_code  # noqa: E402

DEV = "cuda:0"
REG = 0.05
N_NARROW = 288  # byte offset of the narrow-chunk count in the Sinkhorn workspace


def _slabs(n0):
    """Row slabs of the smem-staged kernel's CTAs (one per SM, sk_slab)."""
    nblk = min(torch.cuda.get_device_properties(0).multi_processor_count, n0)
    base, rem = divmod(n0, nblk)
    out, b0 = [], 0
    for b in range(nblk):
        n = base + (1 if b < rem else 0)
        out.append((b0, b0 + n))
        b0 += n
    return out


def expected_narrow(M, cmax):
    """Chunks (2 rows of one slab) whose smallest cost encodes below 2^22 and that hold no NaN."""
    Mh = M.cpu().numpy()
    c2, kappa = _constants(REG, np.float32(cmax))
    nan_row = np.isnan(Mh).any(1)
    row_min = np.where(nan_row, np.float32(0), np.nanmin(np.where(np.isnan(Mh), np.inf, Mh), 1)).astype(np.float32)
    count = 0
    for lo, hi in _slabs(Mh.shape[0]):
        for r in range(lo, hi, 2):
            rows = slice(r, min(r + 2, hi))
            if not nan_row[rows].any() and _q(row_min[rows].min(keepdims=True), c2, kappa)[0][0] < LIMIT:
                count += 1
    return count


def _uniform_cost(n0, n1, seed, lo=0.6):
    """Costs in [lo, 1) x 1000 with one entry at the maximum 1000: every chunk narrow unless a case lowers a cost."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    M = 1000.0 * (lo + (1.0 - lo) * torch.rand(n0, n1, generator=g, device=DEV))
    M[0, 0] = 1000.0
    return M


def _case_inputs(name):
    """(M, cmax) of a named case; M is n0 x n1 fp32 on the device (contiguous: ldm = n1)."""
    if name.startswith("pitch"):  # n1 across the pitch rule; d = 784 keeps the costs concentrated (narrow)
        from test_gpu_sinkhorn_compact import _cost
        M, cmax = _cost(2048, int(name[5:]), 784, 7)
        return M, cmax
    if name == "mixed":
        # some rows hold a cost below cost_max / 2 (wide chunks): a few scattered rows, a run of chunks, one whole
        # slab, and the ragged 1-row last chunk of slab 0 (63 rows at 132 SMs)
        n = 8192
        M = _uniform_cost(n, n, 11)
        slabs = _slabs(n)
        rows = [5, 62, 700, 701, 2049, 4000, 8191] + list(range(1000, 1040)) + list(range(*slabs[5]))
        rows.append(slabs[0][1] - 1)
        for k, r in enumerate(rows):
            M[r, (97 * k) % n] = 100.0
        return M, M.max().reshape(1)
    if name == "edge":
        # one chunk whose largest code is exactly 2^22 - 1 (narrow) and one at exactly 2^22 (wide)
        n0, n1 = 2048, 8192
        M = _uniform_cost(n0, n1, 12)
        c2, kappa = _constants(REG, np.float32(1000.0))
        M[300, 17] = float(cost_with_code(LIMIT - 1, np.float32(1000.0), c2, kappa))
        M[600, 8000] = float(cost_with_code(LIMIT, np.float32(1000.0), c2, kappa))
        return M, M.max().reshape(1)
    if name == "nan":
        n0, n1 = 2048, 8192
        M = _uniform_cost(n0, n1, 13)
        M[100, 33] = float("nan")
        return M, torch.tensor([1000.0], device=DEV)
    raise KeyError(name)


CASES = ["mixed", "edge", "nan", "pitch7508", "pitch7512", "pitch8192"]


def _run(out):
    """Every case in this interpreter (the format switch is read once per process) -> out (.npz)."""
    from cfm_b200 import _ffi
    from cfm_b200.optimal_transport import OTPlanSampler
    res = {}
    # C2 end to end: cost GEMM, solve, draw and gather through sample_plan
    N, D = 8192, 784
    g = torch.Generator().manual_seed(0)
    x0, x1 = torch.randn(N, D, generator=g).to(DEV), torch.randn(N, D, generator=g).to(DEV)
    s = OTPlanSampler("sinkhorn", reg=REG, normalize_cost=True, num_iter_max=100, stop_thr=0.0, warn=False)
    seen = []
    finish = s._finish
    s._finish = lambda cp: (seen.append(cp), finish(cp))[1]
    np.random.seed(0)
    a, b = s.sample_plan(x0, x1)
    cp, B = seen[-1], s._last_bufs
    res["c2_pairs"] = torch.cat([a, b], 1).cpu().numpy()
    res["c2_lu"], res["c2_lv"] = cp.log_u.cpu().numpy(), cp.log_v.cpu().numpy()
    res["c2_st"], res["c2_err"] = cp.status.cpu().numpy(), cp.err.cpu().numpy()
    res["c2_nn"] = B["ws_sk"][N_NARROW:N_NARROW + 4].cpu().numpy().view(np.int32)
    res["c2_expect"] = np.array([expected_narrow(B["M"][:, :N], float(cp.cost_max.item()))])
    del s, B, cp, x0, x1
    for name in CASES:
        M, cmax = _case_inputs(name)
        n0, n1 = M.shape
        ws = _ffi.workspace(_ffi.lib().cfm_sinkhorn_workspace_bytes(n0, n1), torch.device(DEV))
        s = OTPlanSampler("sinkhorn", reg=REG, normalize_cost=True, precision="fp32", stall_tol=0.0,
                          num_iter_max=100, stop_thr=0.0, warn=False)
        bufs = {"log_u": torch.empty(n0, dtype=torch.float64, device=DEV),
                "log_v": torch.empty(n1, dtype=torch.float64, device=DEV), "ws_sk": ws}
        cp = s._solve_sinkhorn(M, cmax, n0, n1, REG, True, bufs=bufs)
        res[name + "_lu"], res[name + "_lv"] = cp.log_u.cpu().numpy(), cp.log_v.cpu().numpy()
        res[name + "_st"], res[name + "_err"] = cp.status.cpu().numpy(), cp.err.cpu().numpy()
        res[name + "_nn"] = ws[N_NARROW:N_NARROW + 4].cpu().numpy().view(np.int32)
        res[name + "_expect"] = np.array([expected_narrow(M, float(cmax.item()))])
        del M, ws, bufs, cp
        torch.cuda.empty_cache()
    np.savez(out, **res)


@pytest.fixture(scope="module")
def runs(tmp_path_factory):
    d = tmp_path_factory.mktemp("narrow")
    out = {}
    for mode in ("narrow", "q24"):
        env = dict(os.environ)
        env.pop("CFM_SK_Q24", None)
        if mode == "q24":
            env["CFM_SK_Q24"] = "1"
        path = str(d / (mode + ".npz"))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), path], env=env, cwd=os.path.dirname(HERE),
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        out[mode] = dict(np.load(path))
    return out


def _same_bits(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def _same_err(a, b):
    """The marginal error is a float64 sum the CTAs add atomically in whatever order they arrive, so its last bits
    vary from solve to solve with either width; everything else is compared bit for bit."""
    return _same_bits(a, b) or (np.isfinite(a).all() and np.abs(a - b).max() <= 1e-12 * np.abs(b).max())


def _chunks(n0):
    return sum((hi - lo + 1) // 2 for lo, hi in _slabs(n0))


@pytest.mark.gpu
def test_c2_sample_plan_is_bit_identical_to_the_3_byte_stream_and_every_chunk_is_narrow(runs):
    nar, wide = runs["narrow"], runs["q24"]
    for key in ("c2_pairs", "c2_lu", "c2_lv", "c2_st"):
        assert _same_bits(nar[key], wide[key]), key
    assert _same_err(nar["c2_err"], wide["c2_err"])
    assert nar["c2_st"].tolist()[1:] == [100, 0, 4], nar["c2_st"]
    assert int(nar["c2_nn"][0]) == _chunks(8192) == int(nar["c2_expect"][0])
    assert int(wide["c2_nn"][0]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", CASES)
def test_narrow_chunks_are_bit_identical_to_the_3_byte_stream(runs, name):
    nar, wide = runs["narrow"], runs["q24"]
    for key in ("_lu", "_lv", "_st"):
        assert _same_bits(nar[name + key], wide[name + key]), name + key
    assert _same_err(nar[name + "_err"], wide[name + "_err"])
    st = nar[name + "_st"].tolist()
    assert st[1] == 100 and st[3] == 4, st
    expect = int(nar[name + "_expect"][0])
    assert int(nar[name + "_nn"][0]) == (0 if name == "pitch7508" else expect)
    assert int(wide[name + "_nn"][0]) == 0
    n0 = 8192 if name == "mixed" else 2048
    total = _chunks(n0)
    if name == "mixed":
        assert 0 < expect < total - 20  # wide chunks in scattered rows, a run, a whole slab and a ragged chunk
    elif name in ("edge", "nan"):
        assert expect == total - 1  # 2^22 - 1 stays narrow, 2^22 and NaN make their chunks wide
    else:
        assert expect == total


@pytest.mark.gpu
def test_narrow_stream_ignores_stale_workspace():
    """Zeroed, all-ones and foreign workspaces, among them one whose last solve wrote the other width for the same
    chunks (a slab of wide chunks before an all-narrow one and back), give the same bits."""
    from cfm_b200 import _ffi
    from test_gpu_sinkhorn_compact import _solve
    n0, n1 = 2048, 8192
    M = _uniform_cost(n0, n1, 21)
    W = M.clone()
    W[::7, 5] = 10.0  # every slab has wide chunks: carved at the 3-byte pitch
    cm, cw = M.max().reshape(1), W.max().reshape(1)
    ws = _ffi.workspace(_ffi.lib().cfm_sinkhorn_workspace_bytes(n0, n1), torch.device(DEV))
    count = lambda: int(ws[N_NARROW:N_NARROW + 4].cpu().numpy().view(np.int32)[0])  # noqa: E731
    for iters in (1, 2, 3, 11, 100):
        for target, tmax, other, omax in ((M, cm, W, cw), (W, cw, M, cm)):
            got = []
            for history in ("zeros", "ones", "other", "self"):
                if history == "zeros":
                    ws.fill_(0x00)
                elif history == "ones":
                    ws.fill_(0xFF)
                else:
                    src, smax = (other, omax) if history == "other" else (target, tmax)
                    _, _, st2 = _solve(src, smax, n0, n1, "fp32", 100, ws)
                    assert st2[3] == 4
                lu, lv, st = _solve(target, tmax, n0, n1, "fp32", iters, ws)
                assert st[3] == 4 and st[1] == iters
                got.append((lu.cpu().numpy(), lv.cpu().numpy(), count()))
            for lu, lv, nn in got[1:]:
                assert np.array_equal(lu, got[0][0]) and np.array_equal(lv, got[0][1]), iters
                assert nn == got[0][2]
            assert (got[0][2] == _chunks(n0)) == (target is M)


@pytest.mark.gpu
def test_narrow_stream_against_generic_kernel_and_float64_oracle():
    """The float64 oracle gates of the 3-byte stream at a shape whose chunks are all narrow."""
    from cfm_b200 import _ffi
    from test_gpu_sinkhorn_compact import _cost, _solve
    from test_gpu_sinkhorn_compact import test_compact_stream_against_generic_kernel_and_float64_oracle as against
    n0, n1, d = 2048, 8192, 784
    M, cmax = _cost(n0, n1, d, n0 + n1)  # the same costs the gate draws
    ws = _ffi.workspace(_ffi.lib().cfm_sinkhorn_workspace_bytes(n0, n1), torch.device(DEV))
    _solve(M, cmax, n0, n1, "fp32", 3, ws)
    assert int(ws[N_NARROW:N_NARROW + 4].cpu().numpy().view(np.int32)[0]) == _chunks(n0)
    against(n0, n1, d)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    _run(sys.argv[1])


@pytest.mark.gpu
def test_narrow_count_is_cleared_by_solves_that_write_no_copy():
    """Every solver clears the count at its start: after an all-narrow solve, the generic fp32 kernel, a shape whose
    M stays in the L2 and a float64-regime solve on the same workspace leave 0 at byte 288."""
    from cfm_b200 import _ffi
    from test_gpu_sinkhorn_compact import _solve
    n0, n1 = 2048, 8192
    M = _uniform_cost(n0, n1, 31)
    cm = M.max().reshape(1)
    ws = _ffi.workspace(_ffi.lib().cfm_sinkhorn_workspace_bytes(n0, n1), torch.device(DEV))
    count = lambda: int(ws[N_NARROW:N_NARROW + 4].cpu().numpy().view(np.int32)[0])  # noqa: E731
    small = M[:256].contiguous()  # 8 MB: stays in the L2, fp32 sweep without a copy
    for solve in (lambda: _solve(M, cm, n0, n1, "fp32-generic", 3, ws),
                  lambda: _solve(small, cm, 256, n1, "fp32", 3, ws),
                  lambda: _solve(M, cm, n0, n1, "fp64", 3, ws)):
        _solve(M, cm, n0, n1, "fp32", 3, ws)
        assert count() == _chunks(n0)
        solve()
        assert count() == 0
