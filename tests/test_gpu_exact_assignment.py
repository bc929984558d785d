"""The exact assignment solver (assign.cu) on every code path its launcher picks, up to the n = 8192 that exact OT
accepts (equal batches, or the lcm-replicated problem of two unequal ones).  cfm_assign_exact_f32 picks the path
from n alone: assign_fast_kernel<KCB> up to n = 4096, with KCB = 1, 2 or 4 columns per thread and the first
cache_rows rows of M staged in shared memory; above that assign_kernel, with its per-column arrays in shared memory
while they fit and in the global workspace beyond.  The sizes tested are the edges of those classes, derived from a
restatement of the launcher's rule, and every solve is compared with SciPy's linear_sum_assignment on the same fp32
costs in float64.

The two kernels start from different greedy matchings (assign_kernel: each row claims its row-minimum column; the
fast kernel then also reduces the columns and lets each free column claim its column-minimum row), and every
augmentation matches exactly one more row.  So on a finite matrix the augmentation count in status[1] is predicted
exactly by a NumPy restatement of the start, which also shows which kernel ran.

The tests stop short of n = 8192 in global memory (N_E2E, and an lcm of 5700 for unequal batches): a solve there
takes 25-32 s on an H100.  SciPy takes most of this module's time (half a minute of host time and more for each
squared-distance matrix above 5000), so each matrix is solved by SciPy once, and every solve the selected tests
need is started on a thread pool before the first test runs."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest
import torch

from cfm_b200 import _ffi
from cfm_b200.optimal_transport import OTPlanSampler
from oracle import coupling as oc
from test_gpu_round2 import _unequal_batch_sizes_vs_lp

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SMEM_CAP = 200 * 1024  # shared memory either kernel may take (cfm_assign_exact_f32)
N_MAX = 8192           # _MAX_EXPANDED: the largest replicated problem exact OT accepts
N_E2E = 6144           # global memory; a solve at N_MAX takes 32 s on an H100 (700 W), this one about 15 s


def _launch_class(n):
    """The launch cfm_assign_exact_f32 makes for n: kernel, threads nt, columns per thread KCB, rows of M staged in
    shared memory (fast kernel), and where the per-column arrays live."""
    nt = min(1024, max(64, -(-n // 32) * 32))
    if n <= 4096:
        kcb = -(-n // nt)
        kcb = 4 if kcb == 3 else kcb
        cache_rows = min(n, max(0, SMEM_CAP - (32 * n + 16)) // (4 * n))
        return dict(kernel=f"fast<{kcb}>", nt=nt, kcb=kcb, cache_rows=cache_rows, mode="smem")
    smem = (29 * n + 7) // 8 * 8 + 8 * n + 16  # asg_smem_bytes
    return dict(kernel="assign_kernel", nt=nt, kcb=0, cache_rows=0, mode="smem" if smem <= SMEM_CAP else "global")


def _regime(n):
    c = _launch_class(n)
    return (c["kernel"], c["mode"],
            c["nt"] == 64,                      # the 64-thread floor
            n <= c["nt"] - 32,                  # a whole warp of padding columns
            n <= (c["kcb"] - 1) * c["nt"],      # the last column slot is padding on every thread
            c["cache_rows"] == n)               # every row of M staged in shared memory


def _describe(n):
    c = _launch_class(n)
    return f"{n}-{c['kernel']}-{c['mode']}-nt{c['nt']}-cache{c['cache_rows']}"


# both sides of every change of regime; then the first n of every regime but the smallest
BOUNDARY_N = sorted({m for n in range(2, N_MAX + 1) if _regime(n) != _regime(n - 1) for m in (n - 1, n)})
EDGE_N = [n for n in BOUNDARY_N if _regime(n) != _regime(n - 1)]


def _greedy_matches(M, normalize, two_claim):
    """Rows matched by the kernels' greedy start, restated in float64 NumPy for a finite M.
    - Costs are float64(fp32(M / max M)) with normalize (fp32 division rounds to nearest, like __fdiv_rn).
    - u_i is the row minimum, ties to the lowest column.  In ascending row order, each row claims its argmin column
      if that column is free.
    - two_claim (the fast kernel): v_j = min_i (c_ij - u_i), ties to the lowest row.  In ascending column order, each
      free column claims its argmin row if that row is free too."""
    M = np.asarray(M, dtype=np.float32)
    C = (M / M.max() if normalize else M).astype(np.float64)
    n = C.shape[0]
    row4col, col4row = np.full(n, -1), np.full(n, -1)
    for i, j in enumerate(C.argmin(1)):
        if row4col[j] < 0:
            row4col[j], col4row[i] = i, j
    if two_claim:
        for j, i in enumerate((C - C.min(1)[:, None]).argmin(0)):
            if row4col[j] < 0 and col4row[i] < 0:
                row4col[j], col4row[i] = i, j
    return int((col4row >= 0).sum())


def _predicted_augmentations(M, normalize=False):
    n = M.shape[0]
    return n - _greedy_matches(M, normalize, two_claim=n <= 4096)


# ---- the cost matrices and their SciPy solutions, each computed once ---------------------------------------------
_MATS = {}    # (kind, n) -> fp32 host matrix
_SCIPY = {}   # (kind, n) -> Future of SciPy's sigma on that matrix in float64
_POOL = ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1))


def _matrix(kind, n):
    """The fp32 matrix of a case.  'normalized' is the 'gauss' matrix over its maximum (what the kernel solves with
    normalize = 1); for 'nan', SciPy gets +inf where the kernel gets NaN; 'device' is the device cost kernel's M."""
    key = (kind, n)
    if key in _MATS:
        return _MATS[key]
    g = torch.Generator().manual_seed(n)
    if kind in ("gauss", "device"):
        x0, x1 = torch.randn(n, 8, generator=g), torch.randn(n, 8, generator=g) * 1.5 + 0.3
        if kind == "gauss":
            M = oc.cost_matrix(x0, x1)
        else:
            M = OTPlanSampler("exact")._cost(x0.to(DEV), x1.to(DEV), torch.device(DEV))[0][:, :n].cpu()
    elif kind == "normalized":
        Mg = _matrix("gauss", n).numpy()
        M = torch.from_numpy(Mg / Mg.max())
    elif kind == "mixed_sign":
        M = torch.randn(n, n, generator=g)
    elif kind == "integer":
        M = torch.randint(0, 4, (n, n), generator=g).float()
    elif kind == "sparse":  # +inf off the union of two random permutations
        M = torch.full((n, n), float("inf"))
        rows = torch.arange(n)
        for _ in range(2):
            M[rows, torch.randperm(n, generator=g)] = torch.rand(n, generator=g)
    elif kind == "nan":  # a few NaN entries per row, never a whole row or column
        M = torch.randn(n, n, generator=g)
        M[torch.arange(n).repeat_interleave(3), torch.randint(0, n, (3 * n,), generator=g)] = float("nan")
        assert not M.isnan().all(0).any() and not M.isnan().all(1).any()
    else:
        raise ValueError(kind)
    _MATS[key] = M
    return M


def _scipy(kind, n):
    key = (kind, n)
    if key not in _SCIPY:
        M = _matrix(kind, n)
        if kind == "nan":
            M = torch.where(M.isnan(), float("inf"), M)
        _SCIPY[key] = _POOL.submit(oc.assignment, M)
    return _SCIPY[key]


@pytest.fixture(scope="module", autouse=True)
def _start_scipy(request):
    """Start SciPy on every matrix the selected tests of this module compare against, in the order they run."""
    for item in request.session.items:
        params = getattr(item, "callspec", None) and item.callspec.params
        if item.module is request.module and params and "n" in params:
            _scipy(params.get("kind", "gauss"), params["n"])


# ---- device side ------------------------------------------------------------------------------------------------
def _upload(M, ld=None, fill=0.0):
    """M's fp32 bytes on the device in rows of ld floats, the pad columns set to fill, and max M (upload_cost)."""
    n = M.shape[1]
    ld = (n + 3) // 4 * 4 if ld is None else ld
    buf = torch.full((M.shape[0], ld), fill, dtype=torch.float32, device=DEV)
    buf[:, :n] = M.to(DEV)
    return buf, M.max().reshape(1).to(DEV)


def _solve(buf, cmax, n, normalize=0, ws=None, sigma=None):
    """One cfm_assign_exact_f32 call on the current stream: (sigma, total cost, status, milliseconds)."""
    L = _ffi.lib()
    dev = torch.device(DEV)
    if ws is None:
        ws = _ffi.workspace(L.cfm_assign_workspace_bytes(n), dev).zero_()
    if sigma is None:
        sigma = torch.empty(n, dtype=torch.int32, device=DEV)
    total = torch.zeros(1, dtype=torch.float64, device=DEV)
    status = torch.zeros(4, dtype=torch.int32, device=DEV)
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    _ffi.check(L.cfm_assign_exact_f32(_ffi.ptr(buf), n, buf.stride(0), _ffi.ptr(cmax), normalize, _ffi.ptr(sigma),
                                      _ffi.ptr(total), _ffi.ptr(status), _ffi.ptr(ws), ws.numel(),
                                      _ffi.stream_ptr(dev)), "cfm_assign_exact_f32")
    t1.record()
    t1.synchronize()
    return sigma.cpu().numpy(), float(total.item()), status.cpu().tolist()[:3], t0.elapsed_time(t1)


def _record(record_property, n, st, ms):
    record_property("launch", _describe(n))
    record_property("augmentations", st[1])
    record_property("dijkstra_steps", st[2])
    record_property("solve_ms", round(ms, 3))


def _check_optimal(M, sigma, total, st, ref):
    """sigma is SciPy's, a permutation; the total cost is its float64 sum; no flags; a step per augmentation."""
    n = M.shape[0]
    np.testing.assert_array_equal(sigma, ref)
    assert np.array_equal(np.sort(sigma), np.arange(n))
    picked = M.numpy().astype(np.float64)[np.arange(n), ref]
    assert abs(total - picked.sum()) <= 1e-12 * max(1.0, np.abs(picked).sum())
    assert st[0] == 0 and st[2] >= st[1], st


# ---- 1. both sides of every size class ----------------------------------------------------------------------------
@pytest.mark.parametrize("n", BOUNDARY_N, ids=_describe)
def test_size_class_boundary(n, record_property):
    M = _matrix("gauss", n)
    sigma, total, st, ms = _solve(*_upload(M), n)
    _record(record_property, n, st, ms)
    _check_optimal(M, sigma, total, st, _scipy("gauss", n).result())
    assert st[1] == _predicted_augmentations(M), st


# ---- 2. edge inputs, one n per class -------------------------------------------------------------------------------
@pytest.mark.parametrize("n", EDGE_N, ids=_describe)
@pytest.mark.parametrize("kind", ["normalized", "mixed_sign", "integer", "sparse", "nan"])
def test_edge_costs_against_scipy(kind, n, record_property):
    """normalize = 1 (the fp32 quotient M / max M on the device), mixed-sign costs, integer costs in {0..3} (exact
    ties everywhere: only the optimal cost is unique), +inf off two permutations (forbidden edges) and isolated
    NaN entries (never chosen: SciPy gets +inf there)."""
    M = _matrix("gauss" if kind == "normalized" else kind, n)
    sigma, total, st, ms = _solve(*_upload(M), n, normalize=int(kind == "normalized"))
    _record(record_property, n, st, ms)
    ref = _scipy(kind, n).result()
    if kind == "integer":
        assert np.array_equal(np.sort(sigma), np.arange(n))
        Mn = M.numpy().astype(np.float64)
        assert total == Mn[np.arange(n), sigma].sum() == Mn[np.arange(n), ref].sum()  # integer sums are exact
        assert st[0] == 0 and st[2] >= st[1], st
        again = _solve(*_upload(M), n)
        assert np.array_equal(again[0], sigma) and again[1:3] == (total, st)  # ties are broken deterministically
    else:
        _check_optimal(_matrix(kind, n) if kind == "normalized" else M, sigma, total, st, ref)
    if kind in ("normalized", "mixed_sign", "integer"):
        assert st[1] == _predicted_augmentations(M, kind == "normalized"), st


# mixed-sign costs: the same code paths as squared distances, at about a fifteenth of the solve time above n = 4096
@pytest.mark.parametrize("n", EDGE_N, ids=_describe)
@pytest.mark.parametrize("kind", ["mixed_sign"])
def test_padded_leading_dimension(kind, n, record_property):
    """Rows of M in a wider pitch: pad columns of NaN, -inf or -1e30 would win an argmin if any kernel read one."""
    M = _matrix(kind, n)
    want = _solve(*_upload(M), n)
    _record(record_property, n, want[2], want[3])
    _check_optimal(M, *want[:3], _scipy(kind, n).result())
    for fill in (float("nan"), float("-inf"), -1e30):
        got = _solve(*_upload(M, ld=n + 5, fill=fill), n)
        assert np.array_equal(got[0], want[0]) and got[1:3] == want[1:3], fill


@pytest.mark.parametrize("n", EDGE_N, ids=_describe)
@pytest.mark.parametrize("kind", ["mixed_sign"])
def test_stale_workspace_and_sigma(kind, n, record_property):
    """0xFF bytes, or another problem's leftovers, in the workspace and the sigma buffer give the same bits as a zeroed
    workspace.  Above n = 5534 every per-column array of assign_kernel lives in the workspace."""
    L = _ffi.lib()
    M = _matrix(kind, n)
    buf, cmax = _upload(M)
    want = _solve(buf, cmax, n)
    _record(record_property, n, want[2], want[3])
    ws = _ffi.workspace(L.cfm_assign_workspace_bytes(n), torch.device(DEV))
    sigma = torch.empty(n, dtype=torch.int32, device=DEV)
    for history in ("ones", "other"):
        if history == "ones":
            ws.fill_(0xFF)
            sigma.fill_(-1)
        else:
            _solve(*_upload(_matrix("integer", n)), n, ws=ws, sigma=sigma)
        got = _solve(buf, cmax, n, ws=ws, sigma=sigma)
        assert np.array_equal(got[0], want[0]) and got[1:3] == want[1:3], history


@pytest.mark.parametrize("n", EDGE_N, ids=_describe)
@pytest.mark.parametrize("kind", ["mixed_sign"])
def test_infeasible_rows(kind, n, record_property):
    """Rows 0 and 1 can only take column 0: the solve flags the problem infeasible, the sampler raises, and a healthy
    solve that follows on the same stream is still optimal."""
    M = _matrix(kind, n).clone()
    M[:2, 1:] = float("inf")
    buf, cmax = _upload(M)
    _, _, st, ms = _solve(buf, cmax, n)
    _record(record_property, n, st, ms)
    assert st[0] & _ffi.FLAG_INFEASIBLE, st
    s = OTPlanSampler("exact")
    cp = s._solve_exact(buf, cmax, n, n, False)
    with pytest.raises(RuntimeError, match="no finite assignment"):
        s._report(cp)
    M = _matrix(kind, n)
    _check_optimal(M, *_solve(*_upload(M), n)[:3], _scipy(kind, n).result())


# ---- 3. unequal batches: the lcm-replicated problem, ties at every step -------------------------------------------
@pytest.mark.parametrize("n0,n1", [(256, 224), (256, 144), (256, 240), (256, 136), (256, 200), (75, 76)],
                         ids=lambda v: str(v))
def test_unequal_batches_replicated(n0, n1, record_property):
    """A full batch against a short last batch: lcm = 1792, 2304, 3840, 4352 and 6400, one per size class above
    n = 1024, and 75 x 76 (lcm 5700, global memory; 91 x 90 gives the cap's 8190 but takes 25 s per solve).  Every
    cost appears L/n0 * L/n1 times in the replicated matrix."""
    s = OTPlanSampler("exact")
    s.stage_events = []
    _unequal_batch_sizes_vs_lp(s, n0, n1, 8)
    L = int(np.lcm(n0, n1))
    st = [s.last_info["flags"], s.last_info["iterations"], s.last_info["dijkstra_steps"]]
    a, b = next((a, b) for stage, a, b in s.stage_events if stage == "solve")
    b.synchronize()
    _record(record_property, L, st, a.elapsed_time(b))
    assert st[0] == 0 and st[2] >= st[1], st
    M = s._last_bufs["M"][:, :n1].cpu().numpy()  # the device's own cost matrix, replicated as _solve_exact does
    assert st[1] == _predicted_augmentations(np.repeat(np.repeat(M, L // n0, 0), L // n1, 1)), st


# ---- 4. end to end above 4096 -------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,n", [("device", N_E2E)])
def test_end_to_end_device_cost(kind, n, record_property):
    """_couple at d = 8: the device cost kernel, then the global-memory solve, against SciPy on the device's own
    M."""
    g = torch.Generator().manual_seed(n)
    x0, x1 = torch.randn(n, 8, generator=g), torch.randn(n, 8, generator=g) * 1.5 + 0.3
    s = OTPlanSampler("exact")
    s.stage_events = []
    cp = s._couple(x0.to(DEV), x1.to(DEV), torch.device(DEV))
    st = cp.status.cpu().tolist()[:3]
    _, a, b = s.stage_events[-1]
    _record(record_property, n, st, a.elapsed_time(b))
    M = cp.M[:, :n].cpu()
    assert torch.equal(M, _matrix(kind, n))  # the matrix SciPy was started on
    _check_optimal(M, cp.sigma.cpu().numpy(), float(cp.total_cost.item()), st, _scipy(kind, n).result())
    assert st[1] == _predicted_augmentations(M), st
