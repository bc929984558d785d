"""The Sinkhorn pair draw (`sample.cu`), draw by draw, against a float64 inverse-cdf oracle on every path it takes.

The reference draws with ``np.random.choice(n0 * n1, p=plan.flatten() / plan.sum())``: the flat cdf
``C = cumsum(p) / cumsum(p)[-1]``, ``k = searchsorted(C, u, 'right')``, ``(i, j) = divmod(k, n1)``.  The oracle forms
the plan in float64 from the device's own M, cost_max, log_u and log_v with NumPy's fp32 roundings of the quotients
(``-(fl32(fl32(M / cmax) / reg))``, then a float64 ``+ lu_i + lv_j`` and ``exp``), and the flat cdf from the row-mass cdf
``R`` and the row cdfs ``P_i``: ``C[(i, j)] = (R_i + P_i[j]) / T``, ``T = R_n0``.  ``test_oracle_reproduces_random_choice``
shows that this form is ``np.random.choice`` index for index.

Every draw ``k = (i, j)`` must satisfy
  (a) the bracket  ``C[k-1] - delta <= u < C[k] + delta``, with delta derived below from the kernel's arithmetic, and
  (b) the mass floor: the drawn cell's float64 plan entry is in fp32's normal range, >= 2^-126 (1.18e-38) less the
      weight's rounding.  ``ex2.approx.ftz`` makes a weight below it 0, so a correct crossing never selects it; cells
      of 1.2e-38 to 1e-37 are legitimate draws (the first cell of positive weight when frac = 0).
A draw whose uniform lies farther than delta from both boundaries of its oracle cell is then the oracle's draw exactly.

delta.  Let eta bound the relative error of one kernel weight against the oracle's entry (below).  The fast draw
(``uniform_rows = 1``) takes row ``i = floor(u n0)`` and inverts ``t = frac / n0`` (the row mass it assumes) or
``frac * S`` (the weights' measured sum S, when the walk runs off the row's end) along row i.  Every partial sum of the
weights is within ``eta r_i`` of the oracle's ``P_i``, and the oracle's row boundaries lie ``D_i = |i / n0 - R_i / T|``
from the kernel's, so
    delta_i = D_i + r_i |1 - 1/T| + |r_i - 1/n0| + 2 eta r_i      (flat-cdf units).
D_i and |r_i - 1/n0| are the solver's row-marginal error, which the draw trusts; the test reports their maximum e_r.
The generic draw (``uniform_rows = 0``) totals rows and the plan with the same weights: delta = 2 eta (flat units).
A row-conditional draw inverts against its measured row sum: delta = 2 eta of the row's mass.

eta.  A weight is ``2^x`` with x its log2.  Entries below 2^-64 carry less than n1 2^-64 of any row (< 1e-10 of its
mass here); the others have |x| <= 64.  fp32 rounding of x costs ``ln2 |dx|`` relative, ``ex2.approx.ftz.f32`` 2^-22
and the fp32 sum of a float4 group 2^-23:
  * precise (|M/reg| > 64): x is the float64 exponent of the oracle rounded once to fp32:
        eta = ln2 2^-24 64 + 2^-22 + 2^-23                                    = 3.0e-6
  * fast (|M/reg| <= 64): ``x = fma(M, c2, fl(lv_j log2e) + fl(lu_i log2e))``, c2 = fl(-log2e / fl(reg scale)) three
    roundings off; the oracle's quotient is two roundings off the exact one:
        eta = ln2 2^-24 (5 A + 2 Lv + 2 Lu + 64) + 2^-22 + 2^-23,   A = max|M c2|, Lv = max|lv log2e|, Lu = max|lu log2e|
    (~2e-5 at the shapes below; a row-maximum shift replaces Lu by A + Lv);
  * generic ``draw_kernel<PotEntry>``: ``expf`` of the float64 exponent rounded to fp32 (|e| <= 44.4 for entries
    above 2^-64):  eta = 2^-24 44.4 + 2^-23 = 2.8e-6.
"""
import math
import types

import numpy as np
import pytest
import torch

from cfm_b200 import _ffi
from cfm_b200.optimal_transport import OTPlanSampler

DEV = "cuda:0"
LOG2E = 1.4426950408889634
LN2 = math.log(2.0)
U24 = 2.0 ** -24
EX2 = 2.0 ** -22
GROUP = 2.0 ** -23
FLOOR = 2.0 ** -126 * (1.0 - 1e-4)
ETA_PRECISE = LN2 * U24 * 64 + EX2 + GROUP
ETA_GENERIC = U24 * 44.4 + GROUP
TAIL = 1e-10  # entries below 2^-64, relative to a row's mass


# ----------------------------------------------------------------------------------------------- the oracle (NumPy)
def flat_pick(p, u):
    """np.random.choice's own inversion (numpy/random/mtrand.pyx, legacy ``choice`` with ``p``)."""
    q = p.flatten()
    q = q / q.sum()
    cdf = np.cumsum(q)
    cdf /= cdf[-1]
    return np.divmod(cdf.searchsorted(u, side="right"), p.shape[1])


def hier_pick(rowmass, row_cdf, u):
    """The same inversion from the row-mass cdf and one row's cdf: ``rowmass`` (n0,) float64, ``row_cdf(i)`` the
    cumulative sums of row i.  Returns (i, j); a target past a row's rounded end takes its last cell of positive mass."""
    R = np.concatenate([[0.0], np.cumsum(rowmass)])
    T = R[-1]
    i = np.minimum(np.searchsorted(R[1:] / T, u, side="right"), len(rowmass) - 1)
    j = np.empty_like(i)
    for k in range(len(u)):
        P = row_cdf(int(i[k]))
        jj = int(np.searchsorted((R[i[k]] + P) / T, u[k], side="right"))
        if jj >= len(P):
            jj = int(np.flatnonzero(np.diff(np.concatenate([[0.0], P])) > 0)[-1])
        j[k] = jj
    return i, j


def test_oracle_reproduces_random_choice():
    """The hierarchical oracle is np.random.choice index for index, on plans with zero entries and zero rows too."""
    rs = np.random.RandomState(5)
    for n0, n1, zeros in ((1, 1, 0.0), (1, 7, 0.3), (5, 1, 0.0), (7, 9, 0.0), (13, 6, 0.5), (40, 33, 0.8), (64, 130, 0.2)):
        p = rs.random_sample((n0, n1)) ** 3
        p[rs.random_sample((n0, n1)) < zeros] = 0.0
        if n0 > 3:
            p[2] = 0.0
        if p.sum() == 0.0:
            p[0, -1] = 1.0
        seed = n0 * 100 + n1
        want = np.divmod(np.random.RandomState(seed).choice(p.size, p=p.flatten() / p.sum(), size=5000), n1)
        u = np.random.RandomState(seed).random_sample(5000)
        u = np.concatenate([u, [0.0, np.nextafter(1.0, 0.0)]])
        fi, fj = flat_pick(p, u)
        np.testing.assert_array_equal(fi[:5000], want[0])
        np.testing.assert_array_equal(fj[:5000], want[1])
        hi, hj = hier_pick(p.sum(1), lambda i: np.cumsum(p[i]), u)
        np.testing.assert_array_equal(hi, fi)
        np.testing.assert_array_equal(hj, fj)
        assert np.all(p[hi, hj] > 0.0)


# ----------------------------------------------------------------------------------------------- the oracle (device)
class Plan:
    """float64 plan of a Sinkhorn coupling from the device's own M, cost_max, log_u, log_v (NumPy's fp32 roundings)."""

    def __init__(self, cp):
        self.n0, self.n1 = cp.n0, cp.n1
        self.M, self.cmax, self.normalize = cp.M[:, :cp.n1], cp.cost_max, cp.normalize
        self.reg32 = torch.tensor(np.float32(cp.reg), device=cp.M.device)
        self.lu, self.lv = cp.log_u, cp.log_v
        self.r = torch.cat([self.rows(torch.arange(a, min(a + 1024, self.n0), device=cp.M.device)).sum(1)
                            for a in range(0, self.n0, 1024)]).cpu().numpy()
        self.R = np.concatenate([[0.0], np.cumsum(self.r)])
        self.T = self.R[-1]
        self.e_r = float(np.abs(self.r * self.n0 - 1.0).max())

    def rows(self, idx, lu=True):
        m = self.M[idx]
        if self.normalize:
            m = m / self.cmax  # IEEE fp32 division, __fdiv_rn's rounding
        q = -(m / self.reg32)
        e = q.double() + self.lu[idx, None] if lu else q.double()
        return torch.exp(e + self.lv[None, :])  # the kernel's order of the float64 adds

    def eta_fast(self, row_max_shift=False):
        scale = float(self.cmax.item()) if self.normalize else 1.0
        A = float(self.M.max().item()) / (scale * float(self.reg32.item())) * LOG2E
        Lv = float(self.lv.abs().max().item()) * LOG2E
        Lu = A + Lv if row_max_shift else float(self.lu.abs().max().item()) * LOG2E
        return LN2 * U24 * (5 * A + 2 * Lv + 2 * Lu + 64) + EX2 + GROUP

    def is_precise(self):
        cmax = np.float32(self.cmax.item())
        ratio = np.float32(np.float32(1.0) if self.normalize else cmax) / np.float32(self.reg32.item())
        return not ratio <= np.float32(64.0)

    def delta_rows(self):
        n0, i = self.n0, np.arange(self.n0)
        D = np.abs(i / n0 - self.R[:-1] / self.T)
        return D + self.r * abs(1.0 - 1.0 / self.T) + np.abs(self.r - 1.0 / n0)

    def cell_bounds(self, i, j, chunk=2048):
        """(C[k-1], C[k], p_k) of the drawn cells k = (i, j), in flat-cdf units."""
        lo, hi, pk = (np.empty(len(i)) for _ in range(3))
        it, jt = torch.from_numpy(i).to(DEV), torch.from_numpy(j).to(DEV)
        for a in range(0, len(i), chunk):
            b = min(a + chunk, len(i))
            p = self.rows(it[a:b])
            P = torch.cumsum(p, 1)
            jj = jt[a:b, None]
            Pj = P.gather(1, jj)[:, 0]
            pj = p.gather(1, jj)[:, 0]
            hi[a:b] = Pj.cpu().numpy()
            lo[a:b] = (Pj - pj).cpu().numpy()
            pk[a:b] = pj.cpu().numpy()
        return (self.R[i] + lo) / self.T, (self.R[i] + hi) / self.T, pk

    def row_cdf(self, i):
        return torch.cumsum(self.rows(torch.tensor([i], device=DEV))[0], 0).cpu().numpy()


def sinkhorn(n0, n1, d, ratio, normalize, precision="auto", iters=200, seed=0):
    """A Sinkhorn coupling with max(M)/reg (or 1/reg when normalised) close to ``ratio``."""
    g = torch.Generator().manual_seed(seed + 7 * n1 + n0)
    x0, x1 = torch.randn(n0, d, generator=g), torch.randn(n1, d, generator=g) + 0.3
    reg = 1.0 / ratio if normalize else float(torch.cdist(x0, x1).pow(2).max()) / ratio
    s = OTPlanSampler("sinkhorn", reg=reg, normalize_cost=normalize, num_iter_max=iters, stop_thr=0.0, warn=False,
                      precision=precision)
    cp = s._couple(x0.to(DEV), x1.to(DEV), torch.device(DEV))
    return s, cp


def adversarial_rows(n0):
    """frac = 0, 2^-40 and 1 - 2^-40 in every row (floor(u n0) == i), and u = nextafter(1, 0)."""
    i = np.arange(n0, dtype=np.float64)
    out = [i / n0]
    lo = (i + 2.0 ** -40) / n0
    hi = (i + 1.0 - 2.0 ** -40) / n0
    for _ in range(4):
        lo = np.where(np.floor(lo * n0) < i, np.nextafter(lo, 1.0), lo)
        hi = np.where(np.floor(hi * n0) > i, np.nextafter(hi, 0.0), hi)
    assert np.all(np.floor(lo * n0) == i) and np.all(np.floor(hi * n0) == i)
    return np.concatenate(out + [lo, hi, [np.nextafter(1.0, 0.0)]])


def boundary_uniforms(plan, delta, rows):
    """u = C[(i, jb)] +- 10 delta_i at the float4-group edges and where the 1024-column blocks meet; returns (u,
    oracle i, oracle j) for those whose row is floor(u n0) both for the kernel and the oracle."""
    n0, n1 = plan.n0, plan.n1
    cols = [c for c in (0, 3, 7, 127, 1023, 2047, n1 // 2) if c < n1 - 1]
    us, want_i, want_j = [], [], []
    for i in rows:
        P = plan.row_cdf(i)
        C = (plan.R[i] + P) / plan.T
        for c in cols:
            for sgn in (-10.0, 10.0):
                u = C[c] + sgn * delta[i]
                if not (plan.R[i] / plan.T <= u < plan.R[i + 1] / plan.T and int(u * n0) == i):
                    continue
                j = min(int(np.searchsorted(C, u, side="right")), n1 - 1)
                lo = C[j - 1] if j > 0 else plan.R[i] / plan.T
                if u - lo < delta[i] or C[j] - u <= delta[i]:
                    continue  # cells narrower than 10 delta: u lands near another boundary
                us.append(u), want_i.append(i), want_j.append(j)
    return np.array(us), np.array(want_i, dtype=np.int64), np.array(want_j, dtype=np.int64)


def gate(plan, u, i, j, delta, record_property, tag=""):
    """(a) bracket and (b) mass floor for every draw; returns the number of draws within delta of a boundary."""
    lo, hi, pk = plan.cell_bounds(i, j)
    bad = ~((lo - delta <= u) & (u < hi + delta))
    assert not bad.any(), (tag, int(bad.sum()), u[bad][:4], i[bad][:4], j[bad][:4], lo[bad][:4], hi[bad][:4],
                           delta[bad][:4] if np.ndim(delta) else delta)
    light = pk < FLOOR
    assert not light.any(), (tag, int(light.sum()), i[light][:4], j[light][:4], pk[light][:4], u[light][:4])
    near = int(((u < lo + delta) | (u >= hi - delta)).sum())
    record_property(f"near_boundary{tag}", near)
    return near


def fast_draw(s, cp, u):
    i, j = s._draw(cp, len(u), torch.from_numpy(np.ascontiguousarray(u)).to(DEV))
    return i.cpu().numpy(), j.cpu().numpy()


def check_uniform_rows(s, cp, record_property, n_seeded, boundary_rows=3, seed=1):
    plan = Plan(cp)
    precise = plan.is_precise()
    eta = ETA_PRECISE if precise else plan.eta_fast()
    delta = plan.delta_rows() + (2 * eta + TAIL) * plan.r + 1e-15
    n0 = plan.n0
    u_seed = np.random.RandomState(seed).random_sample(n_seeded)
    ub, bi, bj = boundary_uniforms(plan, delta, sorted({0, n0 // 2, n0 - 1})[:boundary_rows])
    u = np.concatenate([u_seed, adversarial_rows(n0), ub])
    i, j = fast_draw(s, cp, u)
    st = cp.status.cpu().tolist()
    assert st[0] & _ffi.FLAG_NONFINITE == 0, st
    np.testing.assert_array_equal(i, np.minimum((u * n0).astype(np.int64), n0 - 1))
    near = gate(plan, u, i, j, delta[i], record_property)
    nb = len(ub)
    if nb:
        np.testing.assert_array_equal(i[-nb:], bi)
        np.testing.assert_array_equal(j[-nb:], bj)
    for k, v in (("precise", precise), ("vec", plan.n1 % 4 == 0), ("eta", eta), ("e_r", plan.e_r),
                 ("delta_max_rows", float(delta.max() * n0)), ("boundary_draws", nb), ("status", st)):
        record_property(k, v)
    return plan, precise, near


gpu = pytest.mark.gpu

N1S = [1, 3, 4, 31, 130, 1023, 1024, 1025, 2053, 8192, 12288]


# ----------------------------------------------------------------------------------------------- uniform_rows = 1
@gpu
@pytest.mark.parametrize("n1", N1S)
@pytest.mark.parametrize("precise,normalize", [(False, False), (False, True), (True, False), (True, True)])
def test_uniform_rows_draw(n1, precise, normalize, record_property):
    """cfm_plan_sample with uniform_rows = 1 (sample_plan / sample_pairs): fp32-exponent and precise weights, float4
    and scalar rows, one to twelve 1024-column blocks; the 12288-column solve runs on the generic column-panel kernel."""
    n0 = 96
    s, cp = sinkhorn(n0, n1, 6, 300.0 if precise else 20.0, normalize, iters=150)
    plan, got_precise, _ = check_uniform_rows(s, cp, record_property, 2048)
    assert got_precise == precise
    assert plan.e_r <= 4 * (ETA_PRECISE if precise else plan.eta_fast()), plan.e_r


@gpu
def test_peaked_precise_plan_last_column(record_property):
    """n = 512, d = 2, reg = 0.02: rows whose last columns carry e^-hundreds.  frac = 1 - 2^-40 past a row's fp32
    weight sum must land on the row's last column of positive weight, never on a column the plan gives no mass."""
    g = torch.Generator().manual_seed(4)
    x0, x1 = torch.randn(512, 2, generator=g), torch.randn(512, 2, generator=g)
    s = OTPlanSampler("sinkhorn", reg=0.02, num_iter_max=300, stop_thr=0.0, warn=False)
    cp = s._couple(x0.to(DEV), x1.to(DEV), torch.device(DEV))
    plan, precise, _ = check_uniform_rows(s, cp, record_property, 4096)
    assert precise


@gpu
@pytest.mark.parametrize("batch", [17, 300, 5000])
def test_sample_pairs_batch_size(batch, record_property):
    """sample_pairs(batch_size=...) with fewer and more draws than rows, from the global NumPy stream."""
    g = torch.Generator().manual_seed(batch)
    x0, x1 = torch.randn(256, 8, generator=g), torch.randn(260, 8, generator=g)
    s = OTPlanSampler("sinkhorn", reg=0.05, normalize_cost=True, num_iter_max=100, stop_thr=0.0, warn=False)
    np.random.seed(batch)
    i, j = s.sample_pairs(x0.to(DEV), x1.to(DEV), batch_size=batch)
    np.random.seed(batch)
    u = np.random.random_sample(batch)
    B = s._last_bufs  # the coupling the call drew from: the sampler's per-shape buffers
    plan = Plan(types.SimpleNamespace(n0=256, n1=260, M=B["M"], cost_max=B["cmax"], log_u=B["log_u"],
                                      log_v=B["log_v"], reg=0.05, normalize=True))
    assert not plan.is_precise()
    delta = plan.delta_rows() + (2 * plan.eta_fast() + TAIL) * plan.r
    i, j = i.cpu().numpy(), j.cpu().numpy()
    assert len(i) == batch
    np.testing.assert_array_equal(i, np.minimum((u * 256).astype(np.int64), 255))
    gate(plan, u, i, j, delta[i], record_property)


# ----------------------------------------------------------------------------------------------- row-conditional
@gpu
@pytest.mark.parametrize("precise", [False, True])
@pytest.mark.parametrize("with_log_u", [True, False])
@pytest.mark.parametrize("n1", [130, 1024, 2053])
def test_row_conditional_draw(precise, with_log_u, n1, record_property):
    """cfm_plan_sample_rows (sample_trajectory): with log_u, and with log_u = NULL (row-maximum pass, measured
    total).  Gate on the row's own cdf, delta = 2 eta of the row's mass."""
    n0 = 200
    s, cp = sinkhorn(n0, n1, 5, 300.0 if precise else 20.0, False, iters=150, seed=3)
    plan = Plan(cp)
    assert plan.is_precise() == precise
    eta = ETA_PRECISE if precise else plan.eta_fast(row_max_shift=not with_log_u)
    rs = np.random.RandomState(n1)
    rows = rs.randint(0, n0, 3000)
    u = rs.random_sample(3000)
    rows = np.concatenate([rows, np.arange(n0), np.arange(n0), np.arange(n0), [n0 - 1]])
    u = np.concatenate([u, np.zeros(n0), np.full(n0, 2.0 ** -40), np.full(n0, 1.0 - 2.0 ** -40),
                        [np.nextafter(1.0, 0.0)]])
    rd, ud = torch.from_numpy(rows).to(DEV), torch.from_numpy(u).to(DEV)
    if with_log_u:
        j = s._draw_rows(cp, rd, ud)
    else:
        j = torch.empty(len(u), dtype=torch.int64, device=DEV)
        _ffi.check(_ffi.lib().cfm_plan_sample_rows(
            _ffi.ptr(cp.M), n0, n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max), 0, None, _ffi.ptr(cp.log_v),
            _ffi.ptr(rd), _ffi.ptr(ud), len(u), _ffi.ptr(j), _ffi.ptr(cp.status), _ffi.stream_ptr(torch.device(DEV))),
            "cfm_plan_sample_rows")
    assert cp.status.cpu()[0].item() & _ffi.FLAG_NONFINITE == 0
    j = j.cpu().numpy()
    p = plan.rows(rd)
    P = torch.cumsum(p, 1)
    tot = P[:, -1]
    jt = torch.from_numpy(j).to(DEV)[:, None]
    hi = (P.gather(1, jt)[:, 0] / tot).cpu().numpy()
    pk = p.gather(1, jt)[:, 0]
    lo = hi - (pk / tot).cpu().numpy()
    if not with_log_u:  # the kernel's weights are then pi_ij / max_j pi_ij: the floor applies on that scale
        pk = pk / p.max(1).values
    pk = pk.cpu().numpy()
    delta = 2 * eta + TAIL
    bad = ~((lo - delta <= u) & (u < hi + delta))
    assert not bad.any(), (int(bad.sum()), rows[bad][:4], u[bad][:4], j[bad][:4], lo[bad][:4], hi[bad][:4])
    light = pk < FLOOR
    assert not light.any(), (rows[light][:4], j[light][:4], u[light][:4],
                             p[torch.from_numpy(light).to(DEV)][:2, :4].cpu().numpy())
    record_property("near_boundary", int(((u < lo + delta) | (u >= hi - delta)).sum()))
    record_property("eta", eta)


# ----------------------------------------------------------------------------------------------- uniform_rows = 0
@gpu
@pytest.mark.parametrize("n0", [1, 1023, 1024, 1025, 3000])
def test_generic_draw_kernel(n0, record_property):
    """draw_kernel<PotEntry> (uniform_rows = 0, public C ABI): row_mass_kernel, row_cdf_kernel with one and with
    several rows per thread (n0 > 1024), and the row walk; flat gate, delta = 2 eta_generic."""
    n1 = 40
    s, cp = sinkhorn(n0, n1, 4, 300.0, False, iters=150, seed=5)
    plan = Plan(cp)
    L = _ffi.lib()
    rs = np.random.RandomState(n0)
    u = np.concatenate([rs.random_sample(4096), plan.R[:-1] / plan.T, [0.0, 2.0 ** -40, np.nextafter(1.0, 0.0)]])
    nd = len(u)
    ud = torch.from_numpy(u).to(DEV)
    i = torch.empty(nd, dtype=torch.int64, device=DEV)
    j = torch.empty_like(i)
    st = torch.zeros(4, dtype=torch.int32, device=DEV)
    ws = _ffi.workspace(L.cfm_plan_sample_workspace_bytes(n0), torch.device(DEV))
    _ffi.check(L.cfm_plan_sample(_ffi.ptr(cp.M), n0, n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max), 0,
                                 _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), 0, _ffi.ptr(ud), nd, _ffi.ptr(i), _ffi.ptr(j),
                                 _ffi.ptr(st), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr()), "cfm_plan_sample")
    assert st.cpu().tolist()[0] == 0
    delta = np.full(nd, 2 * ETA_GENERIC + TAIL)
    gate(plan, u, i.cpu().numpy(), j.cpu().numpy(), delta, record_property)
    record_property("rows_per_thread", (n0 + 1023) // 1024)


# ----------------------------------------------------------------------------------------------- dense draw
@gpu
def test_dense_draw_rectangular_exact_ot_is_random_choice():
    """Rectangular exact OT (1024 x 1536, lcm 3072): sample_plan draws from the 1.5M-entry float64 plan on the device
    (cfm_dense_plan_sample_f64), index for index what np.random.choice draws from the same plan and seed."""
    g = torch.Generator().manual_seed(8)
    x0, x1 = torch.randn(1024, 3, generator=g), torch.randn(1536, 3, generator=g)
    x0[:, 0] = torch.arange(1024, dtype=torch.float32)  # distinct rows: x[i] identifies i
    x1[:, 0] = torch.arange(1536, dtype=torch.float32) * 0.5
    s = OTPlanSampler("exact")
    pi = s.get_map(x0.to(DEV), x1.to(DEV))
    assert pi.size >= 1 << 20 and np.count_nonzero(pi) <= 1024 + 1536
    np.random.seed(21)
    a, b = s.sample_plan(x0.to(DEV), x1.to(DEV))
    np.random.seed(21)
    wi, wj = np.divmod(np.random.choice(pi.size, p=pi.flatten() / pi.sum(), size=1024), pi.shape[1])
    assert torch.equal(a.cpu(), x0[wi]) and torch.equal(b.cpu(), x1[wj])
    np.random.seed(22)
    i, j = s.sample_map(pi, 50000)
    np.random.seed(22)
    wi, wj = np.divmod(np.random.choice(pi.size, p=pi.flatten() / pi.sum(), size=50000), pi.shape[1])
    np.testing.assert_array_equal(i, wi)
    np.testing.assert_array_equal(j, wj)


@gpu
def test_dense_draw_sinkhorn_plan(record_property):
    """A float64 Sinkhorn plan from get_map with n0 = 1100 > 1024 rows: sample_map on the device equals
    np.random.choice except where the uniform lies within 1e-12 of a cdf boundary."""
    g = torch.Generator().manual_seed(9)
    x0, x1 = torch.randn(1100, 5, generator=g), torch.randn(1000, 5, generator=g)
    s = OTPlanSampler("sinkhorn", reg=0.05, normalize_cost=True, num_iter_max=100, stop_thr=0.0, warn=False)
    pi = s.get_map(x0.to(DEV), x1.to(DEV))
    assert pi.size >= 1 << 20
    nd = 50000
    np.random.seed(23)
    i, j = s.sample_map(pi, nd)
    np.random.seed(23)
    u = np.random.random_sample(nd)
    wi, wj = flat_pick(pi, u)
    q = pi.flatten() / pi.sum()
    cdf = np.cumsum(q)
    cdf /= cdf[-1]
    k = wi * pi.shape[1] + wj
    lo = np.where(k > 0, cdf[np.maximum(k - 1, 0)], 0.0)
    near = (u - lo < 1e-12) | (cdf[k] - u <= 1e-12)
    diff = (i != wi) | (j != wj)
    assert not (diff & ~near).any(), np.flatnonzero(diff & ~near)[:5]
    record_property("near_boundary", int(near.sum()))
    record_property("differ", int(diff.sum()))
    assert diff.sum() <= near.sum() <= 3


# ----------------------------------------------------------------------------------------------- production shapes
@gpu
@pytest.mark.parametrize("case", ["C2", "C4_shard"])
def test_production_shape(case, record_property):
    """C2: 8192^2, d = 784, reg 0.05, normalised, 100 iterations on the 3-byte stream (status[3] == 4), fp32 weights.
    A C4 shard: 4096^2, d = 512, reg 0.1, not normalised, seeded mixed solver (status[3] == 1), precise weights.
    Every draw of a full batch plus the adversarial set is gated."""
    n, d, reg, normalize, variant = {"C2": (8192, 784, 0.05, True, 4), "C4_shard": (4096, 512, 0.1, False, 1)}[case]
    g = torch.Generator().manual_seed(n + d)
    x0, x1 = torch.randn(n, d, generator=g), torch.randn(n, d, generator=g)
    s = OTPlanSampler("sinkhorn", reg=reg, normalize_cost=normalize, num_iter_max=100, stop_thr=0.0, warn=False)
    cp = s._couple(x0.to(DEV), x1.to(DEV), torch.device(DEV))
    assert cp.status.cpu().tolist()[3] == variant, cp.status.cpu().tolist()
    plan, precise, near = check_uniform_rows(s, cp, record_property, n, seed=n)
    assert precise == (case == "C4_shard")


@gpu
def test_forced_fp32_at_large_cost_over_reg(record_property):
    """precision="fp32" at |M/reg| ~ 200: the solver's fp32 exponents leave row masses away from 1/n0 in the precise
    weights' float64 arithmetic, so the draw totals the row (status[2] == 0).  delta carries the measured e_r."""
    s, cp = sinkhorn(256, 300, 8, 200.0, False, precision="fp32", iters=200, seed=11)
    assert cp.status.cpu().tolist()[2] == 0
    plan, precise, _ = check_uniform_rows(s, cp, record_property, 4096)
    assert precise
