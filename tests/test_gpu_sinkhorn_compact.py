"""The factored Sinkhorn sweep on the 3-byte fixed-point cost stream (sinkhorn_v2.cu, status[3] = 4).

Every shape here streams (fp32 M larger than 3/4 of the L2), so the path actually runs.  Gates: the generic fp32
kernel on the same M (gauge-fixed potentials within 2e-5, as for the fp32 smem-staged kernel), a float64
kernel-space Sinkhorn-Knopp on the device's own M (marginals 1e-5, plan entries 1e-4 of the largest), and
bit-identical results whatever the workspace held before the solve."""
import numpy as np
import pytest
import torch

from cfm_b200 import _ffi
from cfm_b200.optimal_transport import OTPlanSampler

DEV = "cuda:0"
REG = 0.05


def _cost(n0, n1, d, seed):
    g = torch.Generator().manual_seed(seed)
    x0, x1 = torch.randn(n0, d, generator=g), torch.randn(n1, d, generator=g) + 0.1
    s = OTPlanSampler("sinkhorn", reg=REG, normalize_cost=True, warn=False)
    dev = torch.device(DEV)
    M, cmax, _, _ = s._cost(x0.to(dev), x1.to(dev), dev)
    return M.clone(), cmax.clone()


def _solve(M, cmax, n0, n1, precision, iters, ws=None):
    s = OTPlanSampler("sinkhorn", reg=REG, normalize_cost=True, precision=precision, stall_tol=0.0,
                      num_iter_max=iters, stop_thr=0.0, warn=False)
    bufs = None
    if ws is not None:
        bufs = {"log_u": torch.empty(n0, dtype=torch.float64, device=DEV),
                "log_v": torch.empty(n1, dtype=torch.float64, device=DEV), "ws_sk": ws}
    cp = s._solve_sinkhorn(M, cmax, n0, n1, REG, True, bufs=bufs)
    return cp.log_u.clone(), cp.log_v.clone(), cp.status.cpu().tolist()


@pytest.mark.gpu
@pytest.mark.parametrize("n0,n1,d", [(4096, 4096, 64), (4097, 4100, 32), (3000, 8192, 64), (8192, 2048, 64)])
def test_compact_stream_against_generic_kernel_and_float64_oracle(n0, n1, d):
    M, cmax = _cost(n0, n1, d, n0 + n1)
    lu, lv, st = _solve(M, cmax, n0, n1, "fp32", 100)
    assert st[3] == 4 and st[1] == 100, st  # factored sweep on the 3-byte stream
    lu1, lv1, st1 = _solve(M, cmax, n0, n1, "fp32-generic", 100)
    assert st1[3] == 0 and st1[1] == 100
    lu, lv, lu1, lv1 = (t.cpu().numpy() for t in (lu, lv, lu1, lv1))
    assert np.abs((lu + lv.mean()) - (lu1 + lv1.mean())).max() < 2e-5
    assert np.abs((lv - lv.mean()) - (lv1 - lv1.mean())).max() < 2e-5
    # float64 kernel-space Sinkhorn-Knopp (POT's sinkhorn_knopp) on the device's own normalised fp32 M
    Mn = M[:, :n1] / cmax
    K = torch.exp(Mn.double() / -REG)
    u = torch.full((n0,), 1.0 / n0, dtype=torch.float64, device=DEV)
    for _ in range(100):
        v = (1.0 / n1) / (K.T @ u)
        u = (1.0 / n0) / (K @ v)
    ref_rows, ref_cols = u * (K @ v), v * (K.T @ u)
    P = torch.exp((-(Mn / torch.tensor(REG, dtype=torch.float32, device=DEV))).double()
                  + torch.from_numpy(lu).to(DEV)[:, None] + torch.from_numpy(lv).to(DEV)[None, :])
    assert (P.sum(1) / ref_rows - 1).abs().max().item() <= 1e-5
    assert (P.sum(0) / ref_cols - 1).abs().max().item() <= 1e-5
    sel = torch.from_numpy(np.random.RandomState(0).randint(0, n0, size=64)).to(DEV)
    P_ref = u[sel, None] * K[sel] * v[None, :]
    assert (P[sel] - P_ref).abs().max().item() <= 1e-4 * P_ref.max().item()


@pytest.mark.gpu
def test_compact_stream_ignores_stale_workspace():
    """The ring runs ahead across sweeps: a chunk of the 3-byte copy read before the prologue has written it would
    return whatever the workspace held.  Zeros, ones and another coupling's copy must all give the same bits."""
    n0, n1 = 4096, 4096
    M, cmax = _cost(n0, n1, 64, 1)
    M2, cmax2 = _cost(n0, n1, 64, 2)
    ws = _ffi.workspace(_ffi.lib().cfm_sinkhorn_workspace_bytes(n0, n1), torch.device(DEV))
    for iters in (1, 2, 3, 11, 100):
        got = []
        for history in ("zeros", "ones", "other"):
            if history == "zeros":
                ws.fill_(0x00)
            elif history == "ones":
                ws.fill_(0xFF)
            else:
                _, _, st2 = _solve(M2, cmax2, n0, n1, "fp32", 100, ws)
                assert st2[3] == 4
            lu, lv, st = _solve(M, cmax, n0, n1, "fp32", iters, ws)
            assert st[3] == 4 and st[1] == iters
            got.append((lu.cpu().numpy(), lv.cpu().numpy()))
        for lu, lv in got[1:]:
            assert np.array_equal(lu, got[0][0]) and np.array_equal(lv, got[0][1]), iters
