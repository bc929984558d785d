"""Float64 restatement of the device's log-domain Sinkhorn loop (include/cfm_b200.h §a4; csrc/sinkhorn_common.cuh).

Unlike POT's sinkhorn_log (oracle/ot), which updates v then u in one iteration and checks (u, v) after it, the device
solves v^0 = log b - LSE_i(Mr_ij) first (u = 0), and iteration `it` then computes

    u      = log a - LSE_j(Mr_ij + v_j)
    v_next = log b - LSE_i(Mr_ij + u_i)                     (skipped on a last iteration that is no check)
    err    = || b * expm1(v - v_next) ||_2                  (check iterations: it % check_every == 0)

and stops when err < stop_thr, or (stall_tol > 0) when a check after the first improved err by less than that
fraction while err * sqrt(n1) < 1e-5.  It returns the u of the last iteration and the v that iteration's row pass
used.  Everything runs in torch float64 on the device of Mr, so solves up to 8192 x 8192 stay cheap on a GPU."""
import math

import torch

FLAG_NONFINITE, FLAG_NOT_CONVERGED = 1, 4


def mr_precise(M, reg, cmax=None):
    """-M/reg as the float64-potential bodies form it (NumPy's fp32 rounding): fl32(-fl32(M / cmax) / reg), with
    the division by cmax only when given.  An fp32 quotient formed in float64 and rounded once is the correctly
    rounded fp32 quotient (53 >= 2 * 24 + 2 bits), so no fp32 division is needed."""
    m = M.double()
    if cmax is not None:
        m = (m / float(torch.tensor(cmax, dtype=torch.float32))).float().double()
    return (-(m / float(torch.tensor(reg, dtype=torch.float32)))).float().double()


def mr_exact(M, reg, cmax=None):
    """-M / (reg * cmax) in float64 from the fp32 values of M, reg and cmax (the fp32 bodies' exponent, unrounded)."""
    scale = float(torch.tensor(reg, dtype=torch.float32)) * (
        1.0 if cmax is None else float(torch.tensor(cmax, dtype=torch.float32)))
    return -M.double() / scale


class Result:
    def __init__(self, u, v, iters, err, flags, checks):
        self.u, self.v, self.iters, self.err, self.flags, self.checks = u, v, iters, err, flags, checks

    def __repr__(self):
        return f"Result(iters={self.iters}, err={self.err:.3e}, flags={self.flags}, checks={len(self.checks)})"


def sinkhorn_device_loop(Mr, max_iters, check_every=10, stop_thr=0.0, stall_tol=0.0):
    """The device's loop on float64 Mr (n0 x n1, natural-log units).  Returns a Result: u, v (float64 tensors on
    Mr's device), the iteration count, the last checked err, the status flags and the (iteration, err) pairs of
    every check."""
    assert Mr.dtype == torch.float64 and max_iters >= 1 and check_every >= 1
    n0, n1 = Mr.shape
    loga, logb = -math.log(n0), -math.log(n1)
    v = logb - torch.logsumexp(Mr, dim=0)
    u = torch.zeros(n0, dtype=torch.float64, device=Mr.device)
    err, prev = 1.0, -1.0
    converged = False
    checks = []
    iters = 0
    for it in range(max_iters):
        last, check = it == max_iters - 1, it % check_every == 0
        u = loga - torch.logsumexp(Mr + v[None, :], dim=1)
        iters = it + 1
        if last and not check:
            break
        v_next = logb - torch.logsumexp(Mr + u[:, None], dim=0)
        if check:
            err = float(torch.linalg.vector_norm(torch.expm1(v - v_next) / n1))
            checks.append((it, err))
            if err < stop_thr:
                converged = True
                break
            if stall_tol > 0.0 and prev >= 0.0 and err > (1.0 - stall_tol) * prev and err * math.sqrt(n1) < 1e-5:
                converged = True
                break
            prev = err
        if last:
            break
        v = v_next
    flags = (0 if converged else FLAG_NOT_CONVERGED) | (FLAG_NONFINITE if err != err else 0)
    return Result(u, v, iters, err, flags, checks)
