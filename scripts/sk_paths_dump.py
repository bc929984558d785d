"""One Sinkhorn solve on every solver path (status[3] says which kernel body ran) and at the loop's edges: saves
log_u, log_v, status and err of each case to an .npz, so that two checkouts can be compared bit for bit (err, an
atomicAdd sum over the CTAs, only to its last bits).

    python scripts/sk_paths_dump.py --root OLD --out old.npz
    python scripts/sk_paths_dump.py --root NEW --out new.npz --compare old.npz

Cost matrices come from the SIMT fp32 cost kernel (cost_algo=1) or from the host, so both runs solve the same M; a
fingerprint of each M is saved and compared too."""
import argparse
import os
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
ap.add_argument("--out", required=True)
ap.add_argument("--compare", default=None, help="an earlier --out file: report every array that differs")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import cfm_b200  # noqa: E402
from cfm_b200 import _ffi  # noqa: E402

DEV = torch.device("cuda:0")
PREC = {"auto": -1, "fp32": 0, "fp64": 1, "fp32-generic": 2, "fp64-mixed": 3, "fp64-mixed-unscreened": 4}


def cost_from_points(n0, n1, d, seed):
    g = torch.Generator().manual_seed(seed)
    x0, x1 = torch.randn(n0, d, generator=g), torch.randn(n1, d, generator=g)
    s = cfm_b200.OTPlanSampler("sinkhorn", cost_algo=1, warn=False)
    M, cmax, _, _ = s._cost(x0.to(DEV), x1.to(DEV), DEV)
    return M.clone(), cmax.clone()


def cost_from_host(M):
    n0, n1 = M.shape
    buf = torch.zeros((n0, (n1 + 3) // 4 * 4), dtype=torch.float32, device=DEV)
    buf[:, :n1] = M.to(DEV)
    return buf, M.max().reshape(1).float().to(DEV)


def rand_cost(n0, n1, seed, scale, offset):
    g = torch.Generator().manual_seed(seed)
    return cost_from_host(torch.rand(n0, n1, generator=g) * scale + offset)


def solve(M, cmax, n1, reg, normalize, precision, iters, stop_thr=0.0, check_every=10, stall_tol=0.0):
    L = _ffi.lib()
    n0 = M.shape[0]
    lu = torch.empty(n0, dtype=torch.float64, device=DEV)
    lv = torch.empty(n1, dtype=torch.float64, device=DEV)
    st = torch.zeros(4, dtype=torch.int32, device=DEV)
    err = torch.zeros(1, dtype=torch.float64, device=DEV)
    ws = torch.zeros(L.cfm_sinkhorn_workspace_bytes(n0, n1), dtype=torch.uint8, device=DEV)
    _ffi.check(L.cfm_sinkhorn_log_f32(
        _ffi.ptr(M), n0, n1, M.stride(0), float(reg), _ffi.ptr(cmax), int(normalize), iters, float(stop_thr),
        check_every, PREC[precision], float(stall_tol), _ffi.ptr(lu), _ffi.ptr(lv), _ffi.ptr(st), _ffi.ptr(err),
        _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(DEV)), "cfm_sinkhorn_log_f32")
    torch.cuda.synchronize()
    return lu.cpu().numpy(), lv.cpu().numpy(), st.cpu().numpy(), err.cpu().numpy()


def cases():
    """(name, M, cmax, n1, solve keyword arguments)"""
    M, c = cost_from_points(1024, 1024, 64, 1)
    yield "v2_factored_1024", M, c, 1024, dict(reg=0.05, normalize=True, precision="auto", iters=100)
    yield "generic_fp32_forced_1024", M, c, 1024, dict(reg=0.05, normalize=True, precision="fp32-generic", iters=100)
    yield "fp64_1024", M, c, 1024, dict(reg=0.05, normalize=True, precision="fp64", iters=30)
    for pr in ("auto", "fp32-generic"):  # the last iteration is no check / is a check
        yield f"edge_{pr}_23_every_7", M, c, 1024, dict(reg=0.05, normalize=True, precision=pr, iters=23, check_every=7)
        yield f"edge_{pr}_22_every_7", M, c, 1024, dict(reg=0.05, normalize=True, precision=pr, iters=22, check_every=7)
    M, c = cost_from_points(8192, 8192, 784, 2)
    yield "v2_3byte_c2", M, c, 8192, dict(reg=0.05, normalize=True, precision="auto", iters=100)
    M, c = cost_from_points(4096, 4096, 512, 3)
    yield "v2_3byte_4096", M, c, 4096, dict(reg=0.05, normalize=True, precision="auto", iters=100)
    yield "seeded_c4_shard", M, c, 4096, dict(reg=0.1, normalize=False, precision="auto", iters=100)
    yield "seeded_stop_thr", M, c, 4096, dict(reg=0.1, normalize=False, precision="auto", iters=1000, stop_thr=1e-2)
    yield "seeded_23_every_7", M, c, 4096, dict(reg=0.1, normalize=False, precision="auto", iters=23, check_every=7)
    yield "unscreened_mixed_4096", M, c, 4096, dict(reg=0.1, normalize=False, precision="fp64-mixed-unscreened",
                                                    iters=20)
    g = torch.Generator().manual_seed(8)
    M, c = cost_from_host(torch.rand(256, 256, generator=g) * 0.5 + 0.5)
    yield "v2_log_domain", M, c, 256, dict(reg=0.03, normalize=False, precision="fp32", iters=60)
    M, c = cost_from_points(1000, 1001, 64, 4)
    yield "generic_fp32_1000x1001", M, c, 1001, dict(reg=0.05, normalize=True, precision="auto", iters=100)
    M, c = cost_from_points(200, 16384, 64, 5)
    yield "generic_fp32_200x16384", M, c, 16384, dict(reg=0.05, normalize=True, precision="auto", iters=100)
    M, c = rand_cost(64, 14000, 14000, 40.0, 5.0)
    yield "mixed_v_not_staged_64x14000", M, c, 14000, dict(reg=0.05, normalize=False, precision="auto", iters=12)
    for n0, n1 in ((64, 9000), (40, 12288)):
        M, c = rand_cost(n0, n1, n1, 40.0, 5.0)
        yield f"screened_mixed_{n0}x{n1}", M, c, n1, dict(reg=0.05, normalize=False, precision="auto", iters=12)
    M, c = cost_from_points(1024, 1024, 64, 1)
    for pr in ("auto", "fp32-generic"):
        yield f"stop_thr_{pr}", M, c, 1024, dict(reg=0.05, normalize=True, precision=pr, iters=1000, stop_thr=1e-6)
        yield f"stall_tol_{pr}", M, c, 1024, dict(reg=0.05, normalize=True, precision=pr, iters=1000, stop_thr=1e-14,
                                                  stall_tol=0.1)
    M, c = cost_from_points(512, 512, 16, 6)
    for reg in (0.012, 0.015):  # normalised, just past the fp32 regime: the seeded solver reaches its error floor
        yield f"seeded_stall_tol_reg{reg}", M, c, 512, dict(reg=reg, normalize=True, precision="auto", iters=2000,
                                                             stop_thr=1e-14, stall_tol=0.1)
    M[3, 7] = float("nan")
    for name, reg, pr in (("v2", 0.05, "fp32"), ("generic", 0.05, "fp32-generic"), ("fp64", 0.05, "fp64"),
                          ("seeded", 0.01, "auto")):
        yield f"nan_{name}", M, c, 512, dict(reg=reg, normalize=name != "seeded", precision=pr, iters=25)


print("package:", os.path.dirname(cfm_b200.__file__))
print("device:", torch.cuda.get_device_name(DEV))
out = {}
for name, M, cmax, n1, kw in cases():
    Md = M[:, :n1].double()
    fin = torch.isfinite(Md)
    out[name + "/M"] = np.array([Md[fin].sum().item(), (Md[fin] ** 2).sum().item(), (~fin).sum().item()])
    lu, lv, st, err = solve(M, cmax, n1, **kw)
    out.update({name + "/log_u": lu, name + "/log_v": lv, name + "/status": st, name + "/err": err})
    print(f"{name:32s} status {st.tolist()} err {err[0]:.3e}")
np.savez(args.out, **out)

if args.compare:
    old = np.load(args.compare)
    bad = [k for k in sorted(set(old.files) | set(out)) if k not in old.files or k not in out
           or not np.array_equal(old[k], out[k], equal_nan=old[k].dtype.kind == "f")]
    # err is summed with atomicAdd in the order the CTAs arrive: from run to run it may differ in the last bits
    err_rel = max([abs(old[k][0] - out[k][0]) / abs(old[k][0]) for k in bad if k.endswith("/err")] or [0.0])
    bad = [k for k in bad if not k.endswith("/err")]
    print(f"compared {len(out)} arrays with {args.compare}: " + ("bit-identical" if not bad else f"DIFFER: {bad}")
          + f"; largest relative difference of err {err_rel:.1e}")
    sys.exit(1 if bad or err_rel > 1e-14 else 0)
