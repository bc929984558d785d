"""Sinkhorn solve time and bytes moved per solve at C2 (8192 x 8192, d = 784), a 4096 x 4096 d = 512 shard and
the C5 8192 x 8192 d = 128 shard: reg 0.05, normalised cost, 100 iterations, CUDA events around
`OTPlanSampler._solve_sinkhorn` (3 warm-up solves, then --reps).  status[3] names the kernel variant that ran
(4 = factored sweep on the 3-byte cost stream, 3 = factored on fp32 M).  Bytes are what the variant reads and
writes of M (part of each sweep comes from the L2, so the HBM fraction is an upper bound of the DRAM share):
    fp32 sweeps:    (iterations + 1) x n0 x n1 x 4
    3-byte stream:  n0 x n1 x 4 (fp32 prologue) + n0 x ldc (the copy, written once) + iterations x n0 x ldc,
                    ldc = align16(3 n1)
--root DIR runs the package found in DIR (e.g. another checkout, for old/new comparisons); --dump DIR saves
log_u, log_v and the 8192 drawn index pairs of one seeded C2 coupling."""
import argparse
import json
import os
import subprocess
import sys

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
ap.add_argument("--reps", type=int, default=20)
ap.add_argument("--dump", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import cfm_b200  # noqa: E402

print("package:", os.path.dirname(cfm_b200.__file__))
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                     capture_output=True, text=True).stdout.strip())
dev = torch.device("cuda:0")
CONFIGS = [("C2", 8192, 8192, 784), ("shard4096", 4096, 4096, 512), ("C5_8192", 8192, 8192, 128)]
rows = []
for name, n0, n1, d in CONFIGS:
    g = torch.Generator().manual_seed(0)
    x0, x1 = torch.randn(n0, d, generator=g).to(dev), torch.randn(n1, d, generator=g).to(dev)
    s = cfm_b200.OTPlanSampler("sinkhorn", reg=0.05, normalize_cost=True, num_iter_max=100, stop_thr=0.0, warn=False)
    M, cmax, _, _ = s._cost(x0, x1, dev)
    bufs = s._last_bufs
    for _ in range(3):
        cp = s._solve_sinkhorn(M, cmax, n0, n1, 0.05, True, bufs=bufs)
    torch.cuda.synchronize()
    ms = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        cp = s._solve_sinkhorn(M, cmax, n0, n1, 0.05, True, bufs=bufs)
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    st = cp.status.cpu().tolist()
    iters = st[1]
    ldc = (3 * n1 + 15) // 16 * 16
    if st[3] == 4:
        parts = {"fp32_prologue_read": n0 * n1 * 4, "compact_write": n0 * ldc, "compact_reads": iters * n0 * ldc}
    else:
        parts = {"fp32_reads": (iters + 1) * n0 * n1 * 4}
    total = sum(parts.values())
    med = float(np.median(ms))
    row = {"config": name, "n0": n0, "n1": n1, "d": d, "status": st, "solve_ms_median": med,
           "solve_ms_min": float(np.min(ms)), "solve_ms_max": float(np.max(ms)), "bytes": parts,
           "bytes_total": total, "bytes_per_s": total / (med * 1e-3), "hbm_fraction": total / (med * 1e-3) / HBM_PEAK}
    rows.append(row)
    print(json.dumps(row))
    if args.dump and name == "C2":
        os.makedirs(args.dump, exist_ok=True)
        np.random.seed(0)
        cp = s._couple(x0, x1, dev)
        i, j = s._draw(cp, n0)
        np.savez(os.path.join(args.dump, "c2_coupling.npz"), log_u=cp.log_u.cpu().numpy(),
                 log_v=cp.log_v.cpu().numpy(), i=i.cpu().numpy(), j=j.cpu().numpy(), status=np.array(st))
    del s, M, bufs, cp
    torch.cuda.empty_cache()
print("| config | status[3] | solve ms (median of %d) | GB moved | GB/s | of 3.35 TB/s |" % args.reps)
print("|---|---|---|---|---|---|")
for r in rows:
    print("| %s | %d | %.3f | %.2f | %.0f | %.2f |" % (r["config"], r["status"][3], r["solve_ms_median"],
                                                      r["bytes_total"] / 1e9, r["bytes_per_s"] / 1e9, r["hbm_fraction"]))
