"""Phase timeline of one iteration (it = 50) of the smem-staged fp32 Sinkhorn kernel (sinkhorn_v2.cu) at C2
(N = 8192, d = 784, reg 0.05, normalised cost, 100 iterations; CFM_SK_TL=1): %globaltimer marks of thread 0 of the
first and the last CTA, and the earliest / latest end of the chunk loop over all CTAs.  The boundary window is the
time from the earliest sweep end to the exit of the second grid barrier: the part of the iteration in which no CTA
streams rows of its slab.  --root DIR runs the package found in DIR (old/new comparisons)."""
import argparse
import os
import subprocess
import sys

os.environ["CFM_SK_TL"] = "1"
ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
ap.add_argument("--runs", type=int, default=5, help="solves whose iteration-50 marks are printed")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import cfm_b200  # noqa: E402

N, D = 8192, 784
print("package:", os.path.dirname(cfm_b200.__file__))
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                     capture_output=True, text=True).stdout.strip())
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)
x0, x1 = torch.randn(N, D, generator=g).to(dev), torch.randn(N, D, generator=g).to(dev)
s = cfm_b200.OTPlanSampler("sinkhorn", reg=0.05, normalize_cost=True, num_iter_max=100, stop_thr=0.0, warn=False)
M, cmax, _, _ = s._cost(x0, x1, dev)
bufs = s._last_bufs
names = ["sweep start", "last chunk", "partials stored", "barrier 1", "combine done", "barrier 2"]
for _ in range(3):
    s._solve_sinkhorn(M, cmax, N, N, 0.05, True, bufs=bufs)
torch.cuda.synchronize()
windows, spreads, lengths = [], [], []
for run in range(args.runs):
    cp = s._solve_sinkhorn(M, cmax, N, N, 0.05, True, bufs=bufs)
    torch.cuda.synchronize()
    st = cp.status.cpu().tolist()
    # the timeline marks open the Sinkhorn workspace
    tl = np.frombuffer(bufs["ws_sk"][:18 * 8].cpu().numpy().tobytes(), dtype=np.uint64).astype(np.int64)
    first, last, end_min, end_max = tl[0:6], tl[8:14], tl[16], tl[17]
    t0 = min(first[0], last[0])
    rel = lambda t: (int(t) - t0) / 1e3  # noqa: E731
    print(f"run {run} status {st}")
    for tag, m in (("CTA 0   ", first), ("last CTA", last)):
        print("  " + tag + ": " + ", ".join(f"{n} {rel(m[i]):.2f}" for i, n in enumerate(names)) + " (us)")
    b2 = max(first[5], last[5])
    windows.append((b2 - end_min) / 1e3)
    spreads.append((end_max - end_min) / 1e3)
    lengths.append((b2 - t0) / 1e3)
    print(f"  sweep end over all CTAs: earliest {rel(end_min):.2f}, latest {rel(end_max):.2f} (us)")
    print(f"  window (earliest sweep end -> barrier-2 exit) {windows[-1]:.2f} us, straggler spread {spreads[-1]:.2f} us, "
          f"iteration {lengths[-1]:.2f} us")
print(f"median over {args.runs} solves: window {np.median(windows):.2f} us, straggler spread {np.median(spreads):.2f} us, "
      f"iteration {np.median(lengths):.2f} us")
