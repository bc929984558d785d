"""Wide SF2M SDE sampling timing: cfm_b200.sdeint's tensor-core class (per step one pair launch of the fused fp16x3
forward for drift and score, one step kernel, replayed as a CUDA graph) at the MNIST notebook's model, MLP(784, w=256,
time_varying=True) for drift and score (BASELINE config 3's shape), SELU, sigma = 0.1.

* sdeint for B in {256, 1024, 10000} and two grids: ts = linspace(0, 1, 2), dt = 0.01 (the notebook's call, 100
  steps) and ts = linspace(0, 1, 100), dt = 1e-3 (1000 steps);
* against an eager-PyTorch restatement of torchsde's Euler loop over the notebook's SDE.f / SDE.g (sde_timing.py's;
  fp32, TF32 off), which is a lower bound on torchsde's own time;
* the pair launch (cfm_mlp_pair_forward_split_f32) against two single launches of the forward on the same operands
  (cfm_mlp_forward_split_gated_f32), per B, alternating, 20 launches per timed window, medians.

CUDA events after warm-up; the card's name and power limit are read in the same run.  One JSON line per measurement.

    python scripts/sde_tc_timing.py [--reps N]
"""
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ".")
import cfm_b200  # noqa: E402
from cfm_b200 import _ffi  # noqa: E402
from oracle import vector_field as vf  # noqa: E402
from sde_timing import NotebookSDE, card, eager_euler, median_ms  # noqa: E402

DIM, W, SIGMA = 784, 256, 0.1
GRIDS = {"notebook_ts2_dt1e-2": (torch.linspace(0, 1, 2), 1e-2), "ts100_dt1e-3": (torch.linspace(0, 1, 100), 1e-3)}


def pair_vs_two(drift, score, B, reps, dev):
    """(pair, two singles) medians in microseconds per forward of both nets."""
    L = _ffi.lib()
    x = torch.randn(B, DIM, device=dev)
    hi = x.half()
    lo = ((x - hi.float()) * 2048).half()
    t = torch.tensor([0.5], device=dev)
    blobs = [m._prepared(True, torch.device(dev)) for m in (drift, score)]
    one = L.cfm_mlp_workspace_bytes(B, DIM, W, DIM, 2)
    ws = _ffi.workspace(2 * one, dev)
    ya, yb = torch.empty(B, DIM, device=dev), torch.empty(B, DIM, device=dev)
    sp = _ffi.stream_ptr(dev)

    def pair():
        _ffi.check(L.cfm_mlp_pair_forward_split_f32(
            _ffi.ptr(blobs[0]), _ffi.ptr(blobs[1]), _ffi.ptr(hi), _ffi.ptr(lo), B, DIM, W, DIM, 1, _ffi.ptr(t), 0.0,
            drift.act, _ffi.ptr(ya), _ffi.ptr(yb), _ffi.ptr(ws), ws.numel(), sp), "pair")

    def two():
        for blob, y in zip(blobs, (ya, yb)):
            _ffi.check(L.cfm_mlp_forward_split_gated_f32(
                _ffi.ptr(blob), _ffi.ptr(hi), _ffi.ptr(lo), B, DIM, W, DIM, 1, _ffi.ptr(t), 0.0, drift.act,
                _ffi.ptr(y), None, _ffi.ptr(ws), one, sp), "single")

    def window(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1000 / 20

    for _ in range(5):
        pair()
        two()
    torch.cuda.synchronize()
    tp, tt = [], []
    for _ in range(reps):
        tp.append(window(pair))
        tt.append(window(two))
    return statistics.median(tp), statistics.median(tt), min(tp), max(tp), min(tt), max(tt)


@torch.no_grad()
def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 7
    dev = "cuda:0"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = card()
    torch.manual_seed(0)
    drift = cfm_b200.MLP(dim=DIM, w=W, time_varying=True)
    score = cfm_b200.MLP(dim=DIM, w=W, time_varying=True)
    plain = [vf.make_mlp(DIM, w=W, time_varying=True) for _ in range(2)]
    plain[0].load_state_dict(drift.state_dict())
    plain[1].load_state_dict(score.state_dict())
    drift, score = drift.to(dev), score.to(dev)
    plain = [p.to(dev) for p in plain]
    sde = cfm_b200.SDE(drift, score, input_size=(DIM,), sigma=SIGMA)
    nb = NotebookSDE(plain[0], plain[1], input_size=(DIM,), sigma=SIGMA)

    for B in (256, 1024, 10000):
        tp, tt, *spread = pair_vs_two(drift, score, B, max(reps, 15), dev)
        print(json.dumps({"config": f"pair_forward_B{B}_dim{DIM}_w{W}", "pair_us_median": round(tp, 2),
                          "two_singles_us_median": round(tt, 2), "pair_over_two": round(tp / tt, 3),
                          "pair_us_min_max": [round(v, 2) for v in spread[:2]],
                          "two_us_min_max": [round(v, 2) for v in spread[2:]], **info}), flush=True)
        y0 = torch.randn(B, DIM, generator=torch.Generator().manual_seed(1)).to(dev)
        for name, (ts, dt) in GRIDS.items():
            steps = len(cfm_b200.sde.step_schedule(ts, dt)[0]) - 1
            ms, lo, hi = median_ms(lambda: cfm_b200.sdeint(sde, y0, ts, method="euler", dt=dt), 2, reps)
            ys = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=dt)
            ms_e, lo_e, hi_e = median_ms(lambda: eager_euler(nb, y0, ts.to(dev), dt), 1, max(3, reps // 2))
            print(json.dumps({"config": f"sdeint_B{B}_dim{DIM}_w{W}_{name}", "steps": steps,
                              "sdeint_ms_median": round(ms, 3), "sdeint_ms_min_max": [round(lo, 3), round(hi, 3)],
                              "eager_ms_median": round(ms_e, 2), "eager_ms_min_max": [round(lo_e, 2), round(hi_e, 2)],
                              "speedup_median": round(ms_e / ms, 2), "finite": bool(torch.isfinite(ys).all()),
                              "reps": reps, **info}), flush=True)


if __name__ == "__main__":
    main()
