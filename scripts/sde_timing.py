"""SF2M SDE sampling timing: cfm_b200.sdeint (one kernel) against an eager-PyTorch restatement of torchsde's
fixed-step Euler loop driving the notebook's own SDE class (examples/2D_tutorials/SF2M_tutorial.ipynb cell 5) on the
same GPU.  torchsde is not installed, so the comparator is that restatement (one `sde.f` and one `sde.g` call, one
N(0, h) draw and the update per step), not torchsde itself; it pays the per-step launches torchsde would pay and
none of its Brownian-interval bookkeeping, so it is a lower bound on torchsde's time.

Shape: B = 1024, dim 2, MLP(w=64, time_varying=True) drift and score, sigma = 1, ts = linspace(0, 1, 100),
dt = 1e-3 (1000 steps, 2000 MLP evaluations).  Times from CUDA events after warm-up, median of --reps runs, with the
card's name and power limit read in the same run.  One JSON line per implementation.

    python scripts/sde_timing.py [--reps N]
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
import cfm_b200  # noqa: E402
from oracle import vector_field as vf  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def median_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times), min(times), max(times)


class NotebookSDE(torch.nn.Module):
    """The SF2M tutorial's SDE class, verbatim in behaviour."""
    noise_type = "diagonal"
    sde_type = "ito"

    def __init__(self, ode_drift, score, input_size=(3, 32, 32), sigma=1.0):
        super().__init__()
        self.drift, self.score, self.input_size, self.sigma = ode_drift, score, input_size, sigma

    def f(self, t, y):
        y = y.view(-1, *self.input_size)
        if len(t.shape) == len(y.shape):
            x = torch.cat([y, t], 1)
        else:
            x = torch.cat([y, t.repeat(y.shape[0])[:, None]], 1)
        return self.drift(x).flatten(start_dim=1) + self.score(x).flatten(start_dim=1)

    def g(self, t, y):
        return torch.ones_like(y) * self.sigma


@torch.no_grad()
def eager_euler(sde, y0, ts, dt):
    """torchsde's fixed-step Euler loop (grid, update, linear_interp) in eager PyTorch; increments from torch.randn."""
    curr_t = prev_t = ts[0]
    curr_y = prev_y = y0
    ys = [y0]
    for out_t in ts[1:]:
        while curr_t < out_t:
            next_t = min(curr_t + dt, ts[-1])
            h = next_t - curr_t
            prev_t, prev_y = curr_t, curr_y
            dw = torch.randn_like(curr_y) * h.sqrt()
            curr_y = curr_y + sde.f(curr_t, curr_y) * h + sde.g(curr_t, curr_y) * dw
            curr_t = next_t
        t0, t1, t = float(prev_t), float(curr_t), float(out_t)
        ys.append((t1 - t) / (t1 - t0) * prev_y + (t - t0) / (t1 - t0) * curr_y)
    return torch.stack(ys)


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 7
    dev = "cuda:0"
    info = card()
    torch.manual_seed(0)
    drift = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    score = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    plain = [vf.make_mlp(2, w=64, time_varying=True) for _ in range(2)]
    plain[0].load_state_dict(drift.state_dict())
    plain[1].load_state_dict(score.state_dict())
    drift, score = drift.to(dev), score.to(dev)
    plain = [p.to(dev) for p in plain]
    y0 = torch.randn(1024, 2, generator=torch.Generator().manual_seed(1)).to(dev)
    ts = torch.linspace(0, 1, 100)
    ts_dev = ts.to(dev)

    sde = cfm_b200.SDE(drift, score, input_size=(2,), sigma=1.0)
    ms, lo, hi = median_ms(lambda: cfm_b200.sdeint(sde, y0, ts, method="euler", dt=1e-3), 3, reps)
    ys = cfm_b200.sdeint(sde, y0, ts, method="euler", dt=1e-3)
    print(json.dumps({"config": "sf2m_B1024_dim2_w64_ts100_dt1e-3", "impl": "cfm_b200.sdeint (one kernel)",
                      "ms_median": round(ms, 3), "ms_min": round(lo, 3), "ms_max": round(hi, 3), "reps": reps,
                      "steps": 1000, "finite": bool(torch.isfinite(ys).all()), **info}), flush=True)

    nb = NotebookSDE(plain[0], plain[1], input_size=(2,), sigma=1.0)
    ms_e, lo_e, hi_e = median_ms(lambda: eager_euler(nb, y0, ts_dev, 1e-3), 1, max(3, reps // 2))
    print(json.dumps({"config": "sf2m_B1024_dim2_w64_ts100_dt1e-3",
                      "impl": "eager PyTorch restatement of torchsde's Euler loop (notebook SDE class)",
                      "ms_median": round(ms_e, 2), "ms_min": round(lo_e, 2), "ms_max": round(hi_e, 2),
                      "reps": max(3, reps // 2), "steps": 1000, "speedup_median": round(ms_e / ms, 1), **info}),
          flush=True)


if __name__ == "__main__":
    main()
