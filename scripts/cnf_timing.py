"""Exact log-likelihood timing: NeuralODE(cnf_wrapper(MLP(dim=2, w=64, time_varying=True), "exact")) in the CNF
variant of the one-launch kernel against the tutorial's cnf_wrapper on a plain torch MLP in eager PyTorch (the
oracle ODE drivers), on the same GPU.  One JSON line per (config, implementation); times from CUDA events after
warm-up, with the card's name and power limit read in the same run.

    python scripts/cnf_timing.py [--reps N]
"""
import json
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


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def eager(wrapped, solver, z, span, tol):
    """The tutorial's field through the oracle drivers (a decreasing dopri5 span as torchdyn integrates it)."""
    if solver == "euler":
        return vf.euler_trajectory(wrapped, z, span), len(span) - 1
    traj, st = vf.dopri5_trajectory(lambda s, x: -wrapped(-s, x), z, -span, tol, tol)
    return traj, st["nfe"]


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 20
    dev = "cuda:0"
    info = card()
    torch.manual_seed(0)
    m = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    stock = vf.make_mlp(2, w=64, time_varying=True)
    stock.load_state_dict(m.state_dict())
    m, stock = m.to(dev), stock.to(dev)
    g = torch.linspace(-3, 3, 200)
    xx, yy = torch.meshgrid(g, g, indexing="ij")
    grid = torch.stack([xx.reshape(-1), yy.reshape(-1)], 1)
    tut = torch.randn(256, 2, generator=torch.Generator().manual_seed(1))
    configs = [("tutorial_B256_euler_101", tut, "euler", 101, None),
               ("grid_200x200_euler_201", grid, "euler", 201, None),
               ("grid_200x200_dopri5_1e-4", grid, "dopri5", 2, 1e-4)]
    for name, x, solver, n_span, tol in configs:
        z = torch.cat([x, torch.zeros(x.shape[0], 1)], 1).to(dev)
        span = torch.linspace(1, 0, n_span)
        node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m), solver=solver, atol=tol or 1e-4, rtol=tol or 1e-4)
        ms = timed(lambda: node.trajectory(z, span), 3, reps)
        out = node.trajectory(z, span)
        print(json.dumps({"config": name, "impl": "cfm_b200 CNF kernel", "B": x.shape[0], "ms": round(ms, 4),
                          "nfe": node.stats["nfe"], **info}), flush=True)
        wrapped = cfm_b200.cnf_wrapper(stock)
        span_d = span.to(dev)
        box = {}

        def run_eager():
            box["out"] = eager(wrapped, solver, z, span_d, tol)

        ms_e = timed(run_eager, 1, max(1, reps // 10))
        ref, nfe = box["out"]
        ll_gap = (out[-1, :, 2] - ref[-1, :, 2]).abs().max().item()
        print(json.dumps({"config": name, "impl": "eager PyTorch (tutorial cnf_wrapper)", "B": x.shape[0],
                          "ms": round(ms_e, 3), "nfe": nfe, "speedup": round(ms_e / ms, 1),
                          "max_ll_gap": ll_gap, **info}), flush=True)


if __name__ == "__main__":
    main()
