"""Maximum-likelihood CNF training-step timing: the tutorial's cell 4 (Maximum_likelihood_CNF_tutorial.ipynb),

    x0_with_ll = cnf.trajectory(x1_with_ll, t_span=torch.linspace(1, 0, steps + 1))[-1]
    logprob = prior.log_prob(x0_with_ll[..., :-1]) + x0_with_ll[..., -1]
    loss = -torch.mean(logprob); loss.backward(); optimizer.step()

with cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(MLP(dim=2, w=64, time_varying=True), "exact"), solver="euler") (one
forward launch, one backward launch: csrc/ode_small.cu, csrc/cnf_train.cu) against the same cell in eager PyTorch:
the tutorial's cnf_wrapper (torch.func per row) on a plain torch MLP with the same weights, through a grad-enabled
Euler loop over the same span (torchdyn's solver="euler", sensitivity="autograd").  Batches 256 (the tutorial's)
and 4096, 101 span points.  A window is ONE CUDA-event pair around --steps (cfm_b200) or --eager-steps (eager)
consecutive full steps (zero_grad, trajectory, loss, backward, Adam step) after warm-up; the implementations
alternate window by window and the median, minimum and maximum per step over --windows windows are reported.  The
backward kernel's own device time comes from a separate torch.profiler run, with its FLOP count from the shapes.
One JSON line per (batch, implementation) and per (batch, kernel), with the card's name and power limit read in the
same run.

    python scripts/cnf_train_timing.py [--steps N] [--eager-steps N] [--windows N]
"""
import argparse
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
import cfm_b200  # noqa: E402
from oracle import vector_field as vf  # noqa: E402

DIM, W, N_SPAN = 2, 64, 101


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def backward_flops(B, n_span, dim, w):
    """Floating-point operations of one backward launch, from the shapes (csrc/cnf_train.cu): per (row, step) the
    forward with dim tangent chains, the reverse pass of the primal and the tangent chains, grad_x phi and the outer
    products of the 1 + dim (delta, input) pairs per layer; an FMA is two operations."""
    in0, k = dim + 1, 1 + dim
    per = (2 * w * in0 + w * dim          # layer 0 and its tangents
           + 2 * k * 2 * w * w            # layers 1, 2: primal and tangents
           + 2 * dim * w + 3 * dim * w    # layer 3 adjoints, tau_2, e_2
           + 2 * k * 2 * w * w            # W_{l+1}^T of delta and of the tangent adjoints, l = 1, 0
           + 2 * dim * w                  # grad_x phi
           + 2 * k * 2 * w * w            # dW1, dW2 outer products
           + k * 2 * w * in0 + 2 * 2 * dim * w)  # dW0, dW3
    return B * (n_span - 1) * per


def eager_node(model):
    f = cfm_b200.cnf_wrapper(model, likelihood_estimator="exact")

    def trajectory(z, t_span):
        sol = [z]
        for a, b in zip(t_span[:-1], t_span[1:]):
            z = z + (b - a) * f(a, z)
            sol.append(z)
        return torch.stack(sol)

    return trajectory


def make_step(traj_fn, params, prior, x1_with_ll, span):
    opt = torch.optim.Adam(params)

    def step():
        opt.zero_grad()
        x0_with_ll = traj_fn(x1_with_ll, span)[-1]
        logprob = prior.log_prob(x0_with_ll[..., :-1]) + x0_with_ll[..., -1]
        loss = -torch.mean(logprob)
        loss.backward()
        opt.step()
        return loss

    return step


def window(step, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--eager-steps", type=int, default=2)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[256, 4096])
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cnf_train_timing.py needs a CUDA device")
    dev = torch.device("cuda:0")
    info = card()
    prior = torch.distributions.MultivariateNormal(torch.zeros(DIM, device=dev), torch.eye(DIM, device=dev))
    span = torch.linspace(1, 0, N_SPAN, device=dev)
    for B in args.batches:
        torch.manual_seed(0)
        model = cfm_b200.MLP(dim=DIM, w=W, time_varying=True).to(dev)
        plain = vf.make_mlp(DIM, w=W, time_varying=True).to(dev)  # a plain torch MLP with the same weights
        plain.load_state_dict(model.state_dict())
        x1 = torch.randn(B, DIM, device=dev)
        x1_with_ll = torch.cat([x1, torch.zeros(B, 1, device=dev)], dim=-1)
        cnf = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(model, likelihood_estimator="exact"), solver="euler",
                                 sensitivity="adjoint")
        steps = {"cfm_b200": (make_step(cnf.trajectory, list(model.parameters()), prior, x1_with_ll, span),
                              args.steps),
                 "eager": (make_step(eager_node(plain), list(plain.parameters()), prior, x1_with_ll, span),
                           args.eager_steps)}
        for step, _ in steps.values():  # warm-up: module loads, allocator, Adam state
            step()
            step()
        torch.cuda.synchronize()
        times = {k: [] for k in steps}
        for _ in range(args.windows):
            for name, (step, n) in steps.items():
                times[name].append(window(step, n))
        for name, ts in times.items():
            print(json.dumps({"what": "cnf_train_step", "impl": name, "batch": B, "n_span": N_SPAN, "dim": DIM,
                              "w": W, "ms_per_step_median": statistics.median(ts), "ms_min": min(ts),
                              "ms_max": max(ts), "steps_per_window": steps[name][1], "windows": args.windows,
                              **info}), flush=True)

        # the kernels' own device time, in a profiled run of its own
        step = steps["cfm_b200"][0]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                step()
            torch.cuda.synchronize()
        for tag, key in (("backward", "cnf_euler_backward_kernel"), ("forward", "ode_small_kernel")):
            evs = [e for e in prof.key_averages() if key in e.key]
            us = sum(e.device_time_total for e in evs) / max(1, sum(e.count for e in evs))
            rec = {"what": "cnf_kernel", "kernel": tag, "batch": B, "n_span": N_SPAN, "dim": DIM, "w": W,
                   "us_per_call": us, "calls": sum(e.count for e in evs), **info}
            if tag == "backward":
                fl = backward_flops(B, N_SPAN, DIM, W)
                rec.update({"flops": fl, "tflops_per_s": fl / (us * 1e-6) / 1e12 if us else None})
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
