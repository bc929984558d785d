"""Action-matching training-step timing: cfm_b200.action_matching_loss (one kernel for the loss, the action's input
gradient and all parameter gradients) against the notebook's own eager double-backward lines on the same GPU
(tutorial_training_8_gaussians_to_moons.ipynb, cell 11),

    st = torch.sum(action(torch.cat([xt, t], dim=-1)))
    dsdx, dsdt = torch.autograd.grad(st, (xt, t), create_graph=True, retain_graph=True)
    a0 = action(torch.cat([x0, torch.zeros(batch_size, 1)], dim=-1))
    a1 = action(torch.cat([x1, torch.ones(batch_size, 1)], dim=-1))
    loss = (a0 - a1 + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt).mean(); loss.backward()

for MLP(dim=2, out_dim=1, w=64, time_varying=True) at the tutorial's batch 256 and at 4096.  Two measurements per batch size and
implementation: (a) loss + backward, (b) a full step with torch.optim.Adam (zero_grad, loss, backward, step).  A
window is ONE CUDA-event pair around --steps consecutive steps after warm-up; the two implementations alternate window
by window in the same run, and the median, minimum and maximum over --windows windows are reported per step.  One
JSON line per (batch, measurement, implementation), with the card's name and power limit read in the same run, and
the gap between the two implementations' losses and gradients at that batch.  The fused kernel's own device time is
measured separately with torch.profiler over --steps calls (one more JSON line per batch).

    python scripts/action_train_timing.py [--steps N] [--windows N]
"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
import cfm_b200  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q}


def window_ms(step, steps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def arg(name, default):
    return int(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def main():
    steps, windows = arg("--steps", 1000), arg("--windows", 7)
    if not torch.cuda.is_available():
        raise SystemExit("action_train_timing.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    info = card()
    for B in (256, 4096):
        g = torch.Generator().manual_seed(B)
        x0, x1 = torch.randn(B, 2, generator=g).to(dev), torch.randn(B, 2, generator=g).to(dev)
        t = torch.rand(B, 1, generator=g).to(dev)
        xt_ = t * x1 + (1 - t) * x0
        torch.manual_seed(0)
        fused = cfm_b200.MLP(dim=2, out_dim=1, w=64, time_varying=True).to(dev)
        eager = cfm_b200.MLP(dim=2, out_dim=1, w=64, time_varying=True).to(dev)
        eager.load_state_dict(fused.state_dict())

        def fused_loss():
            return cfm_b200.action_matching_loss(fused, xt_, t, x0, x1)

        def eager_loss():  # the notebook's lines; MLP.forward under autograd is the plain torch.nn.Sequential
            tt = t.clone().requires_grad_(True)
            xt = xt_.detach().requires_grad_(True)
            st = torch.sum(eager(torch.cat([xt, tt], dim=-1)))
            dsdx, dsdt = torch.autograd.grad(st, (xt, tt), create_graph=True, retain_graph=True)
            xt.requires_grad, tt.requires_grad = False, False
            a0 = eager(torch.cat([x0, torch.zeros(B, 1, device=dev)], dim=-1))
            a1 = eager(torch.cat([x1, torch.ones(B, 1, device=dev)], dim=-1))
            return (a0 - a1 + 0.5 * (dsdx**2).sum(1, keepdims=True) + dsdt).mean()

        # the two implementations compute the same thing at this batch (b3's gradient is 0 in both)
        lf, le = fused_loss(), eager_loss()
        lf.backward()
        le.backward()
        gap = max(((a.grad - b.grad).abs().max() / b.grad.abs().max()).item()
                  for a, b in list(zip(fused.parameters(), eager.parameters()))[:7])
        parity = {"loss_abs_gap": abs(lf.item() - le.item()), "loss": le.item(), "grad_gap_over_max_abs": gap,
                  "b3_grads": [fused.net[6].bias.grad.item(), eager.net[6].bias.grad.item()]}

        # the kernel alone, from the profiler's device timeline
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                fused_loss()
            torch.cuda.synchronize()
        kern = [e for e in prof.events() if "mlp_action_train_kernel" in e.name]
        us = sum(e.device_time for e in kern) / max(len(kern), 1)
        print(json.dumps({"B": B, "measure": "kernel", "impl": "mlp_action_train_kernel", "us_per_call": round(us, 2),
                          "calls": len(kern), **info}), flush=True)

        def backward_only(model, loss_fn):
            def step():
                model.zero_grad(set_to_none=True)
                loss_fn().backward()
            return step

        def adam_step(model, loss_fn):
            opt = torch.optim.Adam(model.parameters())

            def step():
                opt.zero_grad()
                loss_fn().backward()
                opt.step()
            return step

        for what, make in (("loss+backward", backward_only), ("adam_step", adam_step)):
            impls = {"cfm_b200.action_matching_loss": make(fused, fused_loss), "eager PyTorch": make(eager, eager_loss)}
            for step in impls.values():
                window_ms(step, 200)  # warm-up: module load, allocator, optimizer state
            times = {k: [] for k in impls}
            for _ in range(windows):
                for k, step in impls.items():
                    times[k].append(window_ms(step, steps))
            med = {k: statistics.median(v) for k, v in times.items()}
            for k, v in times.items():
                print(json.dumps({"B": B, "measure": what, "impl": k, "us_per_step_median": round(1e3 * med[k], 2),
                                  "us_min": round(1e3 * min(v), 2), "us_max": round(1e3 * max(v), 2),
                                  "steps_per_window": steps, "windows": windows,
                                  "eager_over_fused": round(med["eager PyTorch"] / med["cfm_b200.action_matching_loss"], 2),
                                  **parity, **info}), flush=True)


if __name__ == "__main__":
    main()
