"""Training-step timing: cfm_b200.flow_matching_loss (one kernel for the loss and all parameter gradients) against the
tutorials' own eager lines on the same GPU,

    vt = model(torch.cat([xt, t[:, None]], dim=-1)); loss = torch.mean((vt - ut) ** 2); loss.backward()

for MLP(dim=2, w=64, time_varying=True) at the tutorial's batch 256 and at 4096.  Two measurements per batch size and
implementation: (a) loss + backward, (b) a full step with torch.optim.Adam (zero_grad, loss, backward, step).  A
window is ONE CUDA-event pair around --steps consecutive steps after warm-up; the two implementations alternate window
by window in the same run, and the median, minimum and maximum over --windows windows are reported per step.  One
JSON line per (batch, measurement, implementation), with the card's name and power limit read in the same run, and
the gap between the two implementations' losses and gradients at that batch.

    python scripts/train_timing.py [--steps N] [--windows N]
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
        raise SystemExit("train_timing.py measures on a CUDA device; none is available")
    dev = "cuda:0"
    info = card()
    for B in (256, 4096):
        g = torch.Generator().manual_seed(B)
        xt, t, ut = (torch.randn(B, 2, generator=g).to(dev), torch.rand(B, generator=g).to(dev),
                     torch.randn(B, 2, generator=g).to(dev))
        torch.manual_seed(0)
        fused = cfm_b200.MLP(dim=2, w=64, time_varying=True).to(dev)
        eager = cfm_b200.MLP(dim=2, w=64, time_varying=True).to(dev)
        eager.load_state_dict(fused.state_dict())

        def fused_loss():
            return cfm_b200.flow_matching_loss(fused, xt, t, ut)

        def eager_loss():  # MLP.forward under autograd is the plain torch.nn.Sequential
            vt = eager(torch.cat([xt, t[:, None]], dim=-1))
            return torch.mean((vt - ut) ** 2)

        # the two implementations compute the same thing at this batch
        lf, le = fused_loss(), eager_loss()
        lf.backward()
        le.backward()
        gap = max(((a.grad - b.grad).abs().max() / b.grad.abs().max()).item()
                  for a, b in zip(fused.parameters(), eager.parameters()))
        parity = {"loss_rel_gap": abs(lf.item() - le.item()) / le.item(), "grad_gap_over_max_abs": gap}

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
            impls = {"cfm_b200.flow_matching_loss": make(fused, fused_loss), "eager PyTorch": make(eager, eager_loss)}
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
                                  "eager_over_fused": round(med["eager PyTorch"] / med["cfm_b200.flow_matching_loss"], 2),
                                  **parity, **info}), flush=True)


if __name__ == "__main__":
    main()
