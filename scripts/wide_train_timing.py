"""Wide flow-matching training-step timing: the MNIST OT-CFM model of BASELINE config 3,
MLP(784, w=256, time_varying=True) with SELU, at B = 128, 1024 and 8192, through

    loss = cfm_b200.flow_matching_loss(model, xt, t, ut); loss.backward()      (csrc/train_tc.cu, 19 launches)

against the eager lines on a plain torch MLP with the same weights (fp32, TF32 off, as the parity gates need):

    vt = model(torch.cat([xt, t[:, None]], -1)); loss = torch.mean((vt - ut) ** 2); loss.backward()

A window is ONE CUDA-event pair around --steps consecutive steps after warm-up, either loss + backward() or a full
torch.optim.Adam step (zero_grad, loss, backward, step); the implementations alternate window by window and the
median, minimum and maximum per step over --windows windows are reported, beside the loss and gradient agreement of
the two implementations on the same batch.  The library's device time per call comes from a torch.profiler run in a
child process of its own (--profile-only), summed over every kernel one call launches, with the achieved rate against
the FLOP count of the shapes.  The card's name, power limit and SM clock are read in the same run.

    python scripts/wide_train_timing.py [--steps N] [--windows N] [--batches B ...]
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

DIM, W = 784, 256
LIB_KERNELS = ("gemm_wg_splitk_kernel", "split_pair_kernel", "weight_absmax_kernel", "tc_fold_kernel")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30).stdout
    except (OSError, subprocess.SubprocessError):
        q = ""
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.strip()}


def step_flops(B, dim=DIM, w=W, out=DIM):
    """Model FLOPs of one loss + gradient call from the shapes (an FMA is two): the forward GEMMs, about as much for
    the weight gradients, and the delta GEMMs (no input gradient).  fp16x3 issues each on the tensor cores three
    times."""
    fwd = 2 * (dim * w + 2 * w * w + w * out)
    return B * (2 * fwd + 2 * (out * w + 2 * w * w))


def batch(B, g):
    return (torch.randn(B, DIM, generator=g).cuda(), torch.rand(B, generator=g).cuda(),
            torch.randn(B, DIM, generator=g).cuda())


def make(model, plain, B):
    g = torch.Generator().manual_seed(B)
    xt, t, ut = batch(B, g)

    def lib_loss():
        return cfm_b200.flow_matching_loss(model, xt, t, ut)

    def eager_loss():
        vt = plain(torch.cat([xt, t[:, None]], -1))
        return torch.mean((vt - ut) ** 2)

    return lib_loss, eager_loss


def window(step, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def profile_only(batches, steps):
    for B in batches:
        torch.manual_seed(0)
        model = cfm_b200.MLP(dim=DIM, w=W, time_varying=True).cuda()
        lib_loss, _ = make(model, None, B)
        for _ in range(3):
            lib_loss().backward()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(steps):
                lib_loss().backward()
            torch.cuda.synchronize()
        evs = [e for e in prof.key_averages() if any(k in e.key for k in LIB_KERNELS)]
        us = sum(e.device_time_total for e in evs) / steps
        fl = step_flops(B)
        per_kernel = {k: sum(e.device_time_total for e in evs if k in e.key) / steps for k in LIB_KERNELS}
        print(json.dumps({"what": "wide_train_kernels", "batch": B, "us_per_call": us, "launches_per_call":
                          sum(e.count for e in evs) / steps, "model_flops": fl,
                          "model_tflops_per_s": fl / (us * 1e-6) / 1e12 if us else None,
                          "issued_tensor_tflops_per_s": 3 * fl / (us * 1e-6) / 1e12 if us else None,
                          "per_kernel_us": per_kernel, **card()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--batches", type=int, nargs="+", default=[128, 1024, 8192])
    ap.add_argument("--profile-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("wide_train_timing.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    if args.profile_only:
        return profile_only(args.batches, args.steps)
    info = card()
    for B in args.batches:
        torch.manual_seed(0)
        model = cfm_b200.MLP(dim=DIM, w=W, time_varying=True).cuda()
        plain = vf.make_mlp(DIM, w=W, time_varying=True).cuda()
        plain.load_state_dict(model.state_dict())
        lib_loss, eager_loss = make(model, plain, B)
        # agreement on the same batch and weights
        model.zero_grad(set_to_none=True)
        plain.zero_grad(set_to_none=True)
        la, lb = lib_loss(), eager_loss()
        la.backward()
        lb.backward()
        gap = max(((p.grad - q.grad).abs().max() / q.grad.abs().max()).item()
                  for p, q in zip(model.parameters(), plain.parameters()))
        agree = {"loss_lib": la.item(), "loss_eager": lb.item(), "grad_max_abs_rel_gap": gap}
        opts = {"cfm_b200": torch.optim.Adam(model.parameters(), lr=1e-5),
                "eager": torch.optim.Adam(plain.parameters(), lr=1e-5)}
        losses = {"cfm_b200": lib_loss, "eager": eager_loss}

        def backward_step(name):
            return lambda: losses[name]().backward()

        def adam_step(name):
            def f():
                opts[name].zero_grad()
                losses[name]().backward()
                opts[name].step()
            return f

        for kind, mk in (("loss_backward", backward_step), ("adam_step", adam_step)):
            steps = {k: mk(k) for k in losses}
            for s in steps.values():
                s()
                s()
            torch.cuda.synchronize()
            times = {k: [] for k in steps}
            for _ in range(args.windows):
                for name, s in steps.items():
                    times[name].append(window(s, args.steps))
            for name, ts in times.items():
                print(json.dumps({"what": "wide_train_step", "step": kind, "impl": name, "batch": B,
                                  "ms_per_step_median": statistics.median(ts), "ms_min": min(ts), "ms_max": max(ts),
                                  "steps_per_window": args.steps, "windows": args.windows, **agree, **info}),
                      flush=True)
    # device time per call, traced in a process of its own
    subprocess.run([sys.executable, __file__, "--profile-only", "--steps", str(args.steps), "--batches",
                    *map(str, args.batches)], check=True)


if __name__ == "__main__":
    main()
