"""Wide action-matching sampling timing: NeuralODE(torch_wrapper(GradModel(MLP(784, out_dim=1, w=256,
time_varying=True)))) on the tensor cores (csrc/grad_tc.cu: per evaluation three primal and three reverse fp16x3 GEMMs;
per Euler step one more launch, replayed as a CUDA graph) at the MNIST notebook's shape, SELU.

* Euler over linspace(0, 1, 100), B in {1024, 10000}, against the stock GradModel (autograd with create_graph=True,
  cfm_b200.GradModel.forward is the reference's body) on a plain fp32 MLP in an eager restatement of torchdyn's Euler
  loop on the same GPU, TF32 off;
* dopri5 at atol = rtol = 1e-4 over [0, 1], B in {1024, 10000} (device only; nfe reported);
* per launch: one Euler trajectory per batch under torch.profiler, the mean device time of each kernel of a step.

Device and eager runs alternate, one call per timed window, CUDA events after warm-up, medians.  The card's name and
power limit are read in the same run.  One JSON line per measurement.

    python scripts/grad_tc_timing.py [--reps N]
"""
import json
import os
import re
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ".")
import cfm_b200  # noqa: E402
from oracle import vector_field as vf  # noqa: E402
from sde_timing import card  # noqa: E402

DIM, W = 784, 256


def eager_euler(wrapper, x, span):
    """torchdyn's fixed-step Euler: x <- x + (t_{n+1} - t_n) f(t_n, x); the state is detached after every step (the
    stock field needs autograd to evaluate, not to be differentiated here)."""
    with torch.enable_grad():
        for a, b in zip(span[:-1], span[1:]):
            x = (x + (b - a) * wrapper(a, x)).detach()
    return x


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def med(v):
    v = sorted(v)
    return v[len(v) // 2]


def per_launch(run, steps):
    """{kernel: mean device us per step} of one call of ``run`` under torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        if e.device_type.name == "CUDA" and e.count >= steps:
            k = re.search(r"(\w+_kernel)(?:<(?:[\w:() ]*::)?(\w+)>)?", e.key)
            name = e.key[:60] if k is None else k.group(1) + (f"<{k.group(2)}>" if k.group(2) else "")
            out[name] = round(out.get(name, 0.0) + e.device_time_total / steps, 2)
    return out


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    dev = "cuda:0"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = card()
    torch.manual_seed(0)
    m = cfm_b200.MLP(dim=DIM, out_dim=1, w=W, time_varying=True)
    plain = vf.make_mlp(DIM, out_dim=1, w=W, time_varying=True)
    plain.load_state_dict(m.state_dict())
    m, plain = m.to(dev), plain.to(dev)
    ref = cfm_b200.torch_wrapper(cfm_b200.GradModel(plain))
    span = torch.linspace(0, 1, 100)
    span_dev = span.to(dev)

    for B in (1024, 10000):
        x = torch.randn(B, DIM, generator=torch.Generator().manual_seed(B)).to(dev)
        node = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(cfm_b200.GradModel(m)), solver="euler")

        def device():
            with torch.no_grad():
                return node.trajectory(x, span)

        def eager():
            return eager_euler(ref, x, span_dev)

        device()
        eager()
        torch.cuda.synchronize()
        td, te = [], []
        for _ in range(reps):
            td.append(timed(device))
            te.append(timed(eager))
        out = device()
        err = float((out[-1] - eager()).abs().max())
        d, e = med(td), med(te)
        print(json.dumps({"config": f"euler100_B{B}_dim{DIM}_w{W}", "device_ms_median": round(d, 3),
                          "device_ms_min_max": [round(min(td), 3), round(max(td), 3)],
                          "device_us_per_step": round(1000 * d / (span.numel() - 1), 1),
                          "eager_gradmodel_ms_median": round(e, 2),
                          "eager_ms_min_max": [round(min(te), 2), round(max(te), 2)],
                          "speedup_median": round(e / d, 2), "max_abs_diff_to_eager": err,
                          "graph": node.stats["graph"], "reps": reps, **info}), flush=True)
        print(json.dumps({"config": f"euler100_B{B}_per_launch_us_per_step",
                          "kernels": per_launch(device, span.numel() - 1), **info}), flush=True)

        dnode = cfm_b200.NeuralODE(cfm_b200.torch_wrapper(cfm_b200.GradModel(m)), solver="dopri5", atol=1e-4,
                                   rtol=1e-4)
        span2 = torch.linspace(0, 1, 2)

        def dopri():
            with torch.no_grad():
                return dnode.trajectory(x, span2)

        dopri()
        dopri()
        ts = [timed(dopri) for _ in range(reps)]
        out = dopri()
        print(json.dumps({"config": f"dopri5_1e-4_B{B}_dim{DIM}_w{W}", "device_ms_median": round(med(ts), 3),
                          "device_ms_min_max": [round(min(ts), 3), round(max(ts), 3)], "nfe": dnode.stats["nfe"],
                          "accepted": dnode.stats["accepted"], "rejected": dnode.stats["rejected"],
                          "finite": bool(torch.isfinite(out).all()), "reps": reps, **info}), flush=True)


if __name__ == "__main__":
    main()
