"""Wide Hutchinson likelihood timing: NeuralODE(cnf_wrapper(MLP(784, w=256, time_varying=True), "hutch_*")) on the
tensor cores (csrc/cnf_tc.cu: per evaluation the probe, 4 primal + 4 tangent fp16x3 GEMMs and the fold; per Euler step
one more launch, replayed as a CUDA graph) at the MNIST notebook's model (BASELINE config 3's shape), SELU.

* Euler over linspace(1, 0, 101) for both estimators, B in {1024, 10000}, against the reference's
  cnf_wrapper(model, "hutch_gaussian") (cfm_b200.cnf_wrapper.forward is its plain-PyTorch body: torch.func.vjp under
  vmap, randn_like probes) in an eager restatement of torchdyn's Euler loop on the same GPU, fp32, TF32 off;
* dopri5 at atol = rtol = 1e-4 over [1, 0], B = 1024, Gaussian probes (device only; nfe reported).

Device and eager runs alternate, one call per timed window, CUDA events after warm-up, medians.  The card's name and
power limit are read in the same run.  One JSON line per measurement.

    python scripts/cnf_tc_timing.py [--reps N]
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ".")
import cfm_b200  # noqa: E402
from oracle import vector_field as vf  # noqa: E402
from sde_timing import card  # noqa: E402

DIM, W = 784, 256


def eager_euler(wrapper, z, span):
    """torchdyn's fixed-step Euler: x <- x + (t_{n+1} - t_n) f(t_n, x)."""
    x = z
    for a, b in zip(span[:-1], span[1:]):
        x = x + (b - a) * wrapper(a, x)
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


def main():
    reps = int(sys.argv[sys.argv.index("--reps") + 1]) if "--reps" in sys.argv else 5
    dev = "cuda:0"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    info = card()
    torch.manual_seed(0)
    m = cfm_b200.MLP(dim=DIM, w=W, time_varying=True)
    plain = vf.make_mlp(DIM, w=W, time_varying=True)
    plain.load_state_dict(m.state_dict())
    m, plain = m.to(dev), plain.to(dev)
    ref = cfm_b200.cnf_wrapper(plain, likelihood_estimator="hutch_gaussian")
    span = torch.linspace(1, 0, 101)
    span_dev = span.to(dev)

    for B in (1024, 10000):
        z = torch.cat([torch.randn(B, DIM, generator=torch.Generator().manual_seed(B)), torch.zeros(B, 1)], 1).to(dev)
        nodes = {est: cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator=est), solver="euler")
                 for est in ("hutch_gaussian", "hutch_rademacher")}

        def device(est):
            with torch.no_grad():
                return nodes[est].trajectory(z, span)

        def eager():
            with torch.no_grad():
                return eager_euler(ref, z, span_dev)

        for est in nodes:
            device(est)
        eager()
        torch.cuda.synchronize()
        t = {"hutch_gaussian": [], "hutch_rademacher": [], "eager": []}
        for _ in range(reps):
            for est in nodes:
                t[est].append(timed(lambda: device(est)))
            t["eager"].append(timed(eager))
        out = device("hutch_gaussian")
        e = med(t["eager"])
        for est in nodes:
            d = med(t[est])
            print(json.dumps({"config": f"euler100_{est}_B{B}_dim{DIM}_w{W}", "device_ms_median": round(d, 3),
                              "device_ms_min_max": [round(min(t[est]), 3), round(max(t[est]), 3)],
                              "eager_hutch_gaussian_ms_median": round(e, 2),
                              "eager_ms_min_max": [round(min(t["eager"]), 2), round(max(t["eager"]), 2)],
                              "speedup_median": round(e / d, 2), "finite": bool(torch.isfinite(out).all()),
                              "reps": reps, **info}), flush=True)

    B = 1024
    z = torch.cat([torch.randn(B, DIM, generator=torch.Generator().manual_seed(B)), torch.zeros(B, 1)], 1).to(dev)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(m, likelihood_estimator="hutch_gaussian"), solver="dopri5",
                              atol=1e-4, rtol=1e-4)
    span2 = torch.linspace(1, 0, 2)

    def dopri():
        with torch.no_grad():
            return node.trajectory(z, span2)

    dopri()
    dopri()
    ts = [timed(dopri) for _ in range(reps)]
    out = dopri()
    print(json.dumps({"config": f"dopri5_1e-4_hutch_gaussian_B{B}_dim{DIM}_w{W}", "device_ms_median": round(med(ts), 3),
                      "device_ms_min_max": [round(min(ts), 3), round(max(ts), 3)], "nfe": node.stats["nfe"],
                      "accepted": node.stats["accepted"], "rejected": node.stats["rejected"],
                      "finite": bool(torch.isfinite(out).all()), "reps": reps, **info}), flush=True)


if __name__ == "__main__":
    main()
