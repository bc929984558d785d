"""Golden vectors for cfm_b200.cnf_wrapper: the exact-likelihood field [f(t, x), tr(df/dx)] as computed by the
reference's OWN cnf_wrapper, whose definition lives in a notebook cell
(examples/2D_tutorials/Maximum_likelihood_CNF_tutorial.ipynb).  The cell's source is read from the checkout and
executed here, on a seeded reference MLP(dim=2, w=64, time_varying=True), in float32 and float64.

    PYTHONPATH=oracle:<torchcfm checkout> TORCHCFM_SRC=<torchcfm checkout> python tests/golden/make_golden_cnf.py

This pins the column order (log-density LAST) and the sign (+div) to the reference.  Only the .npz is kept.
"""
import json
import os

import numpy as np
import torch

import ot  # noqa: F401  (oracle/ot shim)
assert "oracle" in ot.__version__
import torchcfm  # noqa: E402
from torchcfm.models import MLP  # noqa: E402

SRC = os.environ["TORCHCFM_SRC"]
assert os.path.realpath(torchcfm.__file__).startswith(os.path.realpath(SRC)), torchcfm.__file__
HERE = os.path.dirname(os.path.abspath(__file__))
NOTEBOOK = os.path.join(SRC, "examples", "2D_tutorials", "Maximum_likelihood_CNF_tutorial.ipynb")


def reference_cnf_wrapper():
    cells = json.load(open(NOTEBOOK))["cells"]
    src = [("".join(c["source"])) for c in cells if c["cell_type"] == "code"]
    cell = [s for s in src if "class cnf_wrapper" in s]
    assert len(cell) == 1
    ns = {"torch": torch}
    exec(compile(cell[0], NOTEBOOK, "exec"), ns)
    return ns["cnf_wrapper"]


def main():
    cnf_wrapper = reference_cnf_wrapper()
    torch.manual_seed(20)
    model = MLP(dim=2, w=64, time_varying=True)
    out = {f"w_{k}": v.detach().numpy().copy() for k, v in model.state_dict().items()}
    g = torch.Generator().manual_seed(21)
    ts = [1.0, 0.73, 0.5, 0.125, 0.0]
    x = torch.randn(len(ts), 37, 3, generator=g) * 1.5  # [x1, x2, ll]; the ll column is ignored by the field
    out["t"] = np.asarray(ts, dtype=np.float64)
    out["x"] = x.numpy().astype(np.float64)
    for name, dtype in (("f32", torch.float32), ("f64", torch.float64)):
        wrapped = cnf_wrapper(model.to(dtype), likelihood_estimator="exact")
        with torch.no_grad():
            out[f"out_{name}"] = np.stack([
                wrapped(torch.tensor(t, dtype=dtype), x[i].to(dtype)).numpy() for i, t in enumerate(ts)])
    path = os.path.join(HERE, "cnf_vectors.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
