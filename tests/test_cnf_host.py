"""CPU checks of the exact-likelihood (CNF) path: cnf_wrapper against the reference's own cnf_wrapper
(tests/golden/cnf_vectors.npz), the time-reversed MLP behind decreasing spans, and the float64 CNF oracle
(tests/cnf_oracle.py) on a case with a closed-form answer."""
import os

import numpy as np
import pytest
import torch

import cnf_oracle as co
from conftest import ROOT
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import models


@pytest.fixture(scope="module")
def golden_cnf():
    return dict(np.load(os.path.join(ROOT, "tests", "golden", "cnf_vectors.npz")))


def _mlp_from_golden(g, dtype):
    m = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    m.load_state_dict({k[2:]: torch.from_numpy(v) for k, v in g.items() if k.startswith("w_")})
    return m.to(dtype)


@pytest.mark.parametrize("name,dtype,tol", [("f64", torch.float64, 1e-12), ("f32", torch.float32, 1e-6)])
def test_cnf_wrapper_forward_matches_the_reference_cell(golden_cnf, name, dtype, tol):
    g = golden_cnf
    wrapped = cfm_b200.cnf_wrapper(_mlp_from_golden(g, dtype), likelihood_estimator="exact")
    for i, t in enumerate(g["t"]):
        out = wrapped(torch.tensor(t, dtype=dtype), torch.from_numpy(g["x"][i]).to(dtype))
        ref = g[f"out_{name}"][i]
        assert out.shape == ref.shape == (37, 3)
        err = np.abs(out.detach().double().numpy() - ref).max()
        assert err <= tol * max(1.0, np.abs(ref).max()), (t, err)


def test_cnf_wrapper_constructor_and_estimators():
    torch.manual_seed(0)
    m = cfm_b200.MLP(dim=2, w=32, time_varying=True)
    w = cfm_b200.cnf_wrapper(m)
    assert w.model is m and w.div_fn is models.exact_div_fn and w.eps_fn is None
    assert w.likelihood_estimator == "exact"
    hg = cfm_b200.cnf_wrapper(m, likelihood_estimator="hutch_gaussian")
    assert hg.div_fn is models.div_fn_hutch_trace and hg.eps_fn is torch.randn_like
    hr = cfm_b200.cnf_wrapper(m, likelihood_estimator="hutch_rademacher")
    assert hr.div_fn is models.div_fn_hutch_trace
    eps = hr.eps_fn(torch.empty(64, 2))
    assert set(eps.unique().tolist()) <= {-1.0, 1.0}
    with pytest.raises(NotImplementedError, match="likelihood estimator bogus is not implemented"):
        cfm_b200.cnf_wrapper(m, likelihood_estimator="bogus")
    # the Hutchinson estimate with eps = e_k summed over k is the exact trace
    z = torch.randn(5, 3)
    t = torch.tensor(0.3)
    exact = w(t, z)[:, -1]
    total = torch.zeros(5)
    for k in range(2):
        hr.eps_fn = lambda x, k=k: torch.nn.functional.one_hot(torch.full(x.shape[:1], k), 2).to(x)
        total = total + hr(t, z)[:, -1]
    assert torch.allclose(total, exact, atol=1e-5)


def test_cnf_wrapper_trains_with_autograd():
    """Maximum-likelihood training backpropagates through forward() (plain PyTorch on any device)."""
    torch.manual_seed(1)
    m = cfm_b200.MLP(dim=2, w=32, time_varying=True)
    w = cfm_b200.cnf_wrapper(m)
    z = torch.cat([torch.randn(16, 2), torch.zeros(16, 1)], 1)
    for t in torch.linspace(1, 0, 4)[:-1]:
        z = z - (1 / 3) * w(t, z)
    z[:, -1].sum().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in m.parameters())
    assert m.net[0].weight.grad.abs().sum() > 0


def test_time_reversed_mlp_is_the_reparametrised_field():
    torch.manual_seed(2)
    m = cfm_b200.MLP(dim=3, w=32, time_varying=True)
    r = m._time_reversed()
    assert r is m._time_reversed()  # cached per weight version
    assert sorted(m.state_dict()) == sorted(cfm_b200.MLP(dim=3, w=32, time_varying=True).state_dict())
    x, s = torch.randn(50, 3, dtype=torch.float64), 0.37
    col = torch.full((50, 1), s, dtype=torch.float64)
    f_rev = vf.mlp_forward_from_state(r.state_dict(), torch.cat([x, col], 1))
    f_neg = -vf.mlp_forward_from_state(m.state_dict(), torch.cat([x, -col], 1))
    assert torch.equal(f_rev, f_neg)
    with torch.no_grad():
        m.net[6].bias.add_(1.0)
    r2 = m._time_reversed()
    assert torch.equal(r2.net[6].bias, -m.net[6].bias)
    m.act = cfm_b200._ffi.ACT_SILU
    assert m._time_reversed().act == cfm_b200._ffi.ACT_SILU


def test_oracle_reversed_dopri5_returns_to_the_start():
    torch.manual_seed(3)
    mc = vf.make_mlp(2, w=32, time_varying=True, dtype=torch.float64)
    f = lambda t, z: vf.wrapped_forward(mc, t, z)  # noqa: E731
    x0 = torch.randn(64, 2, dtype=torch.float64)
    fwd, _ = co.dopri5_any_direction(f, x0, torch.linspace(0, 1, 3, dtype=torch.float64), 1e-9, 1e-9)
    back, st = co.dopri5_any_direction(f, fwd[-1], torch.linspace(1, 0, 3, dtype=torch.float64), 1e-9, 1e-9)
    assert back.shape == (3, 64, 2) and st["accepted"] >= 2
    assert torch.allclose(back[1], fwd[1], atol=1e-5)  # the global error of a 1e-9 local tolerance
    assert torch.allclose(back[-1], x0, atol=1e-5)


@pytest.mark.parametrize("solver", ["euler", "dopri5"])
def test_oracle_analytic_affine_field_gives_minus_trace(solver):
    """SELU is linear (lambda x) where every hidden pre-activation is positive, so f is affine in x with
    A = lambda^3 W3 W2 W1 W0x, tr(df/dx) is the constant tr(A) and ll over [1, 0] is exactly -tr(A)."""
    mc = co.positive_selu_mlp(dim=2, w=64, seed=5)
    tr = co.affine_trace(mc, 2)
    assert abs(tr) > 1e-3
    seen = []
    f = co.recording(co.cnf_field(mc), seen)
    g = torch.Generator().manual_seed(6)
    z = torch.cat([2 * torch.randn(128, 2, generator=g, dtype=torch.float64),
                   torch.zeros(128, 1, dtype=torch.float64)], 1)
    span = torch.linspace(1, 0, 101, dtype=torch.float64)
    if solver == "euler":
        traj = co.euler_any_direction(f, z, span)
    else:
        traj, _ = co.dopri5_any_direction(f, z, span[[0, -1]], 1e-6, 1e-6)
    assert co.min_preactivation(mc, seen) > 0.0
    ll = traj[-1][:, -1]
    assert torch.allclose(ll, torch.full_like(ll, -tr), rtol=0, atol=1e-12 * max(1.0, abs(tr)) * 100)


def test_cnf_abi_entry_points_are_declared_and_bound():
    from cfm_b200 import _ffi
    assert _ffi.SIGNATURES["cfm_ode_small_cnf_supported"][1] == [_ffi._i64, _ffi._i, _ffi._i]
    assert (_ffi.SIGNATURES["cfm_ode_small_cnf_trajectory_f32"][1]
            == _ffi.SIGNATURES["cfm_ode_small_trajectory_f32"][1])
