"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the sampling path (B).

* ``make_mlp`` / ``mlp_forward``: the reference vector field
  (torchcfm/models/models.py:4-21): Linear-SELU-Linear-SELU-Linear-SELU-Linear
  with the submodule name ``net`` so state_dicts interchange.  Pure torch; float64
  available for the parity gate.
* ``wrapped_forward``: torchcfm/utils.py:44-52 -- ``t`` appended as the LAST input
  column, one scalar shared by the batch.
* ``dopri5_trajectory``: torchdyn >=1.0.6 ``NeuralODE(solver='dopri5').trajectory``
  as used by examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb
  :332-338.  torchdyn is NOT in the reference tree and not installed; the driver is
  restated from its published source (numerics/odeint.py::_adaptive_odeint,
  numerics/solvers/ode.py::DormandPrince45, numerics/utils.py::{hairer_norm,
  init_step,adapt_step}; SURVEY.md Appendix B).  PARITY UNPINNED: the reference
  holds no numeric test of any trajectory (tests/test_models.py only constructs).
  ``record=[]`` collects one entry per step attempt (t, dt, ratio, accepted,
  clipped), for tests that must know which controller branches a case takes.
"""
import torch


def make_mlp(dim, out_dim=None, w=64, time_varying=False, dtype=torch.float32):
    """models.py:4-18."""
    out_dim = dim if out_dim is None else out_dim

    class _MLP(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.net = torch.nn.Sequential(
                torch.nn.Linear(dim + (1 if time_varying else 0), w), torch.nn.SELU(),
                torch.nn.Linear(w, w), torch.nn.SELU(),
                torch.nn.Linear(w, w), torch.nn.SELU(),
                torch.nn.Linear(w, out_dim))

        def forward(self, x):  # models.py:20-21
            return self.net(x)

    return _MLP().to(dtype)


def mlp_forward_from_state(state, x, dtype=torch.float64, act="selu"):
    """models.py:20-21 evaluated from a state_dict in ``dtype`` (float64 gate), on the device of ``x``.
    ``act="silu"``: the SiLU variant of the MLP (the library's ACT_SILU)."""
    f = {"selu": torch.nn.functional.selu, "silu": torch.nn.functional.silu}[act]
    h = x.to(dtype)
    for li in (0, 2, 4, 6):
        W = state[f"net.{li}.weight"].to(device=h.device, dtype=dtype)
        b = state[f"net.{li}.bias"].to(device=h.device, dtype=dtype)
        h = h @ W.T + b
        if li != 6:
            h = f(h)
    return h


def wrapped_forward(model, t, x):
    """utils.py:51-52."""
    return model(torch.cat([x, t.repeat(x.shape[0])[:, None]], 1))


# ---- Dormand-Prince 5(4) tableau (standard; torchdyn DormandPrince45) ----------
_C = (0.0, 1 / 5, 3 / 10, 4 / 5, 8 / 9, 1.0, 1.0)
_A = (
    (),
    (1 / 5,),
    (3 / 40, 9 / 40),
    (44 / 45, -56 / 15, 32 / 9),
    (19372 / 6561, -25360 / 2187, 64448 / 6561, -212 / 729),
    (9017 / 3168, -355 / 33, 46732 / 5247, 49 / 176, -5103 / 18656),
    (35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84),
)
_B5 = (35 / 384, 0.0, 500 / 1113, 125 / 192, -2187 / 6784, 11 / 84, 0.0)
_BERR = (35 / 384 - 1951 / 21600, 0.0, 500 / 1113 - 22642 / 50085, 125 / 192 - 451 / 720,
         -2187 / 6784 + 12231 / 42400, 11 / 84 - 649 / 6300, -1.0 / 60.0)


def hairer_norm(z):
    """torchdyn numerics/utils.py::hairer_norm -- RMS over ALL elements."""
    return z.abs().pow(2).mean().sqrt()


def init_step(f, f0, x0, t0, order, atol, rtol):
    """torchdyn numerics/utils.py::init_step (Hairer's starting step)."""
    scale = atol + torch.abs(x0) * rtol
    d0, d1 = hairer_norm(x0 / scale), hairer_norm(f0 / scale)
    if d0 < 1e-5 or d1 < 1e-5:
        h0 = torch.tensor(1e-6, dtype=x0.dtype, device=x0.device)
    else:
        h0 = 0.01 * d0 / d1
    x_new = x0 + h0 * f0
    f_new = f(t0 + h0, x_new)
    d2 = hairer_norm((f_new - f0) / scale) / h0
    if d1 <= 1e-15 and d2 <= 1e-15:
        h1 = torch.max(torch.tensor(1e-6, dtype=x0.dtype, device=x0.device), h0 * 1e-3)
    else:
        h1 = (0.01 / max(d1, d2)) ** (1.0 / float(order + 1))
    return torch.min(100 * h0, h1).to(t0)


def adapt_step(dt, error_ratio, safety, min_factor, max_factor, order):
    """torchdyn numerics/utils.py::adapt_step."""
    if error_ratio == 0:
        return dt * max_factor
    if error_ratio < 1:
        min_factor = torch.ones_like(dt)
    exponent = torch.tensor(order, dtype=dt.dtype, device=dt.device).reciprocal()
    factor = torch.min(torch.as_tensor(max_factor, dtype=dt.dtype),
                       torch.max(safety / error_ratio ** exponent,
                                 torch.as_tensor(min_factor, dtype=dt.dtype)))
    return dt * factor


def dopri5_step(f, x, t, dt, k1):
    """torchdyn DormandPrince45.step -- 6 new stages, FSAL k7, 5th-order solution
    and embedded error estimate."""
    ks = [k1]
    for s in range(1, 7):
        xs = x
        for a, k in zip(_A[s], ks):
            if a != 0.0:
                xs = xs + dt * a * k
        ks.append(f(t + _C[s] * dt, xs))
    x_new = xs  # stage 7 argument IS the 5th-order solution (FSAL)
    err = dt * sum(b * k for b, k in zip(_BERR, ks) if b != 0.0)
    return x_new, err, ks[6]


@torch.no_grad()
def dopri5_trajectory(f, x, t_span, atol=1e-4, rtol=1e-4, record=None):
    """torchdyn odeint(..., solver='dopri5') without interpolator: adaptive
    lock-step over the batch, ONE scalar step size (global RMS error norm), every
    t_span entry hit exactly by clipping dt.  Returns (traj, stats).

    ``record``: an optional list; every step attempt appends a dict with the ``t`` it
    started from, the ``dt`` it took (after clipping), its error ``ratio``, whether it
    was ``accepted`` and whether it was ``clipped`` onto a checkpoint (``ckpt_flag``).
    The integration itself does not depend on it."""
    t_span = t_span.to(x)
    t, T = t_span[0], t_span[-1]
    k1 = f(t, x)
    nfe = 1
    dt = init_step(f, k1, x, t, 5, atol, rtol)
    nfe += 1
    sol = [x]
    ckpt = 1
    n_acc = n_rej = 0
    dt_old = None
    ckpt_flag = False
    while t < T:
        if t + dt > T:
            dt = T - t
        if ckpt < len(t_span) and t + dt > t_span[ckpt]:
            # no interpolator: remember dt, land exactly on the checkpoint
            dt_old, ckpt_flag = dt, True
            dt = t_span[ckpt] - t
        x_new, err, k7 = dopri5_step(f, x, t, dt, k1)
        nfe += 6
        tol = atol + rtol * torch.max(x.abs(), x_new.abs())
        ratio = hairer_norm(err / tol)
        accept = bool(ratio <= 1)
        if record is not None:
            record.append({"t": float(t), "dt": float(dt), "ratio": float(ratio), "accepted": accept,
                           "clipped": ckpt_flag})
        if accept:
            if ckpt < len(t_span) and t + dt == t_span[ckpt]:
                sol.append(x_new)
                ckpt += 1
            t, x, k1 = t + dt, x_new, k7
            n_acc += 1
        else:
            n_rej += 1
        if ckpt_flag:  # torchdyn resets dt whether or not the clipped step was accepted
            dt = dt_old - dt
            ckpt_flag = False
        dt = adapt_step(dt, ratio, 0.9, 0.2, 10.0, 5)
    return torch.stack(sol), {"nfe": nfe, "accepted": n_acc, "rejected": n_rej}


@torch.no_grad()
def euler_trajectory(f, x, t_span):
    """torchdyn fixed-step Euler over t_span (solver='euler')."""
    t_span = t_span.to(x)
    sol = [x]
    for a, b in zip(t_span[:-1], t_span[1:]):
        x = x + (b - a) * f(a, x)
        sol.append(x)
    return torch.stack(sol)
