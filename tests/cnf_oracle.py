"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the exact-likelihood (CNF) sampling path, built on
oracle/vector_field.py (which it uses unchanged).

* ``cnf_field``: the tutorial's exact CNF field (examples/2D_tutorials/Maximum_likelihood_CNF_tutorial.ipynb,
  ``cnf_wrapper(model, "exact")``) on a plain torch model: d/dt [x, ll] = [f(t, x), tr(df/dx)] with the trace from
  ``torch.func.jacrev`` + ``vmap`` per row; float64 when the model is.
* ``dopri5_any_direction`` / ``euler_any_direction``: torchdyn's odeint handling of the span direction.  For a
  decreasing span (t_span[1] < t_span[0]) torchdyn integrates f_(s, x) = -f(-s, x) over s = -t_span.  Restated
  from torchdyn's published source like the rest of oracle/vector_field.py; PARITY UNPINNED.
* ``positive_selu_mlp``: an MLP whose hidden pre-activations stay positive on a bounded region, so SELU is linear
  there and the field is affine with the constant trace tr(A), A = lambda^3 W3 W2 W1 W0x.
"""
import torch

from oracle import vector_field as vf

SELU_SCALE = 1.0507009873554804934193349852946


def cnf_field(model):
    def f(t, z):
        t = t.reshape(())
        x = z[:, :-1]

        def u(y):
            return model(torch.cat([y, t[None]]))

        div = torch.vmap(lambda y: torch.trace(torch.func.jacrev(u)(y)))(x)
        dx = model(torch.cat([x, t.repeat(x.shape[0])[:, None]], 1))
        return torch.cat([dx, div[:, None]], 1)

    return f


def _reversed(f):
    return lambda s, z: -f(-s, z)


def dopri5_any_direction(f, x, t_span, atol=1e-4, rtol=1e-4, record=None):
    """(traj, stats) of torchdyn's dopri5 over ``t_span`` in either direction.  ``record``: see
    ``oracle.vector_field.dopri5_trajectory``; for a decreasing span its times are those of the reversed run, -t."""
    if t_span[1] < t_span[0]:
        return vf.dopri5_trajectory(_reversed(f), x, -t_span, atol, rtol, record=record)
    return vf.dopri5_trajectory(f, x, t_span, atol, rtol, record=record)


def euler_any_direction(f, x, t_span):
    if t_span[1] < t_span[0]:
        return vf.euler_trajectory(_reversed(f), x, -t_span)
    return vf.euler_trajectory(f, x, t_span)


def positive_selu_mlp(dim=2, w=64, seed=0, dtype=torch.float64):
    """oracle MLP (time-varying) with large positive biases, small first-layer x weights and non-negative hidden
    weights: for |x| <= ~10 and t in [0, 1] every hidden pre-activation is positive."""
    g = torch.Generator().manual_seed(seed)
    m = vf.make_mlp(dim, w=w, time_varying=True, dtype=dtype)
    with torch.no_grad():
        m.net[0].weight.copy_(0.05 * torch.randn(w, dim + 1, generator=g))
        m.net[0].bias.copy_(3.0 + torch.rand(w, generator=g))
        for li in (2, 4):
            m.net[li].weight.copy_(0.05 * torch.rand(w, w, generator=g))
            m.net[li].bias.copy_(0.5 + torch.rand(w, generator=g))
        m.net[6].weight.copy_(0.1 * torch.randn(dim, w, generator=g))
        m.net[6].bias.copy_(0.1 * torch.randn(dim, generator=g))
    return m


def affine_trace(m, dim):
    """tr(A), A = lambda^3 W3 W2 W1 W0x, in float64: the divergence of ``m`` where SELU is linear."""
    W = [m.net[li].weight.detach().double() for li in (0, 2, 4, 6)]
    A = SELU_SCALE ** 3 * (W[3] @ W[2] @ W[1] @ W[0][:, :dim])
    return float(torch.trace(A))


def recording(f, seen):
    """``f`` that appends every (t, z) it is evaluated at to ``seen``."""
    def g(t, z):
        seen.append((t.detach().clone(), z.detach().clone()))
        return f(t, z)

    return g


def min_preactivation(m, seen):
    """Smallest hidden pre-activation of ``m`` (float64) over the recorded (t, [x, ll]) evaluation points."""
    low = float("inf")
    with torch.no_grad():
        for t, z in seen:
            h = torch.cat([z[:, :-1], t.reshape(()).repeat(z.shape[0])[:, None]], 1).double()
            for li in (0, 2, 4):
                lin = m.net[li]
                h = h @ lin.weight.double().T + lin.bias.double()
                low = min(low, float(h.min()))
                h = torch.nn.functional.selu(h)
    return low
