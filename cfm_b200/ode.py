"""Lock-step ODE sampling driver: drop-in for the way the reference uses torchdyn,

    node = NeuralODE(torch_wrapper(model), solver="dopri5", sensitivity="adjoint",
                     atol=1e-4, rtol=1e-4)
    traj = node.trajectory(x, t_span=torch.linspace(0, 1, 100))

(examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb:332-338;
examples/images/mnist_example.ipynb:67,126-128).  torchdyn is an un-vendored dependency
(setup.py:13); its dopri5 semantics (ONE scalar step for the whole batch, global RMS error norm,
steps clipped to land on every ``t_span`` entry, Hairer initial step) are restated in
oracle/vector_field.py and implemented here with the step controller resident on the device
(csrc/rk.cu): one step = 6 x (stage-input kernel + fused MLP forward) + error norm + control +
commit, enqueued back to back; the host reads a 64-byte state struct once per step only to learn
whether the integration has finished.

Only the hot path the north_star names is accelerated: the vector field must be a
``cfm_b200.models.MLP`` (optionally inside ``torch_wrapper``) on a CUDA device; anything else
raises -- there is no eager fallback.  ``cnf_wrapper(MLP(time_varying=True), "exact")`` is accepted too: its
state carries the log-density column, and the whole trajectory, trace included, runs in the one-launch kernel
(csrc/ode_small.cu, CNF variant).  ``cnf_wrapper(MLP(time_varying=True), "hutch_gaussian" | "hutch_rademacher")``
is accepted for models in the tensor-core class (B >= 128, dim >= 32, dim and w multiples of 8, w >= 32,
out_dim == dim; e.g. the MNIST model): Hutchinson's eps . (J eps) with one device-drawn probe per evaluation
(csrc/cnf_tc.cu), Euler with a captured step or dopri5 on the flat [x, ll] state.  So is
``torch_wrapper(GradModel(MLP(time_varying=True, out_dim=1)))``, the action-matching field grad_x s(t, x): small
actions (w in {32, 64}, dim <= 8) in the gradient variant of the one-launch kernel, actions in the tensor-core class
(B >= 128, dim >= 32, dim and w multiples of 8, w >= 32; e.g. the MNIST shape) as a forward and a reverse pass of
fp16x3 GEMMs (csrc/grad_tc.cu), Euler with a captured step or dopri5.

A decreasing ``t_span`` is integrated as torchdyn does: dopri5 runs the field f_(s, x) = -f(-s, x) over
s = -t_span (for the MLP only a different weight set, ``MLP._time_reversed``), because the step controller
only steps forwards.  For an action s the same weight set gives -s(-t, x), whose gradient is the reversed field.
Euler needs no such step: a negative step already gives the same bits.

Everything here runs without autograd, except one case: the ``cnf_wrapper(mlp, "exact")`` trajectory with autograd
enabled and ``x`` or a parameter of ``mlp`` requiring grad is attached to the graph (the forward is the same launch
with the same bits).  For ``solver="euler"`` and ``mlp`` in the backward class -- ``MLP(time_varying=True)``, w in
{32, 64}, dim <= 8, out_dim == dim, SELU or SiLU, a batch the backward plans -- ``backward()`` gives the exact gradient
of the computed fp32 Euler trajectory (torchdyn's ``sensitivity="autograd"``; it is returned for
``sensitivity="adjoint"`` too, whose continuous adjoint differs by O(h)) for the eight parameters and ``x``, in one
launch of csrc/cnf_train.cu.  Outside the class (dopri5, w = 128, larger batches) ``backward()`` raises
``NotImplementedError`` with the reason.  ``t_span`` requiring grad raises ``ValueError``: there are no time gradients.
"""
import ctypes as C

import torch
from torch.autograd.function import once_differentiable

from . import _ffi
from .models import MLP, GradModel, cnf_wrapper, torch_wrapper


def _unwrap(vf):
    m = vf.model if isinstance(vf, torch_wrapper) else vf
    if not isinstance(m, MLP) or not m.time_varying:
        raise TypeError("cfm_b200.NeuralODE accelerates cfm_b200.models.MLP(time_varying=True) "
                        "vector fields (optionally wrapped in torch_wrapper); got "
                        f"{type(m).__name__}")
    return m


def _unwrap_cnf(vf):
    m = vf.model
    if not isinstance(m, MLP) or not m.time_varying:
        raise TypeError("cfm_b200.NeuralODE accelerates cnf_wrapper(cfm_b200.models.MLP(time_varying=True)); got "
                        f"cnf_wrapper({type(m).__name__})")
    return m


_HUTCH = {"hutch_gaussian": _ffi.HUTCH_GAUSSIAN, "hutch_rademacher": _ffi.HUTCH_RADEMACHER}


def _hutch_refusal(vf, mlp, x):
    """Raise unless the Hutchinson field of ``cnf_wrapper(mlp)`` on the state ``x`` runs on the tensor cores.  Decided
    from the shapes alone, before any device check."""
    B = x.shape[0] if torch.is_tensor(x) and x.dim() == 2 else 0
    if not (mlp.out_dim == mlp.dim and mlp.act in (_ffi.ACT_SELU, _ffi.ACT_SILU) and 0 < B < 2**31
            and _ffi.lib().cfm_cnf_tc_supported(B, mlp.dim, mlp.w)):
        raise NotImplementedError(
            f"cnf_wrapper(likelihood_estimator={vf.likelihood_estimator!r}): the Hutchinson estimators run on the "
            "tensor cores for MLP(dim, w, time_varying=True) with out_dim == dim, SELU or SiLU, in the tensor-core "
            f"class (B >= 128, dim >= 32, dim and w multiples of 8, w >= 32); got B={B}, dim={mlp.dim}, w={mlp.w}, "
            f"out_dim={mlp.out_dim}.  For dim <= 8 use likelihood_estimator='exact': the exact trace costs only dim "
            "tangents there and has no variance")


def _grad_model(vf):
    """The GradModel inside ``torch_wrapper(GradModel(...))`` (or a bare one), else None."""
    m = vf.model if isinstance(vf, torch_wrapper) else vf
    return m if isinstance(m, GradModel) else None


def _unwrap_grad(gm):
    a = gm.action
    if not isinstance(a, MLP):
        raise TypeError("cfm_b200.NeuralODE accelerates torch_wrapper(GradModel(cfm_b200.models.MLP(time_varying=True, "
                        f"out_dim=1))); got GradModel({type(a).__name__})")
    if a.out_dim != 1 or not a.time_varying:
        raise NotImplementedError(
            f"GradModel: no gradient-field kernel for an action MLP with out_dim={a.out_dim}, "
            f"time_varying={a.time_varying} (it takes a scalar action, out_dim == 1, with time_varying=True)")
    return a


def _decreasing(t_span):
    return t_span.numel() >= 2 and bool(t_span[1] < t_span[0])


def _rk_stats(cur, **extra):
    """``NeuralODE.stats`` from the controller state (``_ffi.RkState``) a device run left."""
    return {"nfe": cur.nfe, "accepted": cur.accepted, "rejected": cur.rejected, "t": cur.t,
            "last_ratio": cur.ratio, **extra}


class NeuralODE(torch.nn.Module):
    """Subset of torchdyn.core.NeuralODE used by the reference examples.  ``forward`` returns ``(t_span, traj)``.

    Trajectories are detached, except those of ``cnf_wrapper(mlp, "exact")`` under autograd, which the maximum-likelihood
    tutorial trains through: with ``solver="euler"`` and ``mlp`` in the backward class (see the module docstring)
    gradients reach ``mlp``'s parameters and the initial state; otherwise ``backward()`` raises
    ``NotImplementedError``."""

    def __init__(self, vector_field, solver="dopri5", sensitivity="adjoint", atol=1e-4, rtol=1e-4,
                 **unused):
        super().__init__()
        self.vf = vector_field
        if solver not in ("dopri5", "euler"):
            raise NotImplementedError(f"solver {solver!r}: the CUDA driver provides 'dopri5' and 'euler'")
        self.solver, self.atol, self.rtol = solver, float(atol), float(rtol)
        self.sensitivity = sensitivity  # kept for API parity: cnf_wrapper gradients are the discrete (autograd) ones
        self.stats = {}
        self.use_cuda_graph = True  # replay one captured dopri5 step per iteration
        self.max_burst = 32         # steps enqueued between two host reads of the controller state
        self.min_burst = 4          # ... at least this many: a step enqueued after the end is 15 empty launches (every
                                    # kernel, the fused MLP included, checks the device-side `done` flag), cheaper
                                    # than a host round trip per step
        self.use_fused_small = True  # small MLPs: the whole trajectory in one launch (csrc/ode_small.cu)
        # Row-sharded integration across ranks (cfm_b200.dist.sharded_trajectory(..., lockstep=True)): a
        # torch.distributed group (or True for the default group).  torchdyn's controller uses ONE error norm
        # over the whole batch; with the batch split over ranks, the per-shard sums of squares (one float64
        # per step attempt, three more for the initial step) are all-reduced so that every rank takes exactly
        # the step sequence a single process would take on the full batch.
        self.lockstep = None
        self._plans = {}
        self._cnf_plans = {}  # Hutchinson Euler: plan key -> buffers and the captured step graph
        self._grad_plans = {}  # tensor-core gradient-field Euler, likewise

    def forward(self, x, t_span):
        traj = self.trajectory(x, t_span)
        with torch.no_grad():
            return t_span.to(x.device), traj

    def trajectory(self, x, t_span):
        """(n_span, *x.shape) states at the ``t_span`` points.  Detached, except for ``cnf_wrapper(mlp, "exact")``
        under autograd when ``x`` or a parameter of ``mlp`` requires grad: then the trajectory is on the graph.
        With ``solver="euler"`` and ``mlp`` in the backward class (``cfm_ode_small_cnf_backward_supported``: w in
        {32, 64}, dim <= 8, out_dim == dim, SELU or SiLU) ``backward()`` computes the exact gradient of the computed
        fp32 Euler trajectory in one launch, whatever ``sensitivity`` says; outside the class it raises
        ``NotImplementedError`` with the reason.  The forward is the same launch with the same bits either way."""
        if isinstance(self.vf, cnf_wrapper) and self.vf.eps_fn is not None:
            _hutch_refusal(self.vf, _unwrap_cnf(self.vf), x)
        if isinstance(self.vf, cnf_wrapper) and torch.is_grad_enabled():
            mlp = _unwrap_cnf(self.vf)
            params = list(mlp.parameters())
            if torch.is_tensor(x) and (x.requires_grad or any(p.requires_grad for p in params)):
                if torch.is_tensor(t_span) and t_span.requires_grad:
                    raise ValueError("cnf_wrapper: t_span requires grad, but gradients flow to the state and the "
                                     "model's parameters only; detach it")
                reason = self._cnf_backward_gap(mlp, x)
                if reason is None:
                    return _CnfEulerTrajectory.apply(self, mlp, x, t_span, *params)
                return _NoBackward.apply(reason, lambda: self._trajectory(x, t_span), x, *params)
        with torch.no_grad():
            return self._trajectory(x, t_span)

    def _cnf_backward_gap(self, mlp, x):
        """Why backward() through this cnf_wrapper trajectory is not implemented, or None when it is."""
        if self.vf.eps_fn is not None:
            return (f"gradients through the Hutchinson-estimator trajectory (likelihood_estimator="
                    f"{self.vf.likelihood_estimator!r}) are not implemented; the device path samples it only")
        if self.solver != "euler":
            return (f"gradients through the adaptive {self.solver} solve are not implemented; use solver='euler'")
        B = x.shape[0] if x.dim() == 2 else 0
        if not (mlp.w in (32, 64) and 1 <= mlp.dim <= 8 and mlp.out_dim == mlp.dim
                and mlp.act in (_ffi.ACT_SELU, _ffi.ACT_SILU)
                and _ffi.lib().cfm_ode_small_cnf_backward_supported(B, mlp.dim, mlp.w)):
            return (f"gradients through the exact-likelihood trajectory are not implemented for B={B}, "
                    f"dim={mlp.dim}, w={mlp.w}, out_dim={mlp.out_dim}; the backward kernel takes w in {{32, 64}}, "
                    "dim <= 8, out_dim == dim, SELU or SiLU and the batches cfm_ode_small_cnf_backward_supported "
                    "accepts")
        return None

    def _trajectory(self, x, t_span):
        cnf = isinstance(self.vf, cnf_wrapper)
        gm = None if cnf else _grad_model(self.vf)
        mlp = _unwrap_cnf(self.vf) if cnf else _unwrap_grad(gm) if gm is not None else _unwrap(self.vf)
        if not x.is_cuda:
            raise _ffi.CfmLibraryError("NeuralODE.trajectory needs CUDA inputs (no CPU fallback)")
        dev = x.device
        t_span = torch.as_tensor(t_span, dtype=torch.float32)
        reverse = self.solver == "dopri5" and _decreasing(t_span)  # see the module docstring
        kw = {}
        if cnf and self.vf.eps_fn is not None:
            # the Hutchinson probes' seed, one per call from torch's default CPU generator, drawn first: building the
            # time-reversed net below initialises a module, which draws from the same generator on its first use
            kw["seed"] = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
        with torch.cuda.device(dev):  # the library launches on the CURRENT device: make it the tensors' one
            if reverse:
                mlp, t_span = mlp._time_reversed(), -t_span
            run = (self._cnf_trajectory_on if cnf else self._grad_trajectory_on if gm is not None
                   else self._trajectory_on)
            out = run(mlp, x, t_span, dev, **kw)
        if reverse:
            self.stats["t"] = -self.stats["t"]
        return out

    def _trajectory_on(self, mlp, x, t_span, dev):
        shape = x.shape
        x0 = x.detach().reshape(shape[0], -1).float().contiguous()
        if self.lockstep is not None and self.solver != "dopri5":
            raise NotImplementedError("lock-step sharding applies to the adaptive solver (dopri5)")
        if self.lockstep is None and self.use_fused_small and t_span.numel() >= 2 \
                and _ffi.lib().cfm_ode_small_supported(x0.shape[0], x0.shape[1], mlp.w, mlp.out_dim):
            out = self._fused_small(mlp, x0, t_span.to(dev).contiguous())
        elif self.solver == "euler":
            out = self._euler(mlp, x0, t_span)
        else:
            # the span stays on the host (where callers build it): the plan keeps a device copy and refreshes it only
            # when the values change, so a repeated call neither uploads nor reads back anything before the first kernel
            out = self._dopri5(mlp, x0, t_span.detach().cpu().contiguous())
        return out.reshape(out.shape[0], *shape)

    def _cnf_trajectory_on(self, mlp, x, t_span, dev, seed=None):
        """cnf_wrapper(mlp, "exact"): the state [x, ll] goes through the CNF variant of the one-launch kernel."""
        if self.lockstep is not None:
            raise NotImplementedError("cnf_wrapper: lock-step sharding is not supported; the exact-likelihood path "
                                      "integrates the whole batch in one single-device kernel")
        if x.dim() != 2 or x.shape[1] != mlp.dim + 1:
            raise ValueError(f"cnf_wrapper: expected a state of shape (B, {mlp.dim + 1}) (x and the log-density "
                             f"column), got {tuple(x.shape)}")
        if t_span.numel() < 2:
            raise ValueError("cnf_wrapper: t_span needs at least two points")
        if self.vf.eps_fn is not None:
            _hutch_refusal(self.vf, mlp, x)
            return self._hutch_trajectory(mlp, x.detach().float().contiguous(), t_span, dev, seed)
        if mlp.out_dim != mlp.dim or not _ffi.lib().cfm_ode_small_cnf_supported(x.shape[0], mlp.dim, mlp.w):
            raise NotImplementedError(
                f"cnf_wrapper: no exact-likelihood kernel for B={x.shape[0]}, dim={mlp.dim}, w={mlp.w}, "
                f"out_dim={mlp.out_dim} (it takes w in {{32, 64, 128}}, dim <= 8, out_dim == dim and batches whose "
                "state fits in shared memory); models in the tensor-core class (B >= 128, dim >= 32, dim and w "
                "multiples of 8, w >= 32) take likelihood_estimator='hutch_gaussian' or 'hutch_rademacher'")
        return self._fused_small(mlp, x.detach().float().contiguous(), t_span.to(dev).contiguous(), cnf=True)

    def _hutch_trajectory(self, mlp, z, t_span, dev, seed):
        """cnf_wrapper(mlp, "hutch_*") in the tensor-core class (csrc/cnf_tc.cu): the field is [f, eps . (J eps)] with
        one fresh probe per evaluation, keyed by ``seed`` (drawn by ``_trajectory``)."""
        est = self.vf.likelihood_estimator
        if self.solver == "euler":
            return self._hutch_euler(mlp, z, t_span.to(dev).contiguous(), est, seed)
        B, D = z.shape[0], mlp.dim
        flat = torch.cat([z[:, :D].reshape(-1), z[:, D]])  # the x block [B][D], then the ll block [B]
        return self._dopri5(mlp, flat, t_span.detach().cpu().contiguous(), cnf=(est, seed, B, D))

    def _hutch_euler(self, mlp, z, t_span, est, seed):
        """Euler over ``t_span`` (fp32 on the device): init, then per step the ten launches of one field evaluation and
        the step kernel, captured once as a CUDA graph per plan and replayed."""
        L = _ffi.lib()
        dev = z.device
        B, D, n_span = z.shape[0], mlp.dim, t_span.numel()
        blob = mlp._prepared(True, dev)
        key = (id(mlp), B, D, str(dev), mlp._weights_key(), blob.data_ptr(), mlp.act, est,
               torch.cuda.current_stream(dev).cuda_stream)
        P = self._cnf_plans.get(key)
        if P is None:
            self._cnf_plans.clear()  # one live plan: a new shape / new weights retire the old graph
            f32 = dict(dtype=torch.float32, device=dev)
            st = torch.zeros(C.sizeof(_ffi.CnfTcState), dtype=torch.uint8, device=dev)
            P = {"blob": blob, "st": st, "x": torch.empty((B, D), **f32), "ll": torch.empty(B, **f32),
                 "f": torch.empty((B, D), **f32), "div": torch.empty(B, **f32),
                 "hi": torch.empty((B, D), dtype=torch.float16, device=dev),
                 "lo": torch.empty((B, D), dtype=torch.float16, device=dev),
                 "ws": _ffi.workspace(L.cfm_cnf_tc_workspace_bytes(B, D, mlp.w), dev), "graph": None}
            self._cnf_plans[key] = P
        st, ws = P["st"], P["ws"]
        at = lambda off: C.c_void_p(st.data_ptr() + off)  # noqa: E731

        def step():  # on the current stream, which is the capture stream inside torch.cuda.graph
            sp = _ffi.stream_ptr(dev)
            _ffi.check(L.cfm_cnf_tc_field_f32(
                _ffi.ptr(blob), None, _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]), B, D, mlp.w, mlp.act, _HUTCH[est],
                at(_ffi.CnfTcState.t.offset), at(_ffi.CnfTcState.seed.offset), at(_ffi.CnfTcState.n.offset), 0,
                _ffi.ptr(P["f"]), _ffi.ptr(P["div"]), _ffi.ptr(ws), ws.numel(), sp), "cfm_cnf_tc_field_f32")
            _ffi.check(L.cfm_cnf_tc_euler_step(_ffi.ptr(st), _ffi.ptr(P["x"]), _ffi.ptr(P["ll"]), _ffi.ptr(P["f"]),
                                               _ffi.ptr(P["div"]), _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]), B, D, sp),
                       "cfm_cnf_tc_euler_step")

        traj = torch.empty((n_span, B, D + 1), dtype=torch.float32, device=dev)
        P["span"] = t_span  # read through the state by every step: kept alive with the plan
        _ffi.check(L.cfm_cnf_tc_euler_init(_ffi.ptr(st), _ffi.ptr(z), _ffi.ptr(P["x"]), _ffi.ptr(P["ll"]),
                                           _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]), _ffi.ptr(traj), _ffi.ptr(t_span),
                                           n_span, seed, B, D, _ffi.stream_ptr(dev)), "cfm_cnf_tc_euler_init")
        _ffi.replay_steps(P, step, n_span - 1, self.use_cuda_graph)
        self.stats = {"nfe": n_span - 1, "accepted": n_span - 1, "rejected": 0,
                      "graph": self.use_cuda_graph and P["graph"] is not None}
        return traj

    def _grad_trajectory_on(self, mlp, x, t_span, dev):
        """torch_wrapper(GradModel(mlp)): the field grad_x mlp(t, x) through the gradient variant of the one-launch
        kernel (w in {32, 64}, dim <= 8) or, for actions in the tensor-core class, through the forward and reverse GEMMs
        of csrc/grad_tc.cu.  The two classes are disjoint (dim <= 8 against dim >= 32); any other shape raises before
        any launch."""
        if self.lockstep is not None:
            raise NotImplementedError("GradModel: lock-step sharding is not supported; the gradient-field path "
                                      "integrates the whole batch in one single-device kernel")
        if x.dim() != 2 or x.shape[1] != mlp.dim:
            raise ValueError(f"GradModel: expected a state of shape (B, {mlp.dim}), got {tuple(x.shape)}")
        if t_span.numel() < 2:
            raise ValueError("GradModel: t_span needs at least two points")
        L = _ffi.lib()
        B = x.shape[0]
        x0 = x.detach().float().contiguous()
        if L.cfm_ode_small_grad_supported(B, mlp.dim, mlp.w):
            return self._fused_small(mlp, x0, t_span.to(dev).contiguous(), grad=True)
        if not (B < 2**31 and mlp.act in (_ffi.ACT_SELU, _ffi.ACT_SILU) and L.cfm_grad_tc_supported(B, mlp.dim, mlp.w)):
            raise NotImplementedError(
                f"GradModel: no gradient-field kernel for B={B}, dim={mlp.dim}, w={mlp.w}: the one-launch kernel takes "
                "w in {32, 64}, dim <= 8 and batches whose state fits in shared memory; the tensor-core class takes "
                "B >= 128, dim >= 32, dim and w multiples of 8, w >= 32")
        if self.solver == "euler":
            return self._grad_tc_euler(mlp, x0, t_span.to(dev).contiguous())
        return self._dopri5(mlp, x0, t_span.detach().cpu().contiguous())

    def _grad_tc_euler(self, mlp, x, t_span):
        """Euler over ``t_span`` for an action in the tensor-core class (csrc/grad_tc.cu): init, then per step the six
        launches of one gradient-field evaluation and the step kernel, captured once as a CUDA graph per plan and
        replayed."""
        L = _ffi.lib()
        dev = x.device
        B, D, n_span = x.shape[0], mlp.dim, t_span.numel()
        blob, gblob = mlp._grad_prepared(dev)
        key = (id(mlp), B, D, str(dev), mlp._weights_key(), blob.data_ptr(), gblob.data_ptr(), mlp.act,
               torch.cuda.current_stream(dev).cuda_stream)
        P = self._grad_plans.get(key)
        if P is None:
            self._grad_plans.clear()  # one live plan: a new shape / new weights retire the old graph
            st = torch.zeros(C.sizeof(_ffi.GradTcState), dtype=torch.uint8, device=dev)
            P = {"st": st, "x": torch.empty((B, D), dtype=torch.float32, device=dev),
                 "v": torch.empty((B, D), dtype=torch.float32, device=dev),
                 "hi": torch.empty((B, D), dtype=torch.float16, device=dev),
                 "lo": torch.empty((B, D), dtype=torch.float16, device=dev),
                 "ws": _ffi.workspace(L.cfm_grad_tc_workspace_bytes(B, D, mlp.w), dev), "graph": None}
            self._grad_plans[key] = P
        st, ws = P["st"], P["ws"]
        t_at = C.c_void_p(st.data_ptr() + _ffi.GradTcState.t.offset)

        def step():  # on the current stream, which is the capture stream inside torch.cuda.graph
            sp = _ffi.stream_ptr(dev)
            _ffi.check(L.cfm_grad_tc_field_f32(
                _ffi.ptr(blob), _ffi.ptr(gblob), None, _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]), B, D, mlp.w, mlp.act,
                t_at, _ffi.ptr(P["v"]), _ffi.ptr(ws), ws.numel(), sp), "cfm_grad_tc_field_f32")
            _ffi.check(L.cfm_grad_tc_euler_step(_ffi.ptr(st), _ffi.ptr(P["x"]), _ffi.ptr(P["v"]), _ffi.ptr(P["hi"]),
                                                _ffi.ptr(P["lo"]), B, D, sp), "cfm_grad_tc_euler_step")

        traj = torch.empty((n_span, B, D), dtype=torch.float32, device=dev)
        P["span"] = t_span  # read through the state by every step: kept alive with the plan
        _ffi.check(L.cfm_grad_tc_euler_init(_ffi.ptr(st), _ffi.ptr(x), _ffi.ptr(P["x"]), _ffi.ptr(P["hi"]),
                                            _ffi.ptr(P["lo"]), _ffi.ptr(traj), _ffi.ptr(t_span), n_span, B, D,
                                            _ffi.stream_ptr(dev)), "cfm_grad_tc_euler_init")
        _ffi.replay_steps(P, step, n_span - 1, self.use_cuda_graph)
        self.stats = {"nfe": n_span - 1, "accepted": n_span - 1, "rejected": 0,
                      "graph": self.use_cuda_graph and P["graph"] is not None}
        return traj

    # ------------------------------------------------------------------------------------
    def _fused_small(self, mlp, x0, t_span, cnf=False, grad=False):
        """Launch-bound regime (the 2-D tutorial models): Hairer init, all dopri5 / euler steps, the
        error norms and the controller in ONE cooperative kernel; one host read at the end.  ``cnf``: x0 is the
        [x, ll] state of cnf_wrapper (mlp.dim + 1 columns) and the kernel also integrates the trace.  ``grad``: mlp is
        a scalar action and the field is its gradient in x."""
        L = _ffi.lib()
        dev = x0.device
        B, D = x0.shape  # D: state columns
        n_span = t_span.numel()
        ps = mlp._device_params(dev)
        traj = torch.empty((n_span, B, D), dtype=torch.float32, device=dev)
        st = torch.zeros(ctypes_sizeof_state(), dtype=torch.uint8, device=dev)
        dim = mlp.dim if cnf else D
        ws = _ffi.workspace(L.cfm_ode_small_workspace_bytes(B, dim, mlp.w), dev)
        name = "cfm_ode_small_" + ("cnf_" if cnf else "grad_" if grad else "") + "trajectory_f32"
        _ffi.check(getattr(L, name)(
            *[_ffi.ptr(p) for p in ps], dim, mlp.w, 1, mlp.act, _ffi.ptr(x0), B, _ffi.ptr(t_span), n_span,
            self.atol, self.rtol, 1 if self.solver == "euler" else 0, _ffi.ptr(traj), _ffi.ptr(st),
            _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(dev)), name)
        cur = _ffi.RkState.from_buffer_copy(bytes(st.cpu().numpy().tobytes()))
        if not cur.done:
            raise RuntimeError("dopri5: step budget exhausted")
        self.stats = _rk_stats(cur, graph=False, fused=True)
        return traj

    def _euler(self, mlp, x, t_span):
        L = _ffi.lib()
        ts = t_span.tolist()
        numel = x.numel()
        traj = torch.empty((len(ts),) + tuple(x.shape), dtype=torch.float32, device=x.device)
        traj[0].copy_(x)
        k = torch.empty_like(x)
        for n in range(len(ts) - 1):
            mlp.vector_field(ts[n], traj[n], out=k)
            _ffi.check(L.cfm_axpy_f32(_ffi.ptr(traj[n]), _ffi.ptr(k), ts[n + 1] - ts[n],
                                      _ffi.ptr(traj[n + 1]), numel, _ffi.stream_ptr(x.device)),
                       "cfm_axpy_f32")
        self.stats = {"nfe": len(ts) - 1, "accepted": len(ts) - 1, "rejected": 0}
        return traj

    # -- dopri5 -----------------------------------------------------------------------------
    def _enqueue_step(self, mlp, P):
        """One full dopri5 step, enqueued on the current stream without any host round trip."""
        L = _ffi.lib()
        sp = _ffi.stream_ptr(P["dev"])
        stp, x, xnew, xs, k, numel = P["stp"], P["x"], P["xnew"], P["xs"], P["k"], P["numel"]
        split = P["xs_hi"] is not None
        for stage in range(1, 7):
            out = xs if stage < 6 else xnew
            if split:
                # the stage input goes straight to the MLP as its fp16x3 (hi, lo) operand pair; only stage 6
                # (= xnew, needed by the error norm and the commit) is also kept in fp32
                _ffi.check(L.cfm_rk_stage_input(stp, _ffi.ptr(x), _ffi.ptr(k), _ffi.ptr(out if stage == 6 else None),
                                                _ffi.ptr(P["xs_hi"]), _ffi.ptr(P["xs_lo"]), _ffi.ptr(P["t_stage"]),
                                                _ffi.ptr(xs if stage == 6 else None),  # error partial -> xs (free here)
                                                numel, stage, sp), "cfm_rk_stage_input")
                P["field_split"](P["t_stage"], P["xs_hi"], P["xs_lo"], k[stage], P["done_flag"], stage - 1)
            else:
                _ffi.check(L.cfm_rk_stage_input(stp, _ffi.ptr(x), _ffi.ptr(k), _ffi.ptr(out), None, None,
                                                _ffi.ptr(P["t_stage"]), None, numel, stage, sp), "cfm_rk_stage_input")
                mlp.vector_field(P["t_stage"], out, out=k[stage])
        _ffi.check(L.cfm_rk_error_norm(stp, _ffi.ptr(x), _ffi.ptr(xnew), _ffi.ptr(k),
                                       _ffi.ptr(xs if split else None), numel, sp), "cfm_rk_error_norm")
        if P["group"] is not None:  # lock-step: the error norm is over the rows of ALL ranks
            P["dist"].all_reduce(P["err_acc"], group=P["group"])
        _ffi.check(L.cfm_rk_control(stp, _ffi.ptr(P["t_span"]), P["numel_global"], sp), "cfm_rk_control")
        _ffi.check(L.cfm_rk_commit(stp, _ffi.ptr(x), _ffi.ptr(xnew), _ffi.ptr(k), _ffi.ptr(P["traj"]),
                                   numel, sp), "cfm_rk_commit")

    def _plan(self, mlp, B, D, n_span, dev, cnf=None):
        """Persistent buffers (+ the captured step graph) for one problem shape and weight version.  ``cnf``: the
        Hutchinson estimator of a cnf_wrapper state, laid out flat as the x block [B][D] followed by the ll block [B]
        (numel = B (D + 1)); every cfm_rk_* kernel takes that layout unchanged."""
        grad = cnf is None and _grad_model(self.vf) is not None  # the action's gradient field (csrc/grad_tc.cu)
        key = (id(mlp), B, D, n_span, str(dev), mlp._weights_key(), mlp.mlp_algo, mlp.act, self.lockstep is not None,
               cnf, grad)
        P = self._plans.get(key)
        if P is not None:
            return P
        self._plans.clear()  # one live plan: a new shape / new weights retire the old graph
        st = torch.zeros(ctypes_sizeof_state(), dtype=torch.uint8, device=dev)
        numel = B * D if cnf is None else B * (D + 1)
        shape = (B, D) if cnf is None else (numel,)
        P = {"dev": dev, "numel": numel, "st": st, "stp": _ffi.ptr(st),
             "x": torch.empty(shape, dtype=torch.float32, device=dev),
             "xnew": torch.empty(shape, dtype=torch.float32, device=dev),
             "xs": torch.empty(shape, dtype=torch.float32, device=dev),
             "k": torch.empty((7, *shape), dtype=torch.float32, device=dev),
             "traj": torch.empty((n_span, *shape), dtype=torch.float32, device=dev),
             "t_span": torch.empty(n_span, dtype=torch.float32, device=dev),
             "t_stage": torch.zeros(1, dtype=torch.float32, device=dev),
             "scratch": torch.zeros(4, dtype=torch.float64, device=dev),
             "pinned": torch.empty(ctypes_sizeof_state(), dtype=torch.uint8, pin_memory=True),
             "pinned_init": torch.empty(ctypes_sizeof_state(), dtype=torch.uint8, pin_memory=True),
             "t0": torch.zeros(1, dtype=torch.float32, device=dev), "ts_host": None, "init_graph": None,
             "xs_hi": None, "xs_lo": None, "graph": None, "group": None, "dist": None, "numel_global": numel}
        off = _ffi.RkState.err_acc.offset  # the float64 accumulator inside the device state struct
        P["err_acc"] = st[off:off + 8].view(torch.float64)
        off = _ffi.RkState.done.offset  # int32: non-zero once t has reached t_end
        P["done_flag"] = st[off:off + 4].view(torch.int32)
        if cnf is not None or grad or mlp.tc_path(B):
            # stage inputs go to the MLP as its fp16x3 tensor-core operand pair (hi, lo), written by the RK kernel
            P["xs_hi"] = torch.empty(shape, dtype=torch.float16, device=dev)
            P["xs_lo"] = torch.empty(shape, dtype=torch.float16, device=dev)
        if grad:
            self._grad_fields(mlp, P, B, D)
        elif cnf is None:
            P["field"] = lambda t, x, out, n: mlp.vector_field(t, x, out=out)
            P["field_split"] = lambda t, hi, lo, out, skip, n: mlp.vector_field_split(t, hi, lo, out, skip_flag=skip)
        else:
            self._hutch_fields(mlp, P, B, D, cnf)
        self._plans[key] = P
        return P

    @staticmethod
    def _hutch_fields(mlp, P, B, D, est):
        """The plan's field launchers for the flat [x, ll] state: f into the first B D elements of ``out``, div into the
        last B.  The probe ordinal is the controller's ``nfe`` plus the evaluation's place in the init (0, 1) or the
        step (stage - 1), read on the device, and the seed is the plan's device word."""
        L = _ffi.lib()
        dev = P["dev"]
        blob = mlp._prepared(True, dev)
        ws = _ffi.workspace(L.cfm_cnf_tc_workspace_bytes(B, D, mlp.w), dev)
        P["blob"], P["cnf_ws"] = blob, ws
        P["seed"] = torch.zeros(1, dtype=torch.int64, device=dev)
        nfe = C.c_void_p(P["st"].data_ptr() + _ffi.RkState.nfe.offset)

        def field(t, x, out, n, hi=None, lo=None):
            _ffi.check(L.cfm_cnf_tc_field_f32(
                _ffi.ptr(blob), _ffi.ptr(x), _ffi.ptr(hi), _ffi.ptr(lo), B, D, mlp.w, mlp.act, _HUTCH[est], _ffi.ptr(t),
                _ffi.ptr(P["seed"]), nfe, n, _ffi.ptr(out), C.c_void_p(out.data_ptr() + 4 * B * D), _ffi.ptr(ws),
                ws.numel(), _ffi.stream_ptr(dev)), "cfm_cnf_tc_field_f32")

        P["field"] = field
        P["field_split"] = lambda t, hi, lo, out, skip, n: field(t, None, out, n, hi, lo)

    @staticmethod
    def _grad_fields(mlp, P, B, D):
        """The plan's field launchers for the gradient field of the action ``mlp`` in the tensor-core class: v into
        ``out`` (row stride D, any 4-byte offset), from fp32 x or from the stage kernel's operand pair."""
        L = _ffi.lib()
        dev = P["dev"]
        blob, gblob = mlp._grad_prepared(dev)
        ws = _ffi.workspace(L.cfm_grad_tc_workspace_bytes(B, D, mlp.w), dev)
        P["blob"], P["grad_blob"], P["grad_ws"] = blob, gblob, ws

        def field(t, x, out, n, hi=None, lo=None):
            _ffi.check(L.cfm_grad_tc_field_f32(
                _ffi.ptr(blob), _ffi.ptr(gblob), _ffi.ptr(x), _ffi.ptr(hi), _ffi.ptr(lo), B, D, mlp.w, mlp.act,
                _ffi.ptr(t), _ffi.ptr(out), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(dev)), "cfm_grad_tc_field_f32")

        P["field"] = field
        P["field_split"] = lambda t, hi, lo, out, skip, n: field(t, None, out, n, hi, lo)

    def _enqueue_init(self, mlp, P, lock):
        """k1 = f(t0, x) and the Hairer initial step (one extra evaluation), enqueued without a host round trip."""
        L = _ffi.lib()
        sp = _ffi.stream_ptr(P["dev"])
        stp, x, xs, k, numel, ng = P["stp"], P["x"], P["xs"], P["k"], P["numel"], P["numel_global"]
        P["field"](P["t0"], x, k[0], 0)
        _ffi.check(L.cfm_rk_init_sums(stp, _ffi.ptr(x), _ffi.ptr(k[0]), None, _ffi.ptr(P["scratch"]), numel, 0, sp),
                   "cfm_rk_init_sums")
        if lock:
            P["dist"].all_reduce(P["scratch"], group=P["group"])
        _ffi.check(L.cfm_rk_init_probe(stp, _ffi.ptr(x), _ffi.ptr(k[0]), _ffi.ptr(xs), _ffi.ptr(P["t_stage"]),
                                       _ffi.ptr(P["scratch"]), numel, ng, sp), "cfm_rk_init_probe")
        P["field"](P["t_stage"], xs, k[1], 1)
        if lock:  # phase 1 adds into scratch[2] only; keep the already-global scratch[0:2] out of the second reduce
            P["scratch"][2:].zero_()
        _ffi.check(L.cfm_rk_init_sums(stp, _ffi.ptr(x), _ffi.ptr(k[0]), _ffi.ptr(k[1]), _ffi.ptr(P["scratch"]),
                                      numel, 1, sp), "cfm_rk_init_sums")
        if lock:
            P["dist"].all_reduce(P["scratch"][2:3], group=P["group"])
        _ffi.check(L.cfm_rk_init_finish(stp, _ffi.ptr(P["t_span"]), _ffi.ptr(P["scratch"]), ng, sp),
                   "cfm_rk_init_finish")

    def _dopri5(self, mlp, x0, ts_host, cnf=None):
        """``ts_host``: the span as a contiguous fp32 CPU tensor.  ``cnf``: (estimator, seed, B, D) of a Hutchinson
        cnf_wrapper state, ``x0`` then being its flat layout (see ``_plan``); the result is (n_span, B, D + 1)."""
        dev = x0.device
        B, D = x0.shape if cnf is None else cnf[2:]
        numel = x0.numel()
        n_span = ts_host.numel()
        P = self._plan(mlp, B, D, n_span, dev, None if cnf is None else cnf[0])
        if cnf is not None:
            P["seed"].fill_(cnf[1])
        x, traj, st = P["x"], P["traj"], P["st"]
        x.copy_(x0)
        traj[0].copy_(x0)
        if P["ts_host"] is None or not torch.equal(P["ts_host"], ts_host):
            P["t_span"].copy_(ts_host)
            P["t0"].copy_(ts_host[:1])
            P["ts_host"] = ts_host.clone()

        st_host = _ffi.RkState()
        st_host.t, st_host.t_end = float(ts_host[0]), float(ts_host[-1])
        st_host.atol, st_host.rtol = self.atol, self.rtol
        st_host.n_span, st_host.ckpt, st_host.save_slot = n_span, 1, -1
        # pinned staging (the previous call ended with a stream synchronize, so the buffer is free): no pageable copy
        P["pinned_init"].copy_(torch.frombuffer(bytearray(bytes(st_host)), dtype=torch.uint8))
        st.copy_(P["pinned_init"], non_blocking=True)

        lock = self.lockstep is not None
        if lock:
            import torch.distributed as tdist
            P["dist"] = tdist
            P["group"] = None if self.lockstep is True else self.lockstep
            if not (tdist.is_available() and tdist.is_initialized()):
                raise RuntimeError("NeuralODE.lockstep needs an initialised torch.distributed process group")
            cnt = torch.tensor([numel], dtype=torch.int64, device=dev)
            tdist.all_reduce(cnt, group=P["group"])
            P["numel_global"] = int(cnt.item())
            P["group"] = P["group"] if P["group"] is not None else tdist.group.WORLD
        else:
            P["group"], P["numel_global"] = None, numel
        if P["init_graph"] is not None and not lock:
            P["init_graph"].replay()
        else:
            self._enqueue_init(mlp, P, lock)

        if self.use_cuda_graph and not lock and P["graph"] is None:
            # the step is a fixed kernel sequence whose control flow lives in device memory: capture it
            # once (the eager init above has already loaded every kernel) and replay it per step
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._enqueue_step(mlp, P)
            P["graph"] = g
            gi = torch.cuda.CUDAGraph()  # the initial-step sequence (2 MLP evaluations + 4 small kernels) likewise
            with torch.cuda.graph(gi):
                self._enqueue_init(mlp, P, False)
            P["init_graph"] = gi

        pinned = P["pinned"]
        max_steps = 100000
        steps = 0
        cur = st_host
        while steps < max_steps:
            # Steps are enqueued in bursts between host reads of the state.  Every t_span point still to
            # be recorded costs at least one accepted step (the controller clips dt onto it), so that
            # many steps can be enqueued without looking; a step enqueued after t_end is a no-op on the
            # device (done flag), so the bound only has to be safe, not tight.
            burst = max(1 if lock else self.min_burst, min(self.max_burst, n_span - int(cur.ckpt)))
            if not lock and steps == 0 and P.get("last_steps"):
                # the previous trajectory of this plan (same model, same span, same batch shape) is the best predictor
                # of the step count: enqueue exactly that many, then look; a wrong guess costs one more round trip
                burst = max(n_span - 1, min(self.max_burst, P["last_steps"]))
            elif not lock and steps > 0 and P.get("last_steps"):
                burst = max(1, min(burst, 2))
            for _ in range(burst):
                if P["graph"] is not None and not lock:
                    P["graph"].replay()
                else:
                    self._enqueue_step(mlp, P)
            steps += burst
            pinned.copy_(st, non_blocking=True)
            torch.cuda.current_stream(dev).synchronize()
            cur = _ffi.RkState.from_buffer_copy(bytes(pinned.numpy().tobytes()))
            if cur.done:
                break
        else:
            raise RuntimeError("dopri5: step budget exhausted")
        P["last_steps"] = int(cur.accepted) + int(cur.rejected)
        self.stats = _rk_stats(cur, graph=P["graph"] is not None and not lock, lockstep=lock)
        if cnf is None:
            return traj.clone()
        n = B * D  # one copy back to the (n_span, B, D + 1) layout
        return torch.cat([traj[:, :n].view(n_span, B, D), traj[:, n:].view(n_span, B, 1)], 2)


class _CnfEulerTrajectory(torch.autograd.Function):
    """The Euler trajectory of ``cnf_wrapper(mlp, "exact")`` on the graph of ``x`` and the eight parameters of ``mlp``.
    forward is the one-launch CNF kernel, exactly as without autograd; backward is one call of
    ``cfm_ode_small_cnf_euler_backward_f32`` (csrc/cnf_train.cu), which reads every state it needs from the saved
    trajectory and fills a flat gradient buffer in ``parameters()`` order plus the input gradient."""

    @staticmethod
    def forward(ctx, node, mlp, x, t_span, *params):
        if not x.is_cuda:
            raise _ffi.CfmLibraryError("NeuralODE.trajectory needs CUDA inputs (no CPU fallback)")
        dev = x.device
        with torch.cuda.device(dev):
            ts = torch.as_tensor(t_span, dtype=torch.float32).to(dev).contiguous()
            traj = node._cnf_trajectory_on(mlp, x, ts, dev)
        ctx.mlp, ctx.ts, ctx.x_dtype = mlp, ts, x.dtype
        ctx.save_for_backward(traj, *params)  # an in-place update of a parameter before backward() raises
        return traj

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_traj):
        traj, *params = ctx.saved_tensors
        mlp, L = ctx.mlp, _ffi.lib()
        n_span, B, _ = traj.shape
        dev = traj.device
        grads = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
        gz = torch.empty_like(traj[0]) if ctx.needs_input_grad[2] else None
        ws = _ffi.workspace(L.cfm_ode_small_cnf_backward_workspace_bytes(B, n_span, mlp.dim, mlp.w), dev)
        grad_traj = grad_traj.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            _ffi.check(L.cfm_ode_small_cnf_euler_backward_f32(
                *[_ffi.ptr(p) for p in params], mlp.dim, mlp.w, mlp.act, _ffi.ptr(traj), B, _ffi.ptr(ctx.ts), n_span,
                _ffi.ptr(grad_traj), _ffi.ptr(gz), _ffi.ptr(grads), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(dev)),
                "cfm_ode_small_cnf_euler_backward_f32")
        out, o = [], 0
        for p, need in zip(params, ctx.needs_input_grad[4:]):
            out.append(grads[o:o + p.numel()].view(p.shape) if need else None)
            o += p.numel()
        return (None, None, None if gz is None else gz.to(ctx.x_dtype), None, *out)


class _NoBackward(torch.autograd.Function):
    """A trajectory on the graph whose backward() is not implemented: it raises ``NotImplementedError(reason)``
    instead of torch's generic "does not require grad".  forward is ``run()``, unchanged."""

    @staticmethod
    def forward(ctx, reason, run, x, *params):
        ctx.reason = reason
        return run()

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_traj):
        raise NotImplementedError(ctx.reason)


def ctypes_sizeof_state():
    return C.sizeof(_ffi.RkState)
