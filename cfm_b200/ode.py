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
(csrc/ode_small.cu, CNF variant).

A decreasing ``t_span`` is integrated as torchdyn does: dopri5 runs the field f_(s, x) = -f(-s, x) over
s = -t_span (for the MLP only a different weight set, ``MLP._time_reversed``), because the step controller
only steps forwards.  Euler needs no such step: a negative step already gives the same bits.
"""
import ctypes as C

import torch

from . import _ffi
from .models import MLP, cnf_wrapper, torch_wrapper


def _unwrap(vf):
    m = vf.model if isinstance(vf, torch_wrapper) else vf
    if not isinstance(m, MLP) or not m.time_varying:
        raise TypeError("cfm_b200.NeuralODE accelerates cfm_b200.models.MLP(time_varying=True) "
                        "vector fields (optionally wrapped in torch_wrapper); got "
                        f"{type(m).__name__}")
    return m


def _unwrap_cnf(vf):
    if vf.eps_fn is not None:
        raise NotImplementedError(
            f"cnf_wrapper(likelihood_estimator={vf.likelihood_estimator!r}): the Hutchinson estimators draw their "
            "probe vectors from torch's RNG on every call, which no device stream reproduces; the CUDA path "
            "provides the exact trace (likelihood_estimator='exact')")
    m = vf.model
    if not isinstance(m, MLP) or not m.time_varying:
        raise TypeError("cfm_b200.NeuralODE accelerates cnf_wrapper(cfm_b200.models.MLP(time_varying=True)); got "
                        f"cnf_wrapper({type(m).__name__})")
    return m


def _decreasing(t_span):
    return t_span.numel() >= 2 and bool(t_span[1] < t_span[0])


def _rk_stats(cur, **extra):
    """``NeuralODE.stats`` from the controller state (``_ffi.RkState``) a device run left."""
    return {"nfe": cur.nfe, "accepted": cur.accepted, "rejected": cur.rejected, "t": cur.t,
            "last_ratio": cur.ratio, **extra}


class NeuralODE(torch.nn.Module):
    """Subset of torchdyn.core.NeuralODE used by the reference examples."""

    def __init__(self, vector_field, solver="dopri5", sensitivity="adjoint", atol=1e-4, rtol=1e-4,
                 **unused):
        super().__init__()
        self.vf = vector_field
        if solver not in ("dopri5", "euler"):
            raise NotImplementedError(f"solver {solver!r}: the CUDA driver provides 'dopri5' and 'euler'")
        self.solver, self.atol, self.rtol = solver, float(atol), float(rtol)
        self.sensitivity = sensitivity  # irrelevant under no_grad sampling; kept for API parity
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

    @torch.no_grad()
    def forward(self, x, t_span):
        traj = self.trajectory(x, t_span)
        return t_span.to(x.device), traj

    @torch.no_grad()
    def trajectory(self, x, t_span):
        cnf = isinstance(self.vf, cnf_wrapper)
        mlp = _unwrap_cnf(self.vf) if cnf else _unwrap(self.vf)
        if not x.is_cuda:
            raise _ffi.CfmLibraryError("NeuralODE.trajectory needs CUDA inputs (no CPU fallback)")
        dev = x.device
        t_span = torch.as_tensor(t_span, dtype=torch.float32)
        reverse = self.solver == "dopri5" and _decreasing(t_span)  # see the module docstring
        with torch.cuda.device(dev):  # the library launches on the CURRENT device: make it the tensors' one
            if reverse:
                mlp, t_span = mlp._time_reversed(), -t_span
            out = (self._cnf_trajectory_on if cnf else self._trajectory_on)(mlp, x, t_span, dev)
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

    def _cnf_trajectory_on(self, mlp, x, t_span, dev):
        """cnf_wrapper(mlp, "exact"): the state [x, ll] goes through the CNF variant of the one-launch kernel."""
        if self.lockstep is not None:
            raise NotImplementedError("cnf_wrapper: lock-step sharding is not supported; the exact-likelihood path "
                                      "integrates the whole batch in one single-device kernel")
        if x.dim() != 2 or x.shape[1] != mlp.dim + 1:
            raise ValueError(f"cnf_wrapper: expected a state of shape (B, {mlp.dim + 1}) (x and the log-density "
                             f"column), got {tuple(x.shape)}")
        if t_span.numel() < 2:
            raise ValueError("cnf_wrapper: t_span needs at least two points")
        if mlp.out_dim != mlp.dim or not _ffi.lib().cfm_ode_small_cnf_supported(x.shape[0], mlp.dim, mlp.w):
            raise NotImplementedError(
                f"cnf_wrapper: no exact-likelihood kernel for B={x.shape[0]}, dim={mlp.dim}, w={mlp.w}, "
                f"out_dim={mlp.out_dim} (it takes w in {{32, 64, 128}}, dim <= 8, out_dim == dim and batches whose "
                "state fits in shared memory)")
        return self._fused_small(mlp, x.detach().float().contiguous(), t_span.to(dev).contiguous(), cnf=True)

    # ------------------------------------------------------------------------------------
    def _fused_small(self, mlp, x0, t_span, cnf=False):
        """Launch-bound regime (the 2-D tutorial models): Hairer init, all dopri5 / euler steps, the
        error norms and the controller in ONE cooperative kernel; one host read at the end.  ``cnf``: x0 is the
        [x, ll] state of cnf_wrapper (mlp.dim + 1 columns) and the kernel also integrates the trace."""
        L = _ffi.lib()
        dev = x0.device
        B, D = x0.shape  # D: state columns
        n_span = t_span.numel()
        ps = []
        for lin in mlp._linears():
            for p in (lin.weight, lin.bias):
                if p.device != dev or p.dtype != torch.float32:
                    raise _ffi.CfmLibraryError("MLP parameters must be fp32 on the input's CUDA device")
                ps.append(p.detach().contiguous())
        traj = torch.empty((n_span, B, D), dtype=torch.float32, device=dev)
        st = torch.zeros(ctypes_sizeof_state(), dtype=torch.uint8, device=dev)
        dim = mlp.dim if cnf else D
        ws = _ffi.workspace(L.cfm_ode_small_workspace_bytes(B, dim, mlp.w), dev)
        name = "cfm_ode_small_cnf_trajectory_f32" if cnf else "cfm_ode_small_trajectory_f32"
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
                mlp.vector_field_split(P["t_stage"], P["xs_hi"], P["xs_lo"], k[stage], skip_flag=P["done_flag"])
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

    def _plan(self, mlp, B, D, n_span, dev):
        """Persistent buffers (+ the captured step graph) for one problem shape and weight version."""
        key = (id(mlp), B, D, n_span, str(dev), mlp._weights_key(), mlp.mlp_algo, mlp.act, self.lockstep is not None)
        P = self._plans.get(key)
        if P is not None:
            return P
        self._plans.clear()  # one live plan: a new shape / new weights retire the old graph
        st = torch.zeros(ctypes_sizeof_state(), dtype=torch.uint8, device=dev)
        P = {"dev": dev, "numel": B * D, "st": st, "stp": _ffi.ptr(st),
             "x": torch.empty((B, D), dtype=torch.float32, device=dev),
             "xnew": torch.empty((B, D), dtype=torch.float32, device=dev),
             "xs": torch.empty((B, D), dtype=torch.float32, device=dev),
             "k": torch.empty((7, B, D), dtype=torch.float32, device=dev),
             "traj": torch.empty((n_span, B, D), dtype=torch.float32, device=dev),
             "t_span": torch.empty(n_span, dtype=torch.float32, device=dev),
             "t_stage": torch.zeros(1, dtype=torch.float32, device=dev),
             "scratch": torch.zeros(4, dtype=torch.float64, device=dev),
             "pinned": torch.empty(ctypes_sizeof_state(), dtype=torch.uint8, pin_memory=True),
             "pinned_init": torch.empty(ctypes_sizeof_state(), dtype=torch.uint8, pin_memory=True),
             "t0": torch.zeros(1, dtype=torch.float32, device=dev), "ts_host": None, "init_graph": None,
             "xs_hi": None, "xs_lo": None, "graph": None, "group": None, "dist": None, "numel_global": B * D}
        off = _ffi.RkState.err_acc.offset  # the float64 accumulator inside the device state struct
        P["err_acc"] = st[off:off + 8].view(torch.float64)
        off = _ffi.RkState.done.offset  # int32: non-zero once t has reached t_end
        P["done_flag"] = st[off:off + 4].view(torch.int32)
        if mlp.tc_path(B):
            # stage inputs go to the MLP as its fp16x3 tensor-core operand pair (hi, lo), written by the RK kernel
            P["xs_hi"] = torch.empty((B, D), dtype=torch.float16, device=dev)
            P["xs_lo"] = torch.empty((B, D), dtype=torch.float16, device=dev)
        self._plans[key] = P
        return P

    def _enqueue_init(self, mlp, P, lock):
        """k1 = f(t0, x) and the Hairer initial step (one extra evaluation), enqueued without a host round trip."""
        L = _ffi.lib()
        sp = _ffi.stream_ptr(P["dev"])
        stp, x, xs, k, numel, ng = P["stp"], P["x"], P["xs"], P["k"], P["numel"], P["numel_global"]
        mlp.vector_field(P["t0"], x, out=k[0])
        _ffi.check(L.cfm_rk_init_sums(stp, _ffi.ptr(x), _ffi.ptr(k[0]), None, _ffi.ptr(P["scratch"]), numel, 0, sp),
                   "cfm_rk_init_sums")
        if lock:
            P["dist"].all_reduce(P["scratch"], group=P["group"])
        _ffi.check(L.cfm_rk_init_probe(stp, _ffi.ptr(x), _ffi.ptr(k[0]), _ffi.ptr(xs), _ffi.ptr(P["t_stage"]),
                                       _ffi.ptr(P["scratch"]), numel, ng, sp), "cfm_rk_init_probe")
        mlp.vector_field(P["t_stage"], xs, out=k[1])
        if lock:  # phase 1 adds into scratch[2] only; keep the already-global scratch[0:2] out of the second reduce
            P["scratch"][2:].zero_()
        _ffi.check(L.cfm_rk_init_sums(stp, _ffi.ptr(x), _ffi.ptr(k[0]), _ffi.ptr(k[1]), _ffi.ptr(P["scratch"]),
                                      numel, 1, sp), "cfm_rk_init_sums")
        if lock:
            P["dist"].all_reduce(P["scratch"][2:3], group=P["group"])
        _ffi.check(L.cfm_rk_init_finish(stp, _ffi.ptr(P["t_span"]), _ffi.ptr(P["scratch"]), ng, sp),
                   "cfm_rk_init_finish")

    def _dopri5(self, mlp, x0, ts_host):
        """``ts_host``: the span as a contiguous fp32 CPU tensor."""
        dev = x0.device
        B, D = x0.shape
        numel = x0.numel()
        n_span = ts_host.numel()
        P = self._plan(mlp, B, D, n_span, dev)
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
        return traj.clone()


def ctypes_sizeof_state():
    return C.sizeof(_ffi.RkState)
