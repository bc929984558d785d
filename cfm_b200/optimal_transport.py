"""Minibatch OT coupling on H100: drop-in for ``torchcfm.optimal_transport``.

Same constructor, methods, attributes and error behaviour as the reference
``OTPlanSampler`` / ``wasserstein`` (torchcfm/optimal_transport.py:11-303), but the cost
matrix, the solver (log-domain Sinkhorn or exact assignment), the pair draw and the gather
all run as sm_90a kernels behind libcfm_b200.so and the N x N plan is never moved to the
host (the reference round-trips M through ``.cpu().numpy()`` at :87 and draws from a
flattened float64 plan on the CPU at :116-121).  No CPU fallback: without the library or
an sm_90 device every solver call raises.

RNG contract (reference :118): pair sampling consumes the global legacy NumPy stream.
``np.random.choice(p=..., replace=True)`` draws ``random_sample(size)`` and inverts the
cdf; here the same ``np.random.random_sample(size)`` values are drawn on the host and the
inversion runs on the device, so reseeding ``np.random`` reproduces a draw just as in the
reference.
"""
import collections
import ctypes as C
import math
import warnings
from functools import partial
from typing import Optional, Union

import numpy as np
import torch

from . import _ffi

# POT defaults of ot.sinkhorn (the reference never overrides them, :51)
_POT_NUM_ITER_MAX = 1000
_POT_STOP_THR = 1e-9


def _flat2d(x):
    """(bs, *dim) -> (bs, prod(dim))  -- reference :80-83."""
    return x.reshape(x.shape[0], -1) if x.dim() > 2 else x


def _cuda_f32(x, device):
    """Detached contiguous fp32 copy/view of ``x`` on ``device`` (reference detaches at :87)."""
    x = x.detach()
    if x.device != device:
        x = x.to(device, non_blocking=True)
    if x.dtype != torch.float32:
        x = x.float()
    return x.contiguous()


def _pick_device(*tensors):
    for t in tensors:
        if torch.is_tensor(t) and t.is_cuda:
            return t.device
    _ffi.require_device()
    return torch.device("cuda", torch.cuda.current_device())


class _Coupling:
    """Device-side result of one solve: cost matrix + either potentials or a permutation.  For exact OT
    between batches of different sizes (``expand`` = (m0, m1, L)) sigma is the assignment of the
    L x L replicated problem, L = lcm(n0, n1): row a stands for source a // m0, column b for target
    b // m1, every pair carries mass 1 / L."""
    __slots__ = ("M", "cost_max", "n0", "n1", "log_u", "log_v", "sigma", "status", "err",
                 "total_cost", "reg", "normalize", "method", "x0_dev", "x1_dev", "expand")


# Rectangular exact OT is solved as an assignment problem of size lcm(n0, n1); beyond this size the
# replicated cost matrix stops being a sensible use of the exact solver (O(L^3) worst case)
_MAX_EXPANDED = 8192
# pinned staging slots for the uniforms of the pair draw (see OTPlanSampler._uniforms)
_U_RING = 4


class _StageTimer:
    def __init__(self, sink, stage, device):
        self.sink, self.stage, self.device = sink, stage, device

    def __enter__(self):
        if self.sink is not None:
            self.a = torch.cuda.Event(enable_timing=True)
            self.b = torch.cuda.Event(enable_timing=True)
            self.a.record(torch.cuda.current_stream(self.device))
        return self

    def __exit__(self, *exc):
        if self.sink is not None:
            self.b.record(torch.cuda.current_stream(self.device))
            self.sink.append((self.stage, self.a, self.b))
        return False


class OTPlanSampler:
    """OTPlanSampler implements sampling coordinates according to an OT plan (wrt squared
    Euclidean cost) with different implementations of the plan calculation.

    Signature and attributes follow the reference (optimal_transport.py:15-61).  Keyword-only
    extras (not in the reference) tune the device solver:

    num_iter_max, stop_thr : POT's ``numItermax`` / ``stopThr`` for Sinkhorn (defaults 1000, 1e-9).
    precision : 'auto' | 'fp32' | 'fp64' | 'fp64-mixed' exponent arithmetic of the Sinkhorn kernel
        ('fp64-mixed': float64 potentials and exponent arguments, fp32 exponentials, negligible terms screened out in
        fp32 -- what 'auto' resolves to when |M/reg| > 64; 'fp64-mixed-unscreened' evaluates every term and
        'fp32-generic' forces the fp32 arithmetic onto the generic kernel: cross-checks).
    stall_tol : stop once an fp32 fixed point is reached (see include/cfm_b200.h); 0 disables.
    cost_algo : 0 auto (fp16x3 tensor-core path for aligned shapes; SIMT for exact OT), 1 SIMT fp32,
        3 wgmma fp16x3.
    """

    def __init__(
        self,
        method: str,
        reg: float = 0.05,
        reg_m: float = 1.0,
        normalize_cost: bool = False,
        num_threads: Union[int, str] = 1,
        warn: bool = True,
        *,
        num_iter_max: int = _POT_NUM_ITER_MAX,
        stop_thr: float = _POT_STOP_THR,
        precision: str = "auto",
        stall_tol: float = 0.1,
        cost_algo: int = 0,
    ) -> None:
        # ot_fn takes (a, b, M) like the POT callables bound in the reference (:47-57)
        if method == "exact":
            self.ot_fn = partial(self._ot_fn_exact, numThreads=num_threads)
        elif method == "sinkhorn":
            self.ot_fn = partial(self._ot_fn_sinkhorn, reg=reg)
        elif method in ("unbalanced", "partial"):
            self.ot_fn = partial(self._ot_fn_unsupported, method=method)
        else:
            raise ValueError(f"Unknown method: {method}")
        self.method = method
        self.reg = reg
        self.reg_m = reg_m
        self.normalize_cost = normalize_cost
        self.warn = warn
        self.num_iter_max = int(num_iter_max)
        self.stop_thr = float(stop_thr)
        if precision not in ("auto", "fp32", "fp64", "fp32-generic", "fp64-mixed", "fp64-mixed-unscreened"):
            raise ValueError(f"Unknown precision: {precision}")
        self.precision = precision
        self.stall_tol = float(stall_tol)
        if cost_algo not in (0, 1, 3):
            raise ValueError(f"Unknown cost_algo: {cost_algo}")
        self.cost_algo = int(cost_algo)
        self._last_info = {}
        self._pending = collections.deque()  # deferred status words of warn=False calls (event, pinned, coupling)
        self._bufs = collections.OrderedDict()  # (n0, n1, d, device, stream) -> preallocated device buffers
        self._u_ring = {}                       # (n, device) -> pinned uniform staging ring
        self.stage_events = None  # set to a list to collect (stage, start_event, end_event)

    # ------------------------------------------------------------------ status words
    @property
    def last_info(self):
        """Diagnostics of the most recent solve ({"flags", "iterations", ...}); resolves (synchronises on)
        any status word a ``warn=False`` call left pending."""
        self._flush_pending(block=True)
        return self._last_info

    @last_info.setter
    def last_info(self, value):
        self._last_info = value

    def _flush_pending(self, block=False):
        """Evaluate status words whose device->host copy has landed (all of them when ``block``)."""
        while self._pending:
            ev, pinned, cp = self._pending[0]
            if not block and not ev.query():
                break
            ev.synchronize()
            self._pending.popleft()
            self._evaluate_status(cp, pinned.tolist(), None)

    def _buffers(self, n0, n1, d, device, algo):
        """Device buffers of one problem shape, allocated once per (shape, device, stream) and reused by every
        later call on that stream: the cost matrix, the kernels' workspaces, the potentials and the draw's
        index / uniform arrays.  A training loop therefore makes no allocator call (and no cudaMalloc, which
        synchronises the device) in steady state.  Stream-ordered reuse is safe because every consumer of
        a call's buffers is enqueued on the same stream before the next call's producers."""
        L = _ffi.lib()
        stream = torch.cuda.current_stream(device).cuda_stream
        key = (n0, n1, d, str(device), stream, algo, self.method)
        B = self._bufs.get(key)
        if B is not None:
            self._bufs.move_to_end(key)
            return B
        ld = (n1 + 3) // 4 * 4  # 16-byte aligned rows for the float4 / TMA paths
        B = {"ld": ld,
             "M": torch.empty((n0, ld), dtype=torch.float32, device=device),
             "cmax": torch.empty(1, dtype=torch.float32, device=device),
             "ws_cost": _ffi.workspace(L.cfm_sqdist_workspace_bytes(n0, n1, d, algo), device)}
        if self.method == "sinkhorn":
            B["log_u"] = torch.empty(n0, dtype=torch.float64, device=device)
            B["log_v"] = torch.empty(n1, dtype=torch.float64, device=device)
            B["ws_sk"] = _ffi.workspace(L.cfm_sinkhorn_workspace_bytes(n0, n1), device)
            B["ws_draw"] = _ffi.workspace(L.cfm_plan_sample_workspace_bytes(n0), device)
        self._bufs[key] = B
        while len(self._bufs) > 2:  # keep the two most recent shapes (e.g. a ragged last batch)
            self._bufs.popitem(last=False)
        return B

    def _timed(self, stage, device):
        """Context manager recording CUDA events around a stage when profiling is on."""
        return _StageTimer(self.stage_events, stage, device)

    # ------------------------------------------------------------------ device stages
    def _cost(self, x0, x1, device, squared=True):
        """(a3) M = cdist(x0, x1)**2 and its max, on the device (reference :84-86)."""
        L = _ffi.lib()
        a, b = _cuda_f32(_flat2d(x0), device), _cuda_f32(_flat2d(x1), device)
        if a.shape[1] != b.shape[1]:
            raise RuntimeError(f"X1 and X2 must have the same number of columns. "
                               f"X1: {a.shape[1]} X2: {b.shape[1]}")
        n0, n1, d = a.shape[0], b.shape[0], a.shape[1]
        # exact OT needs fp32-FMA-grade costs (sigma must not flip): SIMT path unless overridden;
        # the tensor-core paths (~1e-6 relative, truncating accumulator) serve Sinkhorn
        algo = self.cost_algo if self.cost_algo else (1 if self.method == "exact" else 0)
        B = self._buffers(n0, n1, d, device, algo)
        Mbuf, cmax, ws = B["M"], B["cmax"], B["ws_cost"]
        with torch.cuda.device(device):
            _ffi.check(L.cfm_sqdist_f32(_ffi.ptr(a), _ffi.ptr(b), _ffi.ptr(Mbuf), n0, n1, d, B["ld"],
                                        1 if squared else 0, _ffi.ptr(cmax), algo,
                                        _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(device)),
                       "cfm_sqdist_f32")
        self._last_inputs = (a, b)
        self._last_bufs = B
        return Mbuf, cmax, n0, n1

    def _solve_sinkhorn(self, Mbuf, cmax, n0, n1, reg, normalize, num_iter_max=None,
                        stop_thr=None, bufs=None):
        L = _ffi.lib()
        dev = Mbuf.device
        cp = _Coupling()
        cp.M, cp.cost_max, cp.n0, cp.n1, cp.reg, cp.normalize = Mbuf, cmax, n0, n1, float(reg), bool(normalize)
        cp.method, cp.sigma, cp.total_cost, cp.expand = "sinkhorn", None, None, None
        if bufs is not None and "log_u" in bufs:  # preallocated per shape (see _buffers)
            cp.log_u, cp.log_v, ws = bufs["log_u"], bufs["log_v"], bufs["ws_sk"]
        else:
            cp.log_u = torch.empty(n0, dtype=torch.float64, device=dev)
            cp.log_v = torch.empty(n1, dtype=torch.float64, device=dev)
            ws = _ffi.workspace(L.cfm_sinkhorn_workspace_bytes(n0, n1), dev)
        # the status word and the error are per call: a deferred report may read them after later solves
        cp.status = torch.zeros(4, dtype=torch.int32, device=dev)
        cp.err = torch.zeros(1, dtype=torch.float64, device=dev)
        prec = {"auto": -1, "fp32": 0, "fp64": 1, "fp32-generic": 2, "fp64-mixed": 3,
                "fp64-mixed-unscreened": 4}[self.precision]
        with torch.cuda.device(dev):
            _ffi.check(L.cfm_sinkhorn_log_f32(
                _ffi.ptr(Mbuf), n0, n1, Mbuf.stride(0), float(reg), _ffi.ptr(cmax), int(bool(normalize)),
                int(self.num_iter_max if num_iter_max is None else num_iter_max),
                float(self.stop_thr if stop_thr is None else stop_thr), 10, prec,
                0.0 if (self.stop_thr if stop_thr is None else stop_thr) <= 0 else self.stall_tol,
                _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), _ffi.ptr(cp.status), _ffi.ptr(cp.err),
                _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(dev)), "cfm_sinkhorn_log_f32")
        return cp

    def _solve_exact(self, Mbuf, cmax, n0, n1, normalize):
        """Optimal assignment on the device.  n0 == n1: the LP vertex of uniform marginals is P_sigma / n.
        n0 != n1 (pot.emd takes any pair of marginals, reference :79,87): the transport polytope with
        marginals 1/n0, 1/n1 has vertices whose entries are multiples of 1/L, L = lcm(n0, n1), so the LP
        optimum is the optimal assignment of the L x L problem in which source i is replicated L/n0 times
        and target j L/n1 times -- solved by the same kernel on the replicated cost matrix."""
        L = _ffi.lib()
        dev = Mbuf.device
        cp = _Coupling()
        cp.M, cp.cost_max, cp.n0, cp.n1, cp.reg, cp.normalize = Mbuf, cmax, n0, n1, None, bool(normalize)
        cp.method, cp.log_u, cp.log_v, cp.err, cp.expand = "exact", None, None, None, None
        n, Msolve = n0, Mbuf
        if n0 != n1:
            g = math.gcd(n0, n1)
            m0, m1 = n1 // g, n0 // g
            n = n0 * m0
            if n > _MAX_EXPANDED:
                raise NotImplementedError(
                    f"exact OT between batches of {n0} and {n1} samples needs an assignment problem of size "
                    f"lcm = {n} > {_MAX_EXPANDED}; use equal batch sizes (or sizes with a small lcm)")
            cp.expand = (m0, m1, n)
            ld = (n + 3) // 4 * 4
            Msolve = torch.zeros((n, ld), dtype=torch.float32, device=dev)
            Msolve[:, :n] = Mbuf[:, :n1].repeat_interleave(m0, dim=0).repeat_interleave(m1, dim=1)
        cp.sigma = torch.empty(n, dtype=torch.int32, device=dev)
        cp.total_cost = torch.zeros(1, dtype=torch.float64, device=dev)
        cp.status = torch.zeros(4, dtype=torch.int32, device=dev)
        ws = _ffi.workspace(L.cfm_assign_workspace_bytes(n), dev)
        with torch.cuda.device(dev):
            _ffi.check(L.cfm_assign_exact_f32(
                _ffi.ptr(Msolve), n, Msolve.stride(0), _ffi.ptr(cmax), int(bool(normalize)),
                _ffi.ptr(cp.sigma), _ffi.ptr(cp.total_cost), _ffi.ptr(cp.status), _ffi.ptr(ws),
                ws.numel(), _ffi.stream_ptr(dev)), "cfm_assign_exact_f32")
        return cp

    def _exact_plan(self, cp):
        """float64 host plan of an exact coupling, the array pot.emd returns (reference :87)."""
        sigma = cp.sigma.cpu().numpy().astype(np.int64)
        p = np.zeros((cp.n0, cp.n1), dtype=np.float64)
        if cp.expand is None:
            p[np.arange(cp.n0), sigma] = 1.0 / cp.n0
        else:
            m0, m1, n = cp.expand
            np.add.at(p, (np.arange(n) // m0, sigma // m1), 1.0 / n)
        return p

    def _couple(self, x0, x1, device):
        """cost + solve on the device; nothing is synchronised or copied to the host."""
        with self._timed("cost", device):
            Mbuf, cmax, n0, n1 = self._cost(x0, x1, device)
        if self.method == "exact":
            with self._timed("solve", device):
                cp = self._solve_exact(Mbuf, cmax, n0, n1, self.normalize_cost)
        elif self.method == "sinkhorn":
            with self._timed("solve", device):
                cp = self._solve_sinkhorn(Mbuf, cmax, n0, n1, self.reg, self.normalize_cost,
                                          bufs=self._last_bufs)
        else:
            self._ot_fn_unsupported(None, None, None, method=self.method)
        cp.x0_dev, cp.x1_dev = self._last_inputs  # device fp32 copies made for the cost kernel
        self._last_inputs = None
        return cp

    def _stairs(self, n, dev):
        """cdf of the uniform permutation plan, the float64 sequential cumsum np.random.choice
        forms (:118); cached per (n, device)."""
        cache = self.__dict__.setdefault("_stairs_cache", {})
        st = cache.get((n, dev))
        if st is None:
            stairs = np.cumsum(np.full(n, 1.0 / n))
            stairs /= stairs[-1]
            st = cache[(n, dev)] = torch.from_numpy(stairs).to(dev)
        return st

    def _uniforms(self, n, dev):
        """n uniforms of the global NumPy stream (what np.random.choice consumes at :118) on the device,
        staged through a ring of pinned host slots: a pageable source would make the copy synchronous and
        drain the launch queue on every call (the host could then never run ahead of the GPU).  A slot is
        rewritten only after the copy that last read it has completed (event; normally long done)."""
        key = (n, str(dev))
        ring = self._u_ring.get(key)
        if ring is None:
            ring = self._u_ring[key] = {"k": 0,
                                        "pin": [torch.empty(n, dtype=torch.float64, pin_memory=True)
                                                for _ in range(_U_RING)],
                                        "ev": [None] * _U_RING}
            if len(self._u_ring) > 4:
                self._u_ring.pop(next(iter(self._u_ring)))
        k = ring["k"]
        ring["k"] = (k + 1) % _U_RING
        if ring["ev"][k] is not None:
            ring["ev"][k].synchronize()
        pin = ring["pin"][k]
        pin.numpy()[:] = np.random.random_sample(n)
        u = torch.empty(n, dtype=torch.float64, device=dev)
        u.copy_(pin, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(dev))
        ring["ev"][k] = ev
        return u

    def _draw(self, cp, batch_size, u=None):
        """(a6) inverse-cdf draw on the device from host uniforms of the global NumPy RNG (``u``: those
        uniforms already on the device, float64)."""
        L = _ffi.lib()
        dev = cp.M.device
        if u is None:
            u = self._uniforms(batch_size, dev)
        i = torch.empty(batch_size, dtype=torch.int64, device=dev)
        j = torch.empty(batch_size, dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            if cp.method == "exact":
                n = cp.n0
                st = self._stairs(n, dev)
                _ffi.check(L.cfm_perm_plan_sample(_ffi.ptr(cp.sigma), _ffi.ptr(st), n, _ffi.ptr(u),
                                                  batch_size, _ffi.ptr(i), _ffi.ptr(j),
                                                  _ffi.stream_ptr(dev)), "cfm_perm_plan_sample")
            else:
                ws = _ffi.workspace(L.cfm_plan_sample_workspace_bytes(cp.n0), dev)
                _ffi.check(L.cfm_plan_sample(
                    _ffi.ptr(cp.M), cp.n0, cp.n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max),
                    int(cp.normalize), _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), 1, _ffi.ptr(u), batch_size,
                    _ffi.ptr(i), _ffi.ptr(j), _ffi.ptr(cp.status), _ffi.ptr(ws), ws.numel(),
                    _ffi.stream_ptr(dev)), "cfm_plan_sample")
        return i, j

    def _report(self, cp, defer=False):
        """Numerical guards of get_map (:88-96) + POT's non-convergence warning.  The status word is ALWAYS
        evaluated (the reference's ``warn`` only gates the warnings.warn calls): immediately -- one small
        sync -- or, for ``defer`` (Sinkhorn calls of a warn=False sampler, whose conditions only print),
        once its copy to pinned memory has landed: at the next call or when ``last_info`` is read."""
        if defer:
            # pinned landing slots are allocated ONCE (a fresh pinned block is a cudaHostAlloc, which waits for
            # the device to go idle and would drain the launch queue in the middle of a training loop)
            ring = self.__dict__.get("_status_ring")
            if ring is None:
                ring = self._status_ring = {"k": 0, "buf": torch.empty((16, 4), dtype=torch.int32, pin_memory=True)}
            while len(self._pending) >= 12:  # a slot is reused only after its status word has been evaluated
                self._flush_pending(block=False)
                if len(self._pending) >= 12:
                    ev0, pinned0, cp0 = self._pending.popleft()
                    ev0.synchronize()
                    self._evaluate_status(cp0, pinned0.tolist(), None)
            pinned = ring["buf"][ring["k"]]
            ring["k"] = (ring["k"] + 1) % 16
            pinned.copy_(cp.status, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream(cp.status.device))
            self._pending.append((ev, pinned, cp))
            return None
        self._flush_pending(block=True)
        st = cp.status.cpu().tolist()
        return self._evaluate_status(cp, st, float(cp.err.item()) if cp.err is not None else None)

    def _evaluate_status(self, cp, st, err):
        if cp.method == "exact":  # status = {flags, augmentations, Dijkstra steps, -}
            info = {"flags": st[0], "iterations": st[1], "dijkstra_steps": st[2], "precise": True, "method": cp.method}
        else:                     # status = {flags, iterations, arithmetic, kernel variant}
            info = {"flags": st[0], "iterations": st[1], "precise": bool(st[2]),
                    "arithmetic": ("fp32", "fp64", "fp64-mixed")[st[2]] if 0 <= st[2] <= 2 else st[2],
                    "method": cp.method}
        if err is not None:
            info["err"] = err
        self._last_info = info
        if st[0] & _ffi.FLAG_INFEASIBLE or (cp.method == "exact" and st[0] & _ffi.FLAG_NONFINITE):
            raise RuntimeError("exact OT: the cost matrix has no finite assignment (inf/nan costs)")
        if st[0] & _ffi.FLAG_NONFINITE:
            print("ERROR: p is not finite")
            print("Cost max", float(cp.cost_max.item()))
        if st[0] & _ffi.FLAG_ZERO_MASS and self.warn:
            warnings.warn("Numerical errors in OT plan, reverting to uniform plan.")
        if st[0] & _ffi.FLAG_NOT_CONVERGED and self.warn and cp.method == "sinkhorn" \
                and self.stop_thr > 0:
            warnings.warn("Sinkhorn did not converge. You might want to increase the number of "
                          "iterations `numItermax` or the regularization parameter `reg`.")
        return info

    @staticmethod
    def _gather(x, idx_dev, out=None):
        """(a7) x[idx] on x's device; autograd-preserving torch indexing when x needs grad."""
        if x.requires_grad or not x.is_cuda or x.dtype.itemsize not in (1, 2, 4, 8) \
                or not x.is_contiguous():
            return x[idx_dev.to(x.device)]
        L = _ffi.lib()
        if out is None:
            out = torch.empty((idx_dev.shape[0],) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
        row = int(np.prod(x.shape[1:])) if x.dim() > 1 else 1
        with torch.cuda.device(x.device):  # kernels launch on the CURRENT device: make it the tensors' one
            _ffi.check(L.cfm_gather_rows(_ffi.ptr(x), row, x.dtype.itemsize, _ffi.ptr(idx_dev),
                                         idx_dev.shape[0], _ffi.ptr(out), _ffi.stream_ptr(x.device)),
                       "cfm_gather_rows")
        return out

    def _gather_like_input(self, x, x_dev_f32, idx_dev):
        """Result lives where the input lives (reference: x0[i] on x0's device).  Host inputs
        are gathered on the device from the uploaded copy and copied back."""
        if x.is_cuda or x.requires_grad or x.dtype != torch.float32:
            return self._gather(x, idx_dev)
        g = self._gather(x_dev_f32.reshape((x.shape[0],) + tuple(x.shape[1:])), idx_dev)
        out = torch.empty(g.shape, dtype=g.dtype, pin_memory=x.is_pinned())
        out.copy_(g, non_blocking=x.is_pinned())
        if x.is_pinned():
            torch.cuda.current_stream(g.device).synchronize()
        return out

    # ------------------------------------------------------------------ reference API
    def get_map(self, x0, x1):
        """Compute the OT plan (wrt squared Euclidean cost) between a source and a target
        minibatch; returns the (bs, bs) float64 NumPy plan like the reference (:63-97)."""
        device = _pick_device(x0, x1)
        cp = self._couple(x0, x1, device)
        if cp.method == "exact":
            self._report(cp)
            return self._exact_plan(cp)
        L = _ffi.lib()
        plan = torch.empty((cp.n0, cp.n1), dtype=torch.float64, device=device)
        mass = torch.zeros(1, dtype=torch.float64, device=device)
        _ffi.check(L.cfm_plan_materialize_f64(
            _ffi.ptr(cp.M), cp.n0, cp.n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max),
            int(cp.normalize), _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), _ffi.ptr(plan),
            _ffi.ptr(mass), _ffi.ptr(cp.status), _ffi.stream_ptr(device)), "cfm_plan_materialize_f64")
        if abs(float(mass.item())) < 1e-8:
            cp.status[0] |= _ffi.FLAG_ZERO_MASS
        info = self._report(cp)
        p = plan.cpu().numpy()
        if info["flags"] & _ffi.FLAG_ZERO_MASS:
            p = np.ones_like(p) / p.size
        return p

    def sample_map(self, pi, batch_size, replace=True):
        r"""Draw source and target samples from pi  $(x,z) \sim \pi$ (reference :99-121).

        ``pi`` is a host NumPy plan by contract; large plans drawn with replacement are
        inverted on the device, everything else uses NumPy's own ``choice`` exactly as the
        reference does."""
        pi = np.asarray(pi)
        if replace and pi.size >= (1 << 20) and torch.cuda.is_available():
            L = _ffi.lib()
            dev = torch.device("cuda", torch.cuda.current_device())
            P = torch.from_numpy(np.ascontiguousarray(pi, dtype=np.float64)).to(dev)
            u = torch.from_numpy(np.random.random_sample(batch_size)).to(dev)
            i = torch.empty(batch_size, dtype=torch.int64, device=dev)
            j = torch.empty(batch_size, dtype=torch.int64, device=dev)
            ws = _ffi.workspace(L.cfm_plan_sample_workspace_bytes(pi.shape[0]), dev)
            _ffi.check(L.cfm_dense_plan_sample_f64(_ffi.ptr(P), pi.shape[0], pi.shape[1], _ffi.ptr(u),
                                                   batch_size, _ffi.ptr(i), _ffi.ptr(j), _ffi.ptr(ws),
                                                   ws.numel(), _ffi.stream_ptr(dev)),
                       "cfm_dense_plan_sample_f64")
            return i.cpu().numpy(), j.cpu().numpy()
        p = pi.flatten()
        p = p / p.sum()
        choices = np.random.choice(pi.shape[0] * pi.shape[1], p=p, size=batch_size, replace=replace)
        return np.divmod(choices, pi.shape[1])

    def _finish(self, cp):
        """Evaluate the solve's status word: at once (exact OT may have to raise; warn=True samplers warn
        inside the call like the reference) or deferred (Sinkhorn with warn=False: nothing to raise)."""
        return self._report(cp, defer=(cp.method == "sinkhorn" and not self.warn))

    def _rectangular(self, x0, x1):
        return self.method == "exact" and x0.shape[0] != x1.shape[0]

    def sample_pairs(self, x0, x1, batch_size=None):
        """Device-resident (i, j) int64 index tensors of one coupling (no plan materialised)."""
        self._flush_pending()
        device = _pick_device(x0, x1)
        nd = x0.shape[0] if batch_size is None else batch_size
        if self._rectangular(x0, x1):  # plan is not a permutation: the reference's own host draw on it
            i, j = self.sample_map(self.get_map(x0, x1), nd)
            return torch.from_numpy(i).to(device), torch.from_numpy(j).to(device)
        cp = self._couple(x0, x1, device)
        i, j = self._draw(cp, nd)
        self._finish(cp)
        return i, j

    def sample_plan(self, x0, x1, replace=True):
        r"""Compute the OT plan $\pi$ between a source and a target minibatch and draw source
        and target samples from pi $(x,z) \sim \pi$ (reference :123-145).  Returns
        ``x0[i], x1[j]`` on the inputs' device."""
        if not replace or self._rectangular(x0, x1):
            pi = self.get_map(x0, x1)
            i, j = self.sample_map(pi, x0.shape[0], replace=replace)
            return x0[i], x1[j]
        self._flush_pending()
        device = _pick_device(x0, x1)
        cp = self._couple(x0, x1, device)
        with self._timed("draw", device):
            i, j = self._draw(cp, x0.shape[0])
        with self._timed("gather", device):
            out0 = self._gather_like_input(x0, cp.x0_dev, i)
            out1 = self._gather_like_input(x1, cp.x1_dev, j)
        self._finish(cp)
        return out0, out1

    def sample_plan_with_scipy(self, x0, x1):
        r"""Deterministic permutation coupling (reference :147-182): keeps x0's order and
        returns x1 permuted by the optimal assignment -- here from the device exact solver."""
        device = _pick_device(x0, x1)
        x0f, x1f = _flat2d(x0), _flat2d(x1)
        if x0f.shape[0] != x1f.shape[0]:
            raise ValueError("sample_plan_with_scipy pairs every x0 with one x1: batch sizes must match "
                             f"(got {x0f.shape[0]} and {x1f.shape[0]})")
        Mbuf, cmax, n0, n1 = self._cost(x0f, x1f, device)
        cp = self._solve_exact(Mbuf, cmax, n0, n1, self.normalize_cost)
        self._report(cp)
        return x0f, self._gather(x1f, cp.sigma.to(torch.int64))

    def sample_plan_with_labels(self, x0, x1, y0=None, y1=None, replace=True):
        r"""sample_plan that also carries labels through the draw (reference :184-219)."""
        if not replace or self._rectangular(x0, x1):
            pi = self.get_map(x0, x1)
            i, j = self.sample_map(pi, x0.shape[0], replace=replace)
            return x0[i], x1[j], (y0[i] if y0 is not None else None), (y1[j] if y1 is not None else None)
        self._flush_pending()
        device = _pick_device(x0, x1)
        cp = self._couple(x0, x1, device)
        i, j = self._draw(cp, x0.shape[0])
        out = (self._gather_like_input(x0, cp.x0_dev, i),
               self._gather_like_input(x1, cp.x1_dev, j),
               self._gather(y0, i) if y0 is not None else None,
               self._gather(y1, j) if y1 is not None else None)
        self._finish(cp)
        return out

    def _draw_rows(self, cp, rows, u):
        """Row-conditional draw  j_k ~ pi[rows[k], :] / sum(pi[rows[k], :])  from device uniforms u."""
        if cp.method == "exact":
            # one-hot rows: the draw is sigma[i] whatever u is (clamped: an infeasible solve raises in
            # _report right after, but its sigma must not index out of range before that)
            return cp.sigma.to(torch.int64)[rows].clamp_(0, cp.n1 - 1)
        nxt = torch.empty(rows.shape[0], dtype=torch.int64, device=rows.device)
        _ffi.check(_ffi.lib().cfm_plan_sample_rows(
            _ffi.ptr(cp.M), cp.n0, cp.n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max),
            int(cp.normalize), _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), _ffi.ptr(rows), _ffi.ptr(u), rows.shape[0],
            _ffi.ptr(nxt), _ffi.ptr(cp.status), _ffi.stream_ptr(rows.device)), "cfm_plan_sample_rows")
        return nxt

    def sample_trajectory(self, X):
        """OT trajectories across ``times`` populations (reference :221-251).  The times-1 couplings
        and the per-sample conditional draws  j ~ pi_t[i, :] / sum(pi_t[i, :])  run on the device (no
        plan is materialised, cfm_plan_sample_rows); the uniforms are taken from the global NumPy
        stream in the reference's order -- all draws of transition t, sample by sample, one
        ``random_sample`` each, exactly what ``np.random.choice(n, p=...)`` consumes at :244-246.
        Returns a NumPy array (bs, times, *dim) like the reference's ``np.stack``."""
        times, n = X.shape[1], X.shape[0]
        if not torch.is_tensor(X):
            X = torch.as_tensor(X)
        device = _pick_device(X)
        rows = torch.arange(n, dtype=torch.int64, device=device)
        chain = [rows]
        # the reference solves every coupling before it draws (:233-236); the solves consume no random
        # numbers, so solve -> draw -> release per transition gives the same chain with one cost
        # matrix resident at a time
        for t in range(times - 1):
            cp = self._couple(X[:, t], X[:, t + 1], device)
            u = self._uniforms(n, device)
            nxt = self._draw_rows(cp, rows, u)
            self._finish(cp)
            rows = nxt
            chain.append(rows)
            del cp
        Xh = X.detach()
        out = [self._gather(Xh[:, t].contiguous().to(device), chain[t]).cpu().numpy() for t in range(times)]
        return np.stack(out, axis=1)

    # ------------------------------------------------------------------ ot_fn callables
    @staticmethod
    def _check_uniform(a, b, M):
        n0, n1 = M.shape
        for m, n in ((a, n0), (b, n1)):
            m = np.asarray(m, dtype=np.float64)
            if m.size and not np.allclose(m, 1.0 / n):
                raise NotImplementedError("the device solvers take uniform marginals "
                                          "(OTPlanSampler always passes pot.unif, reference :79)")

    def _upload_cost(self, M):
        dev = _pick_device(M)
        Mt = torch.as_tensor(M, dtype=torch.float32).to(dev)
        n0, n1 = Mt.shape
        ld = (n1 + 3) // 4 * 4
        Mbuf = torch.zeros((n0, ld), dtype=torch.float32, device=dev)
        Mbuf[:, :n1] = Mt
        return Mbuf, Mt.max().reshape(1).contiguous(), n0, n1

    def _ot_fn_exact(self, a, b, M, numThreads=1):
        """(a, b, M) -> float64 plan, the signature of pot.emd as bound at reference :49."""
        self._check_uniform(a, b, np.empty(tuple(M.shape)))
        Mbuf, cmax, n0, n1 = self._upload_cost(M)
        cp = self._solve_exact(Mbuf, cmax, n0, n1, False)
        self._report(cp)
        return self._exact_plan(cp)

    def _ot_fn_sinkhorn(self, a, b, M, reg):
        """(a, b, M) -> float64 plan, the signature of pot.sinkhorn as bound at reference :51."""
        self._check_uniform(a, b, np.empty(tuple(M.shape)))
        Mbuf, cmax, n0, n1 = self._upload_cost(M)
        cp = self._solve_sinkhorn(Mbuf, cmax, n0, n1, reg, False)
        L = _ffi.lib()
        plan = torch.empty((n0, n1), dtype=torch.float64, device=Mbuf.device)
        mass = torch.zeros(1, dtype=torch.float64, device=Mbuf.device)
        _ffi.check(L.cfm_plan_materialize_f64(
            _ffi.ptr(cp.M), n0, n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max), 0,
            _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), _ffi.ptr(plan), _ffi.ptr(mass),
            _ffi.ptr(cp.status), _ffi.stream_ptr(Mbuf.device)), "cfm_plan_materialize_f64")
        self._report(cp)
        return plan.cpu().numpy()

    @staticmethod
    def _ot_fn_unsupported(a, b, M, method):
        raise NotImplementedError(
            f"OTPlanSampler(method={method!r}): unbalanced / partial OT are outside the CUDA hot "
            "path (BASELINE.json north_star names exact and Sinkhorn couplings only)")


def wasserstein(
    x0: torch.Tensor,
    x1: torch.Tensor,
    method: Optional[str] = None,
    reg: float = 0.05,
    power: int = 2,
    **kwargs,
) -> float:
    """Wasserstein-1/2 distance between two minibatches (reference :254-303), solved on the
    device: exact -> optimal assignment cost / n; sinkhorn -> <P, M> of the entropic plan."""
    assert power == 1 or power == 2
    if method == "exact" or method is None:
        kind = "exact"
    elif method == "sinkhorn":
        kind = "sinkhorn"
    else:
        raise ValueError(f"Unknown method: {method}")
    device = _pick_device(x0, x1)
    s = OTPlanSampler(kind, reg=reg, warn=False, num_iter_max=int(kwargs.get("numItermax", 1e7)),
                      stop_thr=float(kwargs.get("stopThr", _POT_STOP_THR)))
    Mbuf, cmax, n0, n1 = s._cost(x0, x1, device, squared=(power == 2))
    if kind == "exact":
        cp = s._solve_exact(Mbuf, cmax, n0, n1, False)
        s._report(cp)
        ret = float(cp.total_cost.item()) / (n0 if cp.expand is None else cp.expand[2])
    else:
        cp = s._solve_sinkhorn(Mbuf, cmax, n0, n1, reg, False, bufs=s._last_bufs)
        out = torch.zeros(1, dtype=torch.float64, device=device)
        _ffi.check(_ffi.lib().cfm_plan_dot_cost(
            _ffi.ptr(cp.M), n0, n1, cp.M.stride(0), cp.reg, _ffi.ptr(cp.cost_max), 0,
            _ffi.ptr(cp.log_u), _ffi.ptr(cp.log_v), _ffi.ptr(out), _ffi.stream_ptr(device)),
            "cfm_plan_dot_cost")
        ret = float(out.item())
    if power == 2:
        ret = math.sqrt(ret)
    return ret


class CouplingStream:
    """Software pipeline over a sequence of HOST minibatches: the upload of batch k+1, the coupling of
    batch k and the download of batch k-1 run on three CUDA streams, so a training loop that feeds
    host batches (the reference's DataLoader -> ``sample_plan`` pattern, e.g.
    examples/images/cifar10/train_cifar10.py:133-140) pays max(copy, compute) per batch instead of
    their sum.  Results, RNG consumption order (the NumPy global stream, reference :118) and warnings
    are those of calling ``sampler.sample_plan`` on each batch in submission order.

        stream = CouplingStream(sampler)
        for x0c, x1c in stream.map(loader):      # loader yields (x0, x1) CPU fp32 tensors
            ...

    ``submit`` / ``collect`` expose the same thing without the generator.  At most ``depth`` batches
    are in flight; ``submit`` blocks on the oldest one when the pipeline is full.
    """

    def __init__(self, sampler, device=None, depth=2):
        if depth < 1:
            raise ValueError("depth must be >= 1")
        _ffi.require_device()
        self.sampler = sampler
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.depth = int(depth)
        self._up = torch.cuda.Stream(self.device)
        self._run = torch.cuda.Stream(self.device)
        self._down = torch.cuda.Stream(self.device)
        self._inflight = []  # FIFO of (done_event, out0_host, out1_host, coupling)
        self._ready = []     # batches whose download already finished because submit had to make room
        # Device-side staging lives in a ring of depth + 1 slots that are allocated once per batch shape: a slot
        # is reused only after its previous batch has been collected, so no allocator call (and no implicit
        # device synchronisation of a cudaMalloc) sits between two batches in steady state.
        self._slots = [None] * (self.depth + 1)
        self._next_slot = 0
        self._primed = set()

    def _slot(self, x0, x1):
        k = self._next_slot
        self._next_slot = (k + 1) % len(self._slots)
        key = (tuple(x0.shape), tuple(x1.shape))
        sl = self._slots[k]
        if sl is None or sl["key"] != key:
            dev, n = self.device, x0.shape[0]
            sl = {"key": key,
                  "a": torch.empty(x0.shape, dtype=torch.float32, device=dev),
                  "b": torch.empty(x1.shape, dtype=torch.float32, device=dev),
                  "g0": torch.empty(x0.shape, dtype=torch.float32, device=dev),
                  "g1": torch.empty((n,) + tuple(x1.shape[1:]), dtype=torch.float32, device=dev),
                  "u_pin": torch.empty(n, dtype=torch.float64, pin_memory=True),
                  "u": torch.empty(n, dtype=torch.float64, device=dev)}
            self._slots[k] = sl
            if key not in self._primed:
                # Results are handed out as fresh pinned tensors (the caller owns them).  A pinned block torch has
                # not cached yet costs a cudaHostAlloc, which waits for the device to go idle and so serialises
                # the pipeline for the first few batches; grow the cache once, up front, to the number of
                # results that can be alive at a time (in flight + a few held by the caller).
                self._primed.add(key)
                grow = [torch.empty(sh, dtype=torch.float32, pin_memory=True)
                        for _ in range(self.depth + 3) for sh in (sl["g0"].shape, sl["g1"].shape)]
                del grow
        return sl

    def submit(self, x0, x1):
        """Enqueue one host batch; returns immediately unless ``depth`` batches are already in flight."""
        for x in (x0, x1):
            if not torch.is_tensor(x) or x.is_cuda or x.dtype != torch.float32 or x.requires_grad:
                raise TypeError("CouplingStream takes CPU float32 tensors that do not require grad; "
                                "device batches need no pipeline (call sample_plan)")
        while len(self._inflight) >= self.depth:
            self._ready.append(self._wait_oldest())
        s, dev = self.sampler, self.device
        sl = self._slot(x0, x1)
        a, b, u = sl["a"], sl["b"], sl["u"]
        # the draw's uniforms: consumed from the NumPy stream now (submission order), staged through pinned
        # memory so that no pageable copy blocks the host behind the running solve
        sl["u_pin"].copy_(torch.from_numpy(np.random.random_sample(x0.shape[0])))
        with torch.cuda.stream(self._up):
            a.copy_(x0, non_blocking=True)
            b.copy_(x1, non_blocking=True)
            u.copy_(sl["u_pin"], non_blocking=True)
            uploaded = torch.cuda.Event()
            uploaded.record(self._up)
        with torch.cuda.stream(self._run):
            self._run.wait_event(uploaded)
            cp = s._couple(a, b, dev)
            i, j = s._draw(cp, x0.shape[0], u)
            g0 = s._gather(a, i, sl["g0"])
            g1 = s._gather(b, j, sl["g1"])
            coupled = torch.cuda.Event()
            coupled.record(self._run)
        with torch.cuda.stream(self._down):
            self._down.wait_event(coupled)
            h0 = torch.empty(g0.shape, dtype=g0.dtype, pin_memory=True)
            h1 = torch.empty(g1.shape, dtype=g1.dtype, pin_memory=True)
            h0.copy_(g0, non_blocking=True)
            h1.copy_(g1, non_blocking=True)
            done = torch.cuda.Event()
            done.record(self._down)
        self._inflight.append((done, h0, h1, cp))

    def _wait_oldest(self):
        done, h0, h1, cp = self._inflight.pop(0)
        done.synchronize()
        self.sampler._report(cp)  # the batch has completed: reading its status word costs no wait
        return h0, h1

    def pending(self):
        return len(self._inflight) + len(self._ready)

    def collect(self):
        """Coupled (x0[i], x1[j]) of the oldest outstanding batch, as pinned CPU tensors."""
        if self._ready:
            return self._ready.pop(0)
        if not self._inflight:
            raise RuntimeError("CouplingStream.collect() with nothing submitted")
        return self._wait_oldest()

    def map(self, batches):
        """Generator: yields the coupled pair of every (x0, x1) in ``batches``, in order."""
        for x0, x1 in batches:
            self.submit(x0, x1)
            while self.pending() >= self.depth:
                yield self.collect()
        while self.pending():
            yield self.collect()
