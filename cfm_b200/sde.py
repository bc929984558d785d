"""Schrodinger-bridge SDE sampling on the device: drop-in for the way the SF2M examples use torchsde,

    sde = SDE(model, score_model, input_size=(2,), sigma=sigma)
    with torch.no_grad():
        sde_traj = torchsde.sdeint(sde, x0, ts=torch.linspace(0, 1, 100), method="euler")

(examples/2D_tutorials/SF2M_tutorial.ipynb cell 5, examples/single_cell/single-cell_example.ipynb cell 16).  torchsde
is an un-vendored dependency; its fixed-step Euler (the step grid, the update and the linear interpolation onto
``ts``) is restated in oracle/sde.py and implemented here: the host tabulates the step grid and the output
interpolation once per ``(ts, dt)``.  Two classes of nets run on the device:

* small nets (w in {32, 64}, both weight sets and the per-row state in shared memory; the 2-D and single-cell
  tutorials): ONE kernel (csrc/ode_small.cu, ``sde_small_kernel``) takes every step, both MLP evaluations per step,
  the noise and the output writes;
* wide nets in the tensor-core class (B >= 128, dim >= 32, dim and w multiples of 8; e.g. the MNIST notebook's
  ``MLP(784, w=256)``): per step, ONE launch of both nets' fused fp16x3 forward on the state's operand pair
  (csrc/mlp_h3.cu; per-layer launches for other widths) and ONE elementwise step kernel (csrc/sde_tc.cu).  The step
  index, time and pointers live in a device struct, so the step is captured once as a CUDA graph and replayed for
  the whole trajectory, with no host round trip.

Only the SF2M shape is accelerated: a ``cfm_b200.SDE`` whose drift and score are ``cfm_b200.MLP(time_varying=True)``
of one shape, a CUDA ``(B, D)`` state and ``method="euler"``.  Anything else raises -- there is no eager fallback.

Noise: torchsde's BrownianInterval stream is not reproduced.  Without ``bm`` the kernel draws its own increments
from a counter-based generator (Philox4x32-10 + Box-Muller, keyed by one 63-bit seed taken from torch's default CPU
generator per call), so ``torch.manual_seed`` reproduces a trajectory and the noise of a row does not depend on the
batch size, the launch shape or the class: a given (seed, step, row, column) draws the same increment in both.
With ``bm`` (a torchsde-style callable ``bm(ta, tb)``) the increments are the
caller's, read from device memory.
"""
import ctypes as C

import numpy as np
import torch

from . import _ffi
from .models import MLP, SDE

_MAX_TABLES = 16
_tables = {}  # (ts dtype, ts bytes, dt, device) -> (grid, out_begin, out_a, out_b, grid as a CPU tensor in ts's dtype)
_MAX_PLANS = 4
_plans = {}   # tensor-core class: plan key (see _tc_plan) -> buffers and the captured step graph
_EAGER = False  # tests: enqueue every step of the tensor-core class eagerly instead of replaying the captured graph


def _refuse_options(method, adaptive, logqp, unsupported):
    if "solver" in unsupported:
        raise NotImplementedError(
            "sdeint has no `solver` argument: torchsde ignores it and integrates with its default method (SRK for Ito "
            "diagonal noise), which cfm_b200 does not provide; pass method='euler' for Euler-Maruyama")
    if unsupported:
        raise NotImplementedError(f"sdeint: unsupported arguments {sorted(unsupported)}")
    if method is None:
        raise NotImplementedError(
            "sdeint(method=None): torchsde's default for Ito SDEs with diagonal noise is SRK, which cfm_b200 does not "
            "provide; pass method='euler' for fixed-step Euler-Maruyama")
    if method != "euler":
        raise NotImplementedError(f"sdeint(method={method!r}): the CUDA path provides method='euler' only")
    if adaptive:
        raise NotImplementedError("sdeint(adaptive=True): the CUDA path takes fixed steps only")
    if logqp:
        raise NotImplementedError("sdeint(logqp=True) is not supported")


def _nets(sde):
    if not isinstance(sde, SDE):
        raise TypeError(f"cfm_b200.sdeint accelerates cfm_b200.SDE; got {type(sde).__name__}")
    d, s = sde.drift, sde.score
    for name, m in (("drift", d), ("score", s)):
        if not isinstance(m, MLP) or not m.time_varying:
            raise TypeError(f"cfm_b200.sdeint: the {name} net must be cfm_b200.MLP(time_varying=True); got "
                            f"{type(m).__name__}")
    size = int(np.prod(sde.input_size))
    if not (d.dim == d.out_dim == s.dim == s.out_dim == size and d.w == s.w and d.act == s.act):
        raise TypeError(
            "cfm_b200.sdeint: drift and score must have dim == out_dim == prod(input_size) and equal w and act; got "
            f"drift (dim={d.dim}, out_dim={d.out_dim}, w={d.w}, act={d.act}), score (dim={s.dim}, out_dim={s.out_dim}, "
            f"w={s.w}, act={s.act}), input_size={tuple(sde.input_size)}")
    return d, s


def step_schedule(ts, dt):
    """torchsde's fixed-step grid and output interpolation for ``ts`` (a 1-D CPU float32 / float64 tensor):
    (grid in ts's dtype [n_steps + 1], out_begin int32 [n_steps + 1], a float32 [n_out], b float32 [n_out]).

    The grid starts at ts[0] with t_{n+1} = min(t_n + dt, ts[-1]) in ts's dtype; steps are taken while t_n < ts[k]
    for each output point in turn.  Output k >= 1 is a * y_n + b * y_{n+1} for the step n that ends at or after
    ts[k] (out_begin[n] <= k < out_begin[n + 1]), a = (t_{n+1} - ts[k]) / h, b = (ts[k] - t_n) / h."""
    T = ts.numpy()
    ft = T.dtype.type
    h, t_end = ft(dt), T[-1]
    t = T[0]
    grid = [t]
    bracket = np.empty(len(T) - 1, dtype=np.int64)
    for k in range(1, len(T)):
        while t < T[k]:
            nxt = min(ft(t + h), t_end)
            if not nxt > t:
                raise ValueError(f"sdeint: dt={dt} does not advance t={float(t)} in {T.dtype}")
            grid.append(nxt)
            t = nxt
        bracket[k - 1] = len(grid) - 2
    grid = np.array(grid, dtype=T.dtype)
    n_steps = len(grid) - 1
    out_begin = (1 + np.searchsorted(bracket, np.arange(n_steps + 1), side="left")).astype(np.int32)
    t0, t1, tk = (grid[bracket].astype(np.float64), grid[bracket + 1].astype(np.float64),
                  T[1:].astype(np.float64))
    a = np.zeros(len(T), dtype=np.float32)
    b = np.ones(len(T), dtype=np.float32)
    a[1:] = (t1 - tk) / (t1 - t0)
    b[1:] = (tk - t0) / (t1 - t0)
    return grid, out_begin, a, b


def _tables_for(ts, dt, dev):
    key = (ts.dtype, ts.numpy().tobytes(), float(dt), str(dev))
    hit = _tables.get(key)
    if hit is not None:
        return hit
    grid, out_begin, a, b = step_schedule(ts, dt)
    hit = (torch.from_numpy(grid.astype(np.float32)).to(dev), torch.from_numpy(out_begin).to(dev),
           torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev), torch.from_numpy(grid))
    if len(_tables) >= _MAX_TABLES:
        _tables.pop(next(iter(_tables)))
    _tables[key] = hit
    return hit


@torch.no_grad()
def sdeint(sde, y0, ts, bm=None, method=None, dt=1e-3, adaptive=False, logqp=False, **unsupported):
    """Subset of torchsde.sdeint: fixed-step Euler-Maruyama of a ``cfm_b200.SDE`` with two
    ``MLP(time_varying=True)`` nets.  Returns ``ys`` of shape (len(ts), B, D), fp32, on y0's device.

    ``bm``: optional callable ``bm(ta, tb) -> (B, D)`` Brownian increment, called once per step in order with 0-d
    tensors in ts's dtype on ts's device.  Without it the kernels draw the increments themselves (module docstring).
    Nets in neither class (module docstring) raise ``NotImplementedError``."""
    _refuse_options(method, adaptive, logqp, unsupported)
    drift, score = _nets(sde)
    if not torch.is_tensor(y0) or not y0.is_cuda:
        raise _ffi.CfmLibraryError("cfm_b200.sdeint needs a CUDA y0 (no CPU fallback)")
    if y0.dim() != 2:
        raise ValueError(f"sdeint: y0 must be (B, D); got shape {tuple(y0.shape)}")
    B, D = y0.shape
    if D != drift.dim:
        raise ValueError(f"sdeint: y0 has {D} columns, the nets take {drift.dim}")
    ts = torch.as_tensor(ts)
    if ts.dim() != 1 or ts.numel() < 2:
        raise ValueError("sdeint: ts must be a 1-D tensor of at least two times")
    if ts.dtype not in (torch.float32, torch.float64):
        raise ValueError(f"sdeint: ts must be float32 or float64; got {ts.dtype}")
    ts_host = ts.detach().cpu().contiguous()
    if not bool((ts_host[1:] > ts_host[:-1]).all()):
        raise ValueError("sdeint: ts must be strictly increasing")
    dt = float(dt)
    if not (dt > 0 and np.isfinite(dt)):
        raise ValueError(f"sdeint: dt must be positive and finite; got {dt}")
    L = _ffi.lib()
    small = bool(L.cfm_sde_small_supported(B, D, drift.w))
    if not small and not (B < 2**31 and L.cfm_sde_tc_supported(B, D, drift.w)):
        raise NotImplementedError(
            f"sdeint: no SDE kernel for B={B}, dim={D}, w={drift.w}: it takes cfm_b200.SDE with drift and score "
            "cfm_b200.MLP(time_varying=True) either of w in {32, 64} whose two weight sets and per-row state fit in "
            "shared memory (one kernel), or in the tensor-core class: B >= 128, dim >= 32, dim and w multiples of 8, "
            "w >= 32")
    dev = y0.device
    pd, psc = (drift._device_params(dev), score._device_params(dev)) if small else (None, None)
    with torch.cuda.device(dev):
        tables = _tables_for(ts_host, dt, dev)
        grid, out_begin, out_a, out_b, grid_host = tables
        n_steps = grid.numel() - 1
        inc, seed = None, 0
        if bm is None:
            seed = int(torch.randint(0, 2**63 - 1, (), dtype=torch.int64))
        else:
            steps = grid_host.to(ts.device)
            incs = []
            for n in range(n_steps):
                w = torch.as_tensor(bm(steps[n], steps[n + 1]))
                if tuple(w.shape) != (B, D):
                    raise ValueError(f"sdeint: bm returned shape {tuple(w.shape)}, expected {(B, D)}")
                incs.append(w.to(device=dev, dtype=torch.float32))
            inc = torch.stack(incs).contiguous()
        x0 = y0.detach().float().contiguous()
        ys = torch.empty((ts.numel(), B, D), dtype=torch.float32, device=dev)
        if not small:
            _tc_euler(sde, drift, score, x0, tables, seed, inc, ys)
            return ys
        arr = C.c_void_p * 8  # host arrays of the 8 device pointers of each net
        _ffi.check(L.cfm_sde_small_euler_f32(
            arr(*[p.data_ptr() for p in pd]), arr(*[p.data_ptr() for p in psc]), D, drift.w, drift.act,
            float(sde.sigma), _ffi.ptr(x0), B, _ffi.ptr(grid), n_steps, _ffi.ptr(out_begin), _ffi.ptr(out_a),
            _ffi.ptr(out_b), ts.numel(), seed, _ffi.ptr(inc), _ffi.ptr(ys), _ffi.stream_ptr(dev)),
            "cfm_sde_small_euler_f32")
    return ys


# ---- tensor-core class ------------------------------------------------------------------------------------------------
def _tc_plan(sde, drift, score, B, D, tables, dev):
    """Buffers of one (shape, both nets' prepared weights, tables, sigma, device, stream): the state y, the nets'
    outputs, the operand pair (hi, lo) of y, the device state struct, the pair forward's workspace, and -- once the
    first step has run eagerly -- the CUDA graph of one step.  The graph holds pointers to these buffers, the prepared
    weight blobs and the tables only; per-call pointers (trajectory, increments) reach it through the state struct."""
    L = _ffi.lib()
    # a net's blob is rebuilt when its weights change in place; a plan keeps its blobs and tables alive, so their
    # addresses name them for as long as the plan exists
    blobs = (drift._prepared(True, dev), score._prepared(True, dev))
    key = (B, D, drift.w, drift.act, float(sde.sigma), tuple(t.data_ptr() for t in blobs + tables[:4]), str(dev),
           torch.cuda.current_stream(dev).cuda_stream)
    P = _plans.get(key)
    if P is not None:
        return P
    if len(_plans) >= _MAX_PLANS:
        _plans.pop(next(iter(_plans)))
    f32 = dict(dtype=torch.float32, device=dev)
    st = torch.zeros(C.sizeof(_ffi.SdeState), dtype=torch.uint8, device=dev)
    P = {"blobs": blobs, "tables": tables, "st": st, "y": torch.empty((B, D), **f32),
         "d": torch.empty((B, D), **f32), "s": torch.empty((B, D), **f32),
         "hi": torch.empty((B, D), dtype=torch.float16, device=dev),
         "lo": torch.empty((B, D), dtype=torch.float16, device=dev),
         "ws": _ffi.workspace(2 * L.cfm_mlp_workspace_bytes(B, D, drift.w, D, 2), dev),
         "t_dev": C.c_void_p(st.data_ptr() + _ffi.SdeState.t.offset), "graph": None}
    _plans[key] = P
    return P


def _tc_enqueue_step(sde, drift, P, B, D, dev):
    """One Euler-Maruyama step: both nets at (t_n, y_n) in one pair launch, then the step kernel."""
    L = _ffi.lib()
    sp = _ffi.stream_ptr(dev)
    grid, out_begin, out_a, out_b, _ = P["tables"]
    ws = P["ws"]
    _ffi.check(L.cfm_mlp_pair_forward_split_f32(
        _ffi.ptr(P["blobs"][0]), _ffi.ptr(P["blobs"][1]), _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]), B, D, drift.w, D, 1,
        P["t_dev"], 0.0, drift.act, _ffi.ptr(P["d"]), _ffi.ptr(P["s"]), _ffi.ptr(ws), ws.numel(), sp),
        "cfm_mlp_pair_forward_split_f32")
    _ffi.check(L.cfm_sde_tc_euler_step(
        _ffi.ptr(P["st"]), _ffi.ptr(P["y"]), _ffi.ptr(P["d"]), _ffi.ptr(P["s"]), _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]),
        _ffi.ptr(grid), _ffi.ptr(out_begin), _ffi.ptr(out_a), _ffi.ptr(out_b), float(sde.sigma), B, D, sp),
        "cfm_sde_tc_euler_step")


def _tc_euler(sde, drift, score, x0, tables, seed, inc, ys):
    """The whole trajectory of the tensor-core class into ``ys``: init, then n_steps replays of the step graph (the
    first call of a plan runs step 0 eagerly, which loads every kernel, then captures the step)."""
    L = _ffi.lib()
    dev = x0.device
    B, D = x0.shape
    n_steps = tables[0].numel() - 1
    P = _tc_plan(sde, drift, score, B, D, tables, dev)
    if x0.data_ptr() % 16:
        x0 = x0.clone()
    _ffi.check(L.cfm_sde_tc_init(
        _ffi.ptr(P["st"]), _ffi.ptr(x0), _ffi.ptr(P["y"]), _ffi.ptr(P["hi"]), _ffi.ptr(P["lo"]), _ffi.ptr(ys),
        _ffi.ptr(inc), seed, _ffi.ptr(tables[0]), n_steps, B, D, _ffi.stream_ptr(dev)), "cfm_sde_tc_init")
    _ffi.replay_steps(P, lambda: _tc_enqueue_step(sde, drift, P, B, D, dev), n_steps, not _EAGER)
