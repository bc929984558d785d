"""TEST INFRASTRUCTURE ONLY -- float64 restatement of torchsde's fixed-step Euler and of cfm_b200's noise stream.

* ``step_grid`` / ``euler_sdeint``: torchsde.sdeint(sde, y0, ts, bm, method="euler", dt=dt) for an Ito SDE with
  diagonal noise of constant scale sigma, as the SF2M examples call it (examples/2D_tutorials/SF2M_tutorial.ipynb
  cell 5).  torchsde is NOT in the reference tree and not installed; the driver is restated from its published source
  (_core/base_solver.py::BaseSDESolver.integrate, _core/methods/euler.py, _core/interp.py::linear_interp).  The grid
  is accumulated in ts's dtype with torch scalar arithmetic, as torchsde does; the state is float64.  The output
  interpolation is written a * y0 + b * y1, which gives y1 exactly at a grid point.  PARITY UNPINNED: no torchsde
  trajectory exists to compare against.
* ``philox4x32_10`` / ``device_normals``: NumPy restatement of the increments the CUDA kernel draws when no
  Brownian motion is supplied (Philox4x32-10, 24-bit uniforms, Box-Muller), in float64 after the uniforms.
"""
import numpy as np
import torch


def step_grid(ts, dt):
    """The step times torchsde's fixed-step loop visits, as 0-d tensors in ts's dtype, and for every output k >= 1
    the index n of the step (t_n, t_{n+1}) that brackets ts[k]."""
    curr_t = ts[0]
    grid = [curr_t]
    bracket = []
    for out_t in ts[1:]:
        while curr_t < out_t:
            next_t = min(curr_t + dt, ts[-1])
            grid.append(next_t)
            curr_t = next_t
        bracket.append(len(grid) - 2)
    return grid, bracket


def linear_interp(t0, y0, t1, y1, t):
    t0, t1, t = float(t0), float(t1), float(t)
    a = (t1 - t) / (t1 - t0)
    b = (t - t0) / (t1 - t0)
    return a * y0 + b * y1


@torch.no_grad()
def euler_sdeint(f, sigma, y0, ts, dt, increments):
    """ys (len(ts), B, D) float64 of y_{n+1} = y_n + f(t_n, y_n) h_n + sigma dW_n, h_n = t_{n+1} - t_n in ts's dtype.
    ``f(t, y)``: float64 drift (t a Python float); ``increments``: (n_steps, B, D), dW_n = increments[n]."""
    grid, _ = step_grid(ts, dt)
    increments = torch.as_tensor(increments).double()
    assert increments.shape[0] == len(grid) - 1, (increments.shape, len(grid))
    prev_t = curr_t = ts[0]
    prev_y = curr_y = y0.double()
    ys = [curr_y]
    n = 0
    for out_t in ts[1:]:
        while curr_t < out_t:
            next_t = min(curr_t + dt, ts[-1])
            h = float(next_t - curr_t)
            prev_t, prev_y = curr_t, curr_y
            curr_y = curr_y + f(float(curr_t), curr_y) * h + sigma * increments[n]
            curr_t = next_t
            n += 1
        ys.append(linear_interp(prev_t, prev_y, curr_t, curr_y, out_t))
    return torch.stack(ys)


# ---- Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11) -----------------------
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: (..., 4), key: (..., 2) uint32 arrays (broadcast) -> (..., 4) uint32."""
    c = [np.asarray(ctr, dtype=np.uint64)[..., i] for i in range(4)]
    k = [np.asarray(key, dtype=np.uint64)[..., i] for i in range(2)]
    for r in range(10):
        if r:
            k = [(k[0] + np.uint64(_W0)) & _MASK, (k[1] + np.uint64(_W1)) & _MASK]
        p0 = np.uint64(_M0) * c[0]
        p1 = np.uint64(_M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & _MASK, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & _MASK]
    return np.stack(c, axis=-1).astype(np.uint32)


def device_normals(seed, n, rows, cols):
    """The standard normals the SDE kernel uses at step n: (len(rows), cols) float64.  Counter (c // 4, r mod 2^32,
    r >> 32, n), key (seed mod 2^32, seed >> 32); u = (x >> 8) 2^-24 + 2^-25; Box-Muller on (u0, u1) for columns
    4q, 4q + 1 (cos, sin) and on (u2, u3) for 4q + 2, 4q + 3."""
    rows = np.asarray(rows, dtype=np.uint64)[:, None]
    c = np.arange(cols, dtype=np.uint64)[None, :]
    ctr = np.stack(np.broadcast_arrays(c >> np.uint64(2), rows & _MASK, rows >> np.uint64(32),
                                       np.full_like(c, n)), axis=-1)
    key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64)
    x = philox4x32_10(ctr, key)
    u = (x >> np.uint32(8)).astype(np.float64) * 2.0**-24 + 2.0**-25
    hi = (c & np.uint64(2)).astype(bool)
    ua = np.where(hi, u[..., 2], u[..., 0])
    ub = np.where(hi, u[..., 3], u[..., 1])
    rad = np.sqrt(-2.0 * np.log(ua))
    odd = (c & np.uint64(1)).astype(bool)
    return rad * np.where(odd, np.sin(2 * np.pi * ub), np.cos(2 * np.pi * ub))
