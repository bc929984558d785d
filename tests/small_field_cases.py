"""TEST INFRASTRUCTURE ONLY -- the edge cases of the one-launch SDE and gradient-field kernels without a device: the
launch rules of sde_small_kernel<U, MAXT> and ode_grad_kernel<U, 256> (csrc/ode_small.cu), restated from the sources;
the cases the GPU tests run (tests/test_gpu_small_field_edges.py); the row positions that matter in each plan; and the
code paths each case reaches.  tests/test_small_field_cases_host.py checks the constants against the source text and
that the table reaches every path in REQUIRED on an H100's 132 SMs and on parts with fewer.

Launch rules:
  * a warp integrates RB = 2 neighbouring rows at a time (a row group); local row j of warp gwarp is row
    (gwarp + (j / RB) * grid * nwarps) * RB + j % RB, so a warp's second group is a second pass over the grid;
  * both planners start at 4 warps per CTA and double while a warp would hold more than one group, up to
    kGradMaxWarps = 8 (gradient field) or kSdeMaxWarps = 16 (SDE); grid = min(ceil(groups / nwarps), SMs);
  * a plan holds at most 1 << 19 groups per warp and 200 KB of shared memory.  The gradient field's planner then halves
    the warps per CTA (its hidden buffers shrink, the per-CTA row state does not) down to one warp; the SDE planner has
    no such fallback and refuses;
  * gradient field: ode_small_plan's layout (kSlots = 9 state rows of dimp floats per row) plus the untransposed W1 and
    W2, dim <= 8, w in {32, 64}; SDE: sde_small_plan (two weight sets, kSdeSlots = 4 state rows per row), dim <= 1024,
    w in {32, 64}.
sdeint runs the small kernel whenever it plans the shape and otherwise the tensor-core class (B >= 128, dim >= 32, dim
and w multiples of 8, w >= 32), or raises.

Batches and dims that depend on the SM count are named and resolved by ``resolve``."""
RB = 2                   # rows per warp evaluation (mlp_small.cuh)
K_SLOTS = 9              # kSlots: x, k1..k7, xnew
K_SDE_SLOTS = 4          # kSdeSlots: y, y before the last step, drift, score
GRAD_MAX_WARPS = 8       # kGradMaxWarps
SDE_MAX_WARPS = 16       # kSdeMaxWarps
SMEM_BUDGET = 200 * 1024
GPW_CAP = 1 << 19        # row groups per warp
MAX_DIM = 1024
H100_SMS = 132


def _up4(n):
    return (n + 3) // 4 * 4


def ode_small_plan(dim, w, nwarps, rpw, cnf=False):
    """{name: float offset, "dimp", "total" (bytes)} of ode_small_plan."""
    s = {"dimp": _up4(dim + (1 if cnf else 0))}
    o = 0
    for name, n in (("wt0", dim * w), ("wtime", w), ("b0", w), ("wt1", w * w), ("b1", w), ("wt2", w * w), ("b2", w),
                    ("wt3", w * dim), ("b3", dim), ("hbuf", nwarps * RB * 2 * w * ((1 + dim) if cnf else 1)),
                    ("xin", nwarps * RB * s["dimp"]), ("state", nwarps * rpw * K_SLOTS * s["dimp"]),
                    ("red", 2 * 3 * 32 + 8)):
        s[name] = o
        o += _up4(n)
    s["total"] = 4 * o
    return s


def grad_smem(dim, w, nwarps, rpw):
    """field_smem_bytes(kGradField, ...): the common layout plus the untransposed W1 and W2."""
    return ode_small_plan(dim, w, nwarps, rpw)["total"] + 2 * w * w * 4


def sde_small_plan(dim, w, nwarps, rpw):
    net = ode_small_plan(dim, w, 0, 0)
    set2 = net["hbuf"]
    hbuf = 2 * set2
    state = hbuf + nwarps * RB * 2 * w
    total = 4 * (state + nwarps * rpw * K_SDE_SLOTS * net["dimp"])
    return {"set2": set2, "hbuf": hbuf, "state": state, "total": total}


def _shape(groups, nwarps, sms):
    grid = min(-(-groups // nwarps), sms)
    return grid, -(-groups // (grid * nwarps))


def _first_warps(groups, max_warps, sms):
    nwarps = 4
    while True:
        grid, gpw = _shape(groups, nwarps, sms)
        if gpw == 1 or nwarps == max_warps:
            return nwarps, grid, gpw
        nwarps *= 2


def plan_grad(B, dim, w, sms):
    """(grid, nwarps, rows per warp, smem bytes) of plan_any(..., kGradField), or None where it refuses."""
    if B <= 0 or dim <= 0 or dim > 8 or w not in (32, 64):
        return None
    groups = -(-B // RB)
    nwarps, grid, gpw = _first_warps(groups, GRAD_MAX_WARPS, sms)
    while True:
        if gpw > GPW_CAP:
            return None
        smem = grad_smem(dim, w, nwarps, gpw * RB)
        if smem <= SMEM_BUDGET:
            return grid, nwarps, gpw * RB, smem
        if nwarps == 1:
            return None
        nwarps //= 2
        grid, gpw = _shape(groups, nwarps, sms)


def plan_sde(B, dim, w, sms):
    """(grid, nwarps, rows per warp, smem bytes) of plan_sde_any, or None where it refuses."""
    if B <= 0 or dim <= 0 or dim > MAX_DIM or w not in (32, 64):
        return None
    nwarps, grid, gpw = _first_warps(-(-B // RB), SDE_MAX_WARPS, sms)
    if gpw > GPW_CAP:
        return None
    smem = sde_small_plan(dim, w, nwarps, gpw * RB)["total"]
    if smem > SMEM_BUDGET:
        return None
    return grid, nwarps, gpw * RB, smem


def tc_supported(B, dim, w):
    """sdeint's tensor-core class (cfm_sde_tc_supported, with sdeint's B < 2^31)."""
    return 128 <= B < 2**31 and dim >= 32 and dim % 8 == 0 and w >= 32 and w % 8 == 0


def _largest(ok, lo, hi):
    """Largest n in [lo, hi) with ok(n), given ok(lo) and not ok(hi), by bisection."""
    assert ok(lo) and not ok(hi), (lo, hi)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if ok(mid) else (lo, mid)
    return lo


def grad_bmax(dim, w, sms):
    return _largest(lambda B: plan_grad(B, dim, w, sms) is not None, 1, 1 << 26)


def sde_bmax(dim, w, sms):
    return _largest(lambda B: plan_sde(B, dim, w, sms) is not None, 1, 1 << 26)


def sde_dmax(w, sms, B=1):
    return _largest(lambda d: plan_sde(B, d, w, sms) is not None, 1, MAX_DIM + 1)


def grad_fallback_batch(dim, w, nwarps, sms):
    """The smallest batch the gradient field plans with ``nwarps`` warps per CTA after falling back from 8 (None if no
    batch does): the first past the largest batch planned with more warps."""
    first8 = RB * 4 * sms + 1  # the first batch with more than 4 groups per CTA: 8 warps
    more = _largest(lambda B: (p := plan_grad(B, dim, w, sms)) is not None and p[1] > nwarps, first8, 1 << 26)
    p = plan_grad(more + 1, dim, w, sms)
    return more + 1 if p is not None and p[1] == nwarps else None


# ---- the cases ------------------------------------------------------------------------------------------------------
# named batches: "bmax" (the largest planned), "bmax+1" (the first refused) and the warp-count batches
def resolve(kind, B, dim, w, sms):
    """The batch a case names on ``sms`` SMs (kind "grad" or "sde")."""
    if isinstance(B, int):
        return B
    bmax = (grad_bmax if kind == "grad" else sde_bmax)(dim, w, sms)
    named = {"bmax": bmax, "bmax+1": bmax + 1,
             "8*SMs-1": 8 * sms - 1,        # 4 warps per CTA, one group each, the last row alone
             "16*SMs-1": 16 * sms - 1,      # 8 warps per CTA
             "32*SMs-1": 32 * sms - 1,      # SDE: 16 warps per CTA, one group each
             "80*SMs+3": 80 * sms + 3}      # SDE: 16 warps per CTA, three groups each
    if B.startswith("fallback"):
        return grad_fallback_batch(dim, w, int(B.split(":")[1]), sms)
    return named[B]


def resolve_dim(w, d, sms):
    return sde_dmax(w, sms) if d == "dmax" else d


# gradient field: every (w, dim) at its largest planned batch (the first refused one raises with no launch); the
# warp-count batches at w in {32, 64}, dim 5: 4 and 8 warps with one group each, then the fewer-warps fallback's 4, 2
# and 1 warp plans (the first batch of each)
GRAD_BMAX = [(w, dim) for w in (32, 64) for dim in range(1, 9)]
GRAD_WARP_BATCHES = ["8*SMs-1", "16*SMs-1", "fallback:4", "fallback:2", "fallback:1"]
GRAD_WARP_SHAPES = [(w, 5, B) for w in (32, 64) for B in GRAD_WARP_BATCHES]
# SDE: (w, dim) at its largest planned batch; dim 64 hands the next batch to the tensor-core class, dims 2, 9, 33 and
# 100 refuse it, "dmax" is the largest dim planned at B = 1
SDE_BMAX = [(w, d) for w in (32, 64) for d in (2, 9, 33, 64, 100, "dmax")]
SDE_WARP_SHAPES = [(w, 3, B) for w in (32, 64) for B in ("8*SMs-1", "16*SMs-1", "32*SMs-1", "80*SMs+3")]
# one-step field dims: both layer-3 branches, dim 8 (the last on the butterfly branch) and 9 (the first lane-strided),
# lanes that loop once (31, 32), twice (33, 63) and three times (65, 100), and the largest planned dim
SDE_FIELD_DIMS = [1, 2, 5, 8, 9, 31, 32, 33, 63, 65, 100, "dmax"]
# own noise on a non-uniform grid (tc_sampler_cases' NOISE_TS / NOISE_DT): both instantiations and a plan whose warps
# hold three row groups
NOISE_SHAPES = [(333, 7, 32, "selu"), (333, 7, 64, "silu"), ("80*SMs+3", 3, 64, "selu")]
# gradient-field dopri5 step for step
GRAD_DOPRI5 = [(w, dim, span) for w in (32, 64) for dim in (1, 5, 8) for span in ((0.0, 1.0), (1.0, 0.0))]


# ---- the row positions ----------------------------------------------------------------------------------------------
def row_of(gwarp, j, grid, nwarps):
    return (gwarp + (j // RB) * grid * nwarps) * RB + j % RB


def edge_rows(B, plan):
    """{position: row} of a plan (grid, nwarps, rpw, smem) at batch B: both rows of the first group, the last CTA's last
    row in its first pass, the first row of a second pass, the batch's last row (alone in its group when B is odd)."""
    grid, nwarps, rpw, _ = plan
    rows = {"first row of a group": 0, "second row of a group": 1,
            "CTA's last row in its first pass": row_of(grid * nwarps - 1, 1, grid, nwarps),
            "batch's last row": B - 1}
    if rpw > RB:
        rows["first row of a second pass"] = row_of(0, RB, grid, nwarps)
    if B % 2:
        rows["lone last row of an odd batch"] = B - 1
    return {k: r for k, r in rows.items() if r < B}


# ---- the paths ------------------------------------------------------------------------------------------------------
def plan_paths(kind, B, plan):
    paths = {f"{kind}: {plan[1]} warps per CTA"}
    if plan[2] > RB:
        paths.add(f"{kind}: 2+ row groups per warp")
    if B % 2:
        paths.add(f"{kind}: odd batch")
    return paths


def reached(sms):
    """{path: [cases reaching it]} of the whole table on ``sms`` SMs."""
    out = {}

    def add(paths, case):
        for p in paths:
            out.setdefault(p, []).append(case)
    for w, dim in GRAD_BMAX:
        B = resolve("grad", "bmax", dim, w, sms)
        add(plan_paths("grad", B, plan_grad(B, dim, w, sms)) | {"grad: largest batch"}, ("grad bmax", w, dim))
        if plan_grad(B + 1, dim, w, sms) is None:
            add({"grad: the next batch refused"}, ("grad bmax+1", w, dim))
    for w, dim, name in GRAD_WARP_SHAPES:
        B = resolve("grad", name, dim, w, sms)
        if B is not None:
            paths = plan_paths("grad", B, plan_grad(B, dim, w, sms))
            if name.startswith("fallback"):
                paths = {p + " (fallback)" if "warps per CTA" in p else p for p in paths}
            add(paths, ("grad warps", w, name))
    for w, d in SDE_BMAX:
        dim = resolve_dim(w, d, sms)
        B = resolve("sde", "bmax", dim, w, sms)
        paths = plan_paths("sde", B, plan_sde(B, dim, w, sms)) | {"sde: largest batch"}
        if plan_sde(B + 1, dim, w, sms) is None:
            paths.add("sde: the next batch runs the tensor-core class" if tc_supported(B + 1, dim, w)
                      else "sde: the next batch refused")
        if d == "dmax" and plan_sde(1, dim + 1, w, sms) is None and not tc_supported(1, dim + 1, w):
            paths.add("sde: the next dim refused")
        add(paths, ("sde bmax", w, d))
    for w, dim, name in SDE_WARP_SHAPES:
        B = resolve("sde", name, dim, w, sms)
        add(plan_paths("sde", B, plan_sde(B, dim, w, sms)), ("sde warps", w, name))
    for d in SDE_FIELD_DIMS:
        for w in (32, 64):
            dim = resolve_dim(w, d, sms)
            lanes = -(-dim // 32)
            add({"sde: layer-3 butterfly branch" if dim <= 8 else f"sde: lane-strided layer 3, {min(lanes, 3)} passes"}
                | ({"sde: dim 8, the last on the butterfly branch"} if dim == 8 else set())
                | ({"sde: dim 9, the first lane-strided"} if dim == 9 else set()), ("sde field", w, d))
    for B, dim, w, _ in NOISE_SHAPES:
        B = resolve("sde", B, dim, w, sms)
        add(plan_paths("sde", B, plan_sde(B, dim, w, sms)) | {f"sde own noise: w = {w}"}, ("noise", B, w))
    return out


REQUIRED = {
    "grad: 4 warps per CTA", "grad: 8 warps per CTA", "grad: 4 warps per CTA (fallback)",
    "grad: 2 warps per CTA (fallback)", "grad: 1 warps per CTA (fallback)", "grad: 2+ row groups per warp",
    "grad: odd batch", "grad: largest batch", "grad: the next batch refused",
    "sde: 4 warps per CTA", "sde: 8 warps per CTA", "sde: 16 warps per CTA", "sde: 2+ row groups per warp",
    "sde: odd batch", "sde: largest batch", "sde: the next batch runs the tensor-core class",
    "sde: the next batch refused", "sde: the next dim refused",
    "sde: layer-3 butterfly branch", "sde: dim 8, the last on the butterfly branch", "sde: dim 9, the first lane-strided",
    "sde: lane-strided layer 3, 1 passes", "sde: lane-strided layer 3, 2 passes", "sde: lane-strided layer 3, 3 passes",
    "sde own noise: w = 32", "sde own noise: w = 64",
}
