"""TEST INFRASTRUCTURE ONLY -- the edge cases of the tensor-core samplers without a device: the launch arithmetic of
the Hutchinson field (cnf_tc.cu on the GEMM core of gemm_tc.cuh / gemm_h3.cuh), of the SDE pair forward
(mlp_pair_h3_kernel, mlp_h3.cu) and of dopri5's stage array (ode.py), restated from the sources; the cases the GPU
tests run (tests/test_gpu_tc_sampler_edges.py and the extended parametrisations of tests/test_gpu_cnf_tc.py and
tests/test_gpu_sde_tc.py); and the code paths each case reaches.  tests/test_tc_sampler_cases_host.py checks that the
table reaches every path in REQUIRED on an H100's 132 SMs and on parts with fewer.

Launch arithmetic:
  * GEMM: 128 x 128 output tiles (kTM, kTN), 64-column K chunks (kHK), tiles walked M-fastest by a persistent grid of
    min(tiles, SMs) CTAs (launch_gemm_wg); CTA c runs tiles c, c + grid, ...
  * epilogue: 32-column chunks, full = col0 + 32 <= n1 (CnfPrimalEpi, CnfTangentEpi); the hidden layers (0..2) write
    act' and the split tangent, the output layer (3) writes f and the float64 partials of div.
  * pair forward: 2 S slabs of 128 rows, S = ceil(B / 128), slab v runs net_of(v) = (v >= S) (0: drift, 1: score),
    grid min(2 S, SMs), CTA c runs slabs c, c + grid, ... in ascending order.
  * dopri5 on the flat [x, ll] state of B (D + 1) floats: stage i's field output k[i] (i = 0..6) starts at byte
    4 i B (D + 1) of the stage array; the field writes f there with ldo = D.

Batches that depend on the SM count are named (BATCH) and resolved by ``batch``."""
import numpy as np
import torch

TM = TN = 128  # kTM, kTN (gemm_tc.cuh)
HK = 64        # kHK (gemm_h3.cuh)
CHUNK = 32     # the epilogue's column chunk (cnf_tc.cu)
SLAB = 128     # rows per slab of the fused forward (mlp_h3.cu)
H100_SMS = 132

BATCH = {
    "128*SMs+1": lambda sms: TM * sms + 1,                      # every GEMM: SMs + 1 M tiles, the last of one row
    "128*ceil(SMs/7)+1": lambda sms: TM * -(-sms // 7) + 1,     # dim 784: 7 N tiles x (ceil(SMs/7) + 1) M tiles
    "64*SMs": lambda sms: 64 * sms,                             # pair: 2 S = SMs slabs, one per CTA
    "64*SMs+1": lambda sms: 64 * sms + 1,                       # pair: 2 S = SMs + 2, a ragged drift slab
    "3*128*SMs-5": lambda sms: 3 * TM * sms - 5,                # pair: 6 slabs per CTA, the last drift slab ragged
}


def batch(B, sms):
    return BATCH[B](sms) if isinstance(B, str) else B


# ---- the cases ------------------------------------------------------------------------------------------------------
# one Hutchinson evaluation, every row against float64 (test_gpu_cnf_tc.py::test_one_evaluation_every_row_...)
FIELD_SHAPES = [(128, 32, 40), (129, 40, 136), (255, 136, 200), (257, 264, 264), (255, 784, 136),
                ("128*SMs+1", 72, 200), ("128*ceil(SMs/7)+1", 784, 256)]
# per-layer weight scales W0..W3 x SCALE_FACTORS: the MNIST shape and a ragged width
SCALE_SHAPES = [(256, 784, 256), (257, 72, 136)]
SCALE_FACTORS = (1.0, 3.0, 0.2, 11.0)
# Euler trajectories (B, dim, w, steps): the shape of the first test, a ragged width, the MNIST shape
EULER_SHAPES = [(256, 64, 128, 20), (257, 72, 200, 20), (257, 784, 256, 4)]
# dopri5 at B (D + 1) = 1, 2 and 3 mod 4 (dim 64, w 128): the stage outputs k[i] at every 4-byte offset mod 16
DOPRI5_SHAPE = (64, 128)
DOPRI5_BATCHES = [256, 129, 130, 131]
# the pair launch against two single launches, w = 256 (the pair kernel's class)
PAIR_SHAPES = [(128, 784, 256), (129, 72, 256), ("64*SMs", 64, 256), ("64*SMs+1", 784, 256),
               ("128*SMs+1", 72, 256), ("3*128*SMs-5", 64, 256)]
# the SDE's own noise against float64: a fused-class and a per-layer shape (B, dim, w, act); an off-grid ts and a dt
# that does not divide the span, so that the step h (and sqrt(h)) changes
NOISE_SHAPES = [(600, 64, 256, "selu"), (300, 72, 136, "silu")]
NOISE_TS = (0.0, 0.0137, 0.05, 0.0501, 0.2, 0.31)
NOISE_DT = 0.07
NOISE_SIGMA = 0.6


def noise_rows(B):
    """The rows the SDE noise test checks: the first three, both sides of every 128-row slab boundary, the last
    three."""
    rows = {0, 1, 2, B - 3, B - 2, B - 1}
    for edge in range(SLAB, B, SLAB):
        rows |= {edge - 1, edge}
    return np.array(sorted(rows))


# ---- the paths ------------------------------------------------------------------------------------------------------
def gemm_launch(n0, n1, sms):
    """(tiles_m, tiles_n, grid) of one GEMM with n0 rows and n1 output columns."""
    tiles_m, tiles_n = -(-n0 // TM), -(-n1 // TN)
    return tiles_m, tiles_n, min(tiles_m * tiles_n, sms)


def field_paths(B, dim, w, sms):
    """The paths one evaluation of cfm_cnf_tc_field_f32 at (B, dim, w) reaches on ``sms`` SMs."""
    paths = set()
    for l in range(4):
        K, n1 = (dim if l == 0 else w), (w if l < 3 else dim)
        layer = "hidden" if l < 3 else "output"
        tiles_m, tiles_n, grid = gemm_launch(B, n1, sms)
        if n1 % CHUNK:
            paths |= {f"partial {layer} chunk: primal", f"partial {layer} chunk: tangent"}
        if n1 % TN == 8:
            paths.add(f"8-column {layer} N tile")
        if K % HK:
            paths.add("layer-0 K tail" if l == 0 else "hidden K tail")
        if tiles_m * tiles_n > grid:
            paths |= {f"CTA runs 2+ tiles: primal {layer}", f"CTA runs 2+ tiles: tangent {layer}"}
    if B % TM == 1:
        paths.add("one-row last M tile")
    return paths


def stage_offsets(B, D):
    """The byte offsets mod 16 of dopri5's stage outputs k[0..6] (and so of f) on the flat [x, ll] state."""
    return sorted({4 * i * B * (D + 1) % 16 for i in range(7)})


def dopri5_paths(B, D):
    return {f"k[i] at byte offset {o} mod 16" for o in stage_offsets(B, D) if o}


def pair_slabs(B, sms):
    """(S, grid, per-CTA slab sequences [[(net, slab, rows)]]) of one pair launch."""
    S = -(-B // SLAB)
    grid = min(2 * S, sms)
    seqs = []
    for c in range(grid):
        seq = []
        for v in range(c, 2 * S, grid):
            net = int(v >= S)
            slab = v - net * S
            seq.append((net, slab, min(SLAB, B - slab * SLAB)))
        seqs.append(seq)
    return S, grid, seqs


def pair_paths(B, sms):
    S, grid, seqs = pair_slabs(B, sms)
    paths = set()
    if S == 1:
        paths.add("pair: S = 1")
    if 2 * S == grid == sms:
        paths.add("pair: 2S = grid = SMs")
    if 2 * S == grid + 2:
        paths.add("pair: 2S = grid + 2")
    if S >= sms:
        paths.add("pair: S >= SMs")
    for seq in seqs:
        nets = [net for net, _, _ in seq]
        if nets.count(0) >= 2 and 1 in nets:
            paths.add("pair: two drift slabs, then a score slab, on one CTA")
        for (n0, _, r0), (n1, _, _) in zip(seq, seq[1:]):
            if n0 == 0 and r0 < SLAB and n1 == 1:
                paths.add("pair: a ragged drift slab, then a score slab, on one CTA")
    return paths


def sde_grid(ts, dt):
    """The fp32 step grid sdeint's tensor-core class walks (cfm_b200.sde.step_schedule)."""
    from cfm_b200 import sde as csde
    return csde.step_schedule(torch.tensor(ts, dtype=torch.float32), dt)[0].astype(np.float32)


def noise_paths(ts, dt):
    g = sde_grid(ts, dt)
    roots = np.sqrt(g[1:] - g[:-1], dtype=np.float32)
    return {"SDE: sqrt(h) of a later step differs from the first step's"} if bool((roots[1:] != roots[0]).any()) \
        else set()


def reached(sms):
    """{path: [cases reaching it]} of the whole table on ``sms`` SMs."""
    out = {}

    def add(paths, case):
        for p in paths:
            out.setdefault(p, []).append(case)
    for B, dim, w in FIELD_SHAPES + SCALE_SHAPES:
        add(field_paths(batch(B, sms), dim, w, sms), ("field", B, dim, w))
    for B, dim, w, _ in EULER_SHAPES:
        add(field_paths(B, dim, w, sms), ("euler", B, dim, w))
    for B in DOPRI5_BATCHES:
        add(field_paths(B, *DOPRI5_SHAPE, sms) | dopri5_paths(B, DOPRI5_SHAPE[0]), ("dopri5", B))
    for B, dim, w in PAIR_SHAPES:
        add(pair_paths(batch(B, sms), sms), ("pair", B, dim))
    add(noise_paths(NOISE_TS, NOISE_DT), ("noise", NOISE_TS, NOISE_DT))
    return out


REQUIRED = {
    "partial hidden chunk: primal", "partial hidden chunk: tangent",
    "8-column hidden N tile", "8-column output N tile",
    "hidden K tail", "layer-0 K tail",
    "CTA runs 2+ tiles: primal hidden", "CTA runs 2+ tiles: tangent hidden",
    "CTA runs 2+ tiles: primal output", "CTA runs 2+ tiles: tangent output",
    "one-row last M tile",
    "k[i] at byte offset 4 mod 16", "k[i] at byte offset 8 mod 16", "k[i] at byte offset 12 mod 16",
    "pair: S = 1", "pair: 2S = grid = SMs", "pair: 2S = grid + 2", "pair: S >= SMs",
    "pair: two drift slabs, then a score slab, on one CTA",
    "pair: a ragged drift slab, then a score slab, on one CTA",
    "SDE: sqrt(h) of a later step differs from the first step's",
}

