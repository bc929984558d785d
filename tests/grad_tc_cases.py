"""TEST INFRASTRUCTURE ONLY -- the edge cases of the tensor-core gradient field (csrc/grad_tc.cu) without a device: its
launch arithmetic restated from the sources, the cases the GPU tests run (tests/test_gpu_grad_tc.py) and the code paths
each case reaches.  tests/test_grad_tc_host.py checks that the table reaches every path in REQUIRED on an H100's 132
SMs and on parts with 114 and 78.

Launch arithmetic (gemm_tc.cuh, gemm_h3.cuh, grad_tc.cu):
  * one evaluation is six GEMMs on B rows: primal layers 0, 1, 2 (K = dim, w, w; N = w) and reverse GEMMs by W2^T, W1^T
    (K = w, N = w) and W0x^T (K = w, N = dim);
  * each GEMM: 128 x 128 output tiles (kTM, kTN) walked M-fastest by a persistent grid of min(tiles, SMs) CTAs; 64-column
    K chunks (kHK), the last zero-filled past K; the epilogue takes 32-column chunks, full = col0 + 32 <= N;
  * v is written with row stride dim at any 4-byte offset: a chunk goes through the staged coalesced store when it is
    full and its base is 16-byte aligned, element by element otherwise.

Batches that depend on the SM count are named (BATCH) and resolved by ``batch``."""
TM = TN = 128  # kTM, kTN (gemm_tc.cuh)
HK = 64        # kHK (gemm_h3.cuh)
CHUNK = 32     # the epilogue's column chunk (gemm_tc.cuh)

BATCH = {
    "128*SMs+1": lambda sms: TM * sms + 1,                   # every GEMM: SMs + 1 M tiles, the last of one row
    "128*ceil(SMs/7)+1": lambda sms: TM * -(-sms // 7) + 1,  # dim 784: 7 N tiles x (ceil(SMs/7) + 1) M tiles
}


def batch(B, sms):
    return BATCH[B](sms) if isinstance(B, str) else B


# one evaluation, every row against float64, SELU and SiLU (test_gpu_grad_tc.py::test_one_evaluation_every_row_...)
FIELD_SHAPES = [(256, 784, 256), (300, 64, 128), (129, 32, 32),
                (128, 32, 40), (129, 40, 136), (255, 136, 200), (257, 264, 264),
                ("128*SMs+1", 72, 200), ("128*ceil(SMs/7)+1", 784, 256)]
# W0..W2 scaled by each factor (W3 stays): the MNIST shape and a ragged width
SCALE_SHAPES = [(256, 784, 256), (257, 72, 136)]
SCALE_FACTORS = (3.0, 0.2, 11.0)
# v written this many floats into a larger buffer
V_OFFSETS = (1, 2, 3)
OFFSET_SHAPE = (257, 72, 136)
# Per-layer factors (W0, W1, W2, W3) that put the four layers' weights in four different binades, so that every s_l and
# 2^k differ (test_grad_tc_host.py asserts it): each hidden layer is the largest at least once and the smallest at least
# once.  The last set puts s_2 / s_1 at 2^20: the reverse chain's scales are a product, so epilogues that undo each
# other's layer scale give the same v unless the wrong scale moves g1 out of fp16's range, as it does there (SELU).
# Run at the MNIST shape and a ragged width, seed LAYER_SCALE_SEED.
LAYER_SCALE_SHAPES = [(256, 784, 256), (257, 72, 136)]
LAYER_SCALE_SETS = [(1.0, 4.0, 0.25, 16.0), (4.0, 0.25, 1.0, 1 / 16), (0.25, 1.0, 4.0, 16.0),
                    (0.25, 1024.0, 1 / 1024, 16.0)]
LAYER_SCALE_SEED = 7
# Nets whose reverse chain nears or passes fp16's 65504 under the W3-only rule 2^k = s_3 2^-7: (act, factors of
# W0..W3, fraction of 65504 that max|g 2^k| reaches under that rule).  W0..W2 x f grows activations and chain alike;
# W0 / c with W1, W2 x c grows only the chain.  MNIST shape RANGE_SHAPE, seed 7, x seed 8, t = 0.3.
RANGE_SHAPE = (256, 784, 256)
RANGE_CASES = [("silu", (25.0, 25.0, 25.0, 1.0), 0.49), ("selu", (0.05, 20.0, 20.0, 1.0), 0.85),
               ("selu", (30.0, 30.0, 30.0, 1.0), 0.92), ("silu", (50.0, 50.0, 50.0, 1.0), 1.96),
               ("selu", (50.0, 50.0, 50.0, 1.0), 2.23), ("selu", (1 / 52, 52.0, 52.0, 1.0), 4.47)]
# W3 scaled by 2^p: v scales by exactly 2^p.  W3_PAST_CLAMP puts max|W3| at 2^-110, past h3_pow2_scale's exponent
# clamp at +-100; W3 = 0 is a zero-initialised last layer.
W3_POWERS = (-60, -12, 6, 60)
W3_PAST_CLAMP = 2.0 ** -110
W3_SHAPE = (257, 72, 136)
# Rows with SELU pre-activations exactly 0 (kink rows): x = 0 rows at t = 0 with zero biases on all units or on half.
KINK_SHAPE = (256, 64, 128)
KINK_BIASES = ("all", "half")
# Euler spans, each also reversed: non-uniform points and one repeated point (a step with h = 0).
SPANS = {"non-uniform": [0.0, 0.01, 0.03, 0.1, 0.2, 0.45, 0.5, 0.8, 1.0],
         "repeated point": [0.0, 0.25, 0.5, 0.5, 0.75, 1.0]}
SPAN_SHAPE = (257, 72, 200)
# Euler trajectories (B, dim, w) over linspace(0, 1, 100), both directions
EULER_SHAPES = [(1024, 784, 256), (257, 72, 200)]
# dopri5 at 1e-4, both directions: the MNIST shape and odd batches at (dim, w) = (64, 128)
DOPRI5_CASES = [(1024, 784, 256), (129, 64, 128), (130, 64, 128), (131, 64, 128)]


def gemms(dim, w):
    """(name, K, N) of the six GEMMs of one evaluation."""
    return [("primal 0", dim, w), ("primal 1", w, w), ("primal 2", w, w),
            ("reverse 2", w, w), ("reverse 1", w, w), ("reverse 0", w, dim)]


def field_paths(B, dim, w, sms):
    paths = set()
    for name, K, N in gemms(dim, w):
        tiles = -(-B // TM) * -(-N // TN)
        if N % CHUNK:
            paths.add("partial chunk at N = dim" if name == "reverse 0" else "partial chunk at N = w")
        if K % HK:
            paths.add("K tail at K = dim" if name == "primal 0" else "K tail at K = w")
        if tiles > sms:
            paths.add("CTA runs 2+ tiles: N = dim" if name == "reverse 0" else "CTA runs 2+ tiles: N = w")
    if B % TM == 1:
        paths.add("one-row last M tile")
    return paths


def offset_paths(offsets):
    return {f"v at byte offset {4 * o % 16} mod 16" for o in offsets if 4 * o % 16}


def reached(sms):
    """{path: [cases reaching it]} of the whole table on ``sms`` SMs."""
    out = {}

    def add(paths, case):
        for p in paths:
            out.setdefault(p, []).append(case)
    for B, dim, w in FIELD_SHAPES + SCALE_SHAPES + LAYER_SCALE_SHAPES + [RANGE_SHAPE, W3_SHAPE, KINK_SHAPE]:
        add(field_paths(batch(B, sms), dim, w, sms), ("field", B, dim, w))
    for B, dim, w in EULER_SHAPES + DOPRI5_CASES + [SPAN_SHAPE]:
        add(field_paths(B, dim, w, sms), ("trajectory", B, dim, w))
    add(offset_paths(V_OFFSETS), ("offsets",) + OFFSET_SHAPE)
    for f in LAYER_SCALE_SETS:
        add({"four distinct layer scales"}, ("layer scales", f))
    for act, f, frac in RANGE_CASES:
        add({f"chain near 65504: {act}" if frac < 1 else f"chain past 65504: {act}"}, ("range", act, f))
        if f[0] < 1:
            add({"chain grows alone"}, ("range", act, f))
    for p in W3_POWERS:
        add({"W3 2^p below 1" if p < 0 else "W3 2^p above 1"}, ("W3", p))
    add({"W3 past the scale clamp"}, ("W3", W3_PAST_CLAMP))
    add({"W3 = 0"}, ("W3", 0.0))
    for bias in KINK_BIASES:
        add({f"kink rows, {bias} biases zero"}, ("kink", bias))
    for name, sp in SPANS.items():
        steps = [b - a for a, b in zip(sp, sp[1:])]
        if 0.0 in steps:
            add({"Euler step h = 0"}, ("span", name))
        if len(set(round(h, 9) for h in steps)) > 2:
            add({"non-uniform Euler span"}, ("span", name))
    return out


REQUIRED = {
    "partial chunk at N = dim", "partial chunk at N = w",
    "K tail at K = dim", "K tail at K = w",
    "CTA runs 2+ tiles: N = dim", "CTA runs 2+ tiles: N = w",
    "one-row last M tile",
    "v at byte offset 4 mod 16", "v at byte offset 8 mod 16", "v at byte offset 12 mod 16",
    "four distinct layer scales",
    "chain near 65504: selu", "chain near 65504: silu", "chain past 65504: selu", "chain past 65504: silu",
    "chain grows alone",
    "W3 2^p below 1", "W3 2^p above 1", "W3 past the scale clamp", "W3 = 0",
    "kink rows, all biases zero", "kink rows, half biases zero",
    "Euler step h = 0", "non-uniform Euler span",
}


def scaled_action(dim, w, seed, factors=(1.0, 1.0, 1.0, 1.0), act="selu"):
    """cfm_b200.MLP(dim, out_dim=1, w, time_varying=True) on the CPU, seeded, with W0..W3 multiplied by ``factors``."""
    import torch

    import cfm_b200
    from cfm_b200 import _ffi
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True)
    if act == "silu":
        m.act = _ffi.ACT_SILU
    with torch.no_grad():
        for li, f in zip((0, 2, 4, 6), factors):
            m.net[li].weight.mul_(f)
    return m


def range_input(B, dim):
    import torch
    return torch.randn(B, dim, generator=torch.Generator().manual_seed(8))
