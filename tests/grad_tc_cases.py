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
    for B, dim, w in FIELD_SHAPES + SCALE_SHAPES:
        add(field_paths(batch(B, sms), dim, w, sms), ("field", B, dim, w))
    for B, dim, w in EULER_SHAPES + DOPRI5_CASES:
        add(field_paths(B, dim, w, sms), ("trajectory", B, dim, w))
    add(offset_paths(V_OFFSETS), ("offsets",) + OFFSET_SHAPE)
    return out


REQUIRED = {
    "partial chunk at N = dim", "partial chunk at N = w",
    "K tail at K = dim", "K tail at K = w",
    "CTA runs 2+ tiles: N = dim", "CTA runs 2+ tiles: N = w",
    "one-row last M tile",
    "v at byte offset 4 mod 16", "v at byte offset 8 mod 16", "v at byte offset 12 mod 16",
}
