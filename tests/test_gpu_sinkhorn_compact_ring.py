"""The 3-byte Sinkhorn stream at its smallest streaming shapes, one per kernel instantiation (n1 = 8192, 4096,
2048).  A slab here has about 5 chunks against a 3-stage ring, so the ring wraps from sweep to sweep within less
than two ring lengths, and the switch from the fp32 prologue to the 3-byte copy falls inside the first ring fill.
The shapes sit just above the point where fp32 M stops fitting in 3/4 of the device's L2 (below it the fp32 sweep
runs)."""
import numpy as np
import pytest
import torch

from cfm_b200 import _ffi
from test_gpu_sinkhorn_compact import _cost, _solve
from test_gpu_sinkhorn_compact import test_compact_stream_against_generic_kernel_and_float64_oracle as _against_oracle

DEV = "cuda:0"


def _smallest_streaming_n0(n1):
    """n0 a little above the largest n0 whose fp32 M (n0 x n1) still fits in 3/4 of the L2."""
    l2 = torch.cuda.get_device_properties(0).L2_cache_size
    return (l2 // 4 * 3) // (4 * n1) + 32 * (8192 // n1)  # 50 MiB L2: 1232, 2464, 4928


@pytest.mark.gpu
@pytest.mark.parametrize("n1", [8192, 4096, 2048])
def test_compact_stream_smallest_streaming_shapes(n1):
    _against_oracle(_smallest_streaming_n0(n1), n1, 64)


@pytest.mark.gpu
def test_compact_stream_ignores_stale_workspace_short_slabs():
    """As test_compact_stream_ignores_stale_workspace, on slabs shorter than two rings: a ring that ran ahead across
    the format switch would issue the first 3-byte chunks before the prologue has written them."""
    n1 = 8192
    n0 = _smallest_streaming_n0(n1)
    M, cmax = _cost(n0, n1, 64, 1)
    M2, cmax2 = _cost(n0, n1, 64, 2)
    ws = _ffi.workspace(_ffi.lib().cfm_sinkhorn_workspace_bytes(n0, n1), torch.device(DEV))
    for iters in (1, 2, 3, 11, 100):
        got = []
        for history in ("zeros", "ones", "other"):
            if history == "zeros":
                ws.fill_(0x00)
            elif history == "ones":
                ws.fill_(0xFF)
            else:
                _, _, st2 = _solve(M2, cmax2, n0, n1, "fp32", 100, ws)
                assert st2[3] == 4
            lu, lv, st = _solve(M, cmax, n0, n1, "fp32", iters, ws)
            assert st[3] == 4 and st[1] == iters
            got.append((lu.cpu().numpy(), lv.cpu().numpy()))
        for lu, lv in got[1:]:
            assert np.array_equal(lu, got[0][0]) and np.array_equal(lv, got[0][1]), iters
