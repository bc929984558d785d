"""The 3-byte Sinkhorn stream with slab chunks resident in shared memory (sinkhorn_v2.cu).  After the prologue the
kernel keeps a run of K slab chunks from the middle of the slab in shared memory for the whole solve and streams
only the rest through a STAGES-deep ring.  These shapes set the number of streamed chunks per sweep against the ring depth: 0 (the whole
slab resident, its last chunk short of R rows), 1, STAGES - 1, STAGES and STAGES + 1, at each kernel instantiation
where the shape can reach it.  A shape streams only when its fp32 M exceeds 3/4 of the L2, and then a slab takes
about as many chunks as fit in shared memory, so fewer streamed chunks than STAGES need the small chunks of a narrow
n1 (the 8-row instantiation).  The shapes are computed from the device's SM count, L2 size and shared memory by the
launcher's rule."""
import numpy as np
import pytest
import torch

from cfm_b200 import _ffi
from test_gpu_sinkhorn_compact import _cost, _solve
from test_gpu_sinkhorn_compact import test_compact_stream_against_generic_kernel_and_float64_oracle as _against_oracle

DEV = "cuda:0"
STAGES = 2          # kV2QStages: depth of the 3-byte ring
STATIC_SMEM = 4352  # the kernel's static shared memory (ptxas -v)


def _rows_per_chunk(n1):
    return 2 if n1 > 4096 else 4 if n1 > 2048 else 8


def _streamed_chunks(n0, n1):
    """(streamed chunks per sweep of the longest slab, rows of its last chunk), by the launcher's rule."""
    props = torch.cuda.get_device_properties(0)
    R = _rows_per_chunk(n1)
    head = (2 * R * 16 * 8 + (9 + STAGES) * 8 + 127) // 128 * 128
    ldc = (3 * n1 + 15) // 16 * 16
    kmax = (props.shared_memory_per_block_optin - STATIC_SMEM - head) // (R * ldc) - STAGES
    rows = -(-n0 // min(props.multi_processor_count, n0))
    nchunks = -(-rows // R)
    return nchunks - min(kmax, nchunks), rows - (nchunks - 1) * R


def _shape(n1_max, streamed):
    """The widest n1 <= n1_max of the instantiation and a streaming n0 whose longest slab streams `streamed` chunks
    per sweep (streamed = 0: a whole slab resident, with a short last chunk)."""
    props = torch.cuda.get_device_properties(0)
    n1_min = n1_max // 2 + 4 if n1_max > 2048 else 4
    step = props.multi_processor_count * _rows_per_chunk(n1_max)
    for n1 in range(n1_max, n1_min - 1, -4):
        n0_min = (props.L2_cache_size // 4 * 3) // (4 * n1) + 1
        for n0 in range(n0_min, n0_min + 4 * step, step // 8 if streamed == 0 else step):
            ns, last_rows = _streamed_chunks(n0, n1)
            if ns == streamed and (streamed > 0 or last_rows < _rows_per_chunk(n1)):
                return n0, n1
    raise AssertionError(f"no streaming shape with {streamed} streamed chunks at n1 <= {n1_max}")


CASES = sorted({(n1_max, s) for n1_max in (8192, 4096) for s in (STAGES, STAGES + 1)}
               | {(2048, s) for s in (0, 1, STAGES - 1, STAGES, STAGES + 1)}, reverse=True)


@pytest.mark.gpu
@pytest.mark.parametrize("n1_max,streamed", CASES)
def test_resident_chunks_against_generic_kernel_and_float64_oracle(n1_max, streamed):
    n0, n1 = _shape(n1_max, streamed)
    _against_oracle(n0, n1, 64)


@pytest.mark.gpu
@pytest.mark.parametrize("n1_max,streamed", CASES)
def test_resident_chunks_ignore_stale_workspace(n1_max, streamed):
    """The resident chunks are filled from the 3-byte copy once per solve, after the prologue has written it: zeros,
    ones and another coupling's copy in the workspace must all give the same bits."""
    n0, n1 = _shape(n1_max, streamed)
    _stale_workspace_bits(n0, n1)


@pytest.mark.gpu
def test_resident_chunks_ragged_shape():
    """Slabs of 31 and 32 rows, a 1-row last chunk, a row pitch that is not 3 n1 and partial column groups."""
    _stale_workspace_bits(4097, 4100)


def _stale_workspace_bits(n0, n1):
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
