"""Hutchinson likelihood of wide MLP flows without a device: the probe restatement (tests/cnf_tc_oracle.py) against
the bit rule and the reference's estimator, the probe ordinals the oracle drivers assign against torchdyn's evaluation
count, the compiled kernels, argument errors of the C entry points (returned before any CUDA call) and the wrapper's
refusals."""
import ctypes
import re
import subprocess

import numpy as np
import pytest
import torch

import cnf_oracle as co
import cnf_tc_oracle as ho
from oracle import sde as osde
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

ERR_ARG = -1  # CFM_ERR_ARG


def test_rademacher_restatement_draws_the_top_bit_of_philox_word_c_mod_4():
    seed, n = 0x1234_5678_9ABC_DEF0 & (2**63 - 1), 7
    rows = np.array([0, 1, 5, 2**32 + 3])
    eps = ho.device_rademacher(seed, n, rows, 12)
    assert eps.shape == (4, 12) and set(np.unique(eps)) <= {-1.0, 1.0}
    for i, r in enumerate(rows):
        for c in range(12):
            ctr = np.array([c // 4, r & 0xFFFFFFFF, r >> 32, n], dtype=np.uint64)
            key = np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint64)
            word = int(osde.philox4x32_10(ctr, key)[c % 4])
            assert eps[i, c] == (-1.0 if word >> 31 else 1.0)
    # a fair sign: 2^16 draws lie within 5 standard deviations of half positive
    big = ho.device_rademacher(3, 0, np.arange(256), 256)
    assert abs((big > 0).mean() - 0.5) < 5 * 0.5 / 256
    # a row's probes do not depend on the rows drawn beside it
    assert np.array_equal(ho.device_rademacher(3, 0, np.array([17]), 256)[0], big[17])
    g = ho.device_probes("hutch_gaussian", seed, n, rows, 12)
    assert np.array_equal(g, osde.device_normals(seed, n, rows, 12))


def _mlp(dim, w, seed, act="selu"):
    torch.manual_seed(seed)
    m = vf.make_mlp(dim, w=w, time_varying=True, dtype=torch.float64)
    if act == "silu":
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("est", ["hutch_gaussian", "hutch_rademacher"])
def test_forward_mode_field_equals_the_reference_vjp_formulation(est, act):
    m = _mlp(16, 32, 1, act)
    x = torch.randn(9, 16, dtype=torch.float64, generator=torch.Generator().manual_seed(2))
    t = torch.tensor(0.37, dtype=torch.float64)
    eps = torch.from_numpy(ho.device_probes(est, 99, 4, np.arange(9), 16))
    f, div = ho.hutch_div(m, t, x, eps)
    ref = ho.reference_div(m, t, x, eps)
    assert torch.allclose(div, ref, rtol=1e-12, atol=1e-12)
    assert torch.allclose(f, vf.wrapped_forward(m, t, x), rtol=0, atol=1e-13)
    # the probes e_k summed over k give the exact trace (cnf_oracle's jacrev field)
    eye = torch.eye(16, dtype=torch.float64)
    tr = sum(ho.hutch_div(m, t, x, eye[k].expand(9, 16))[1] for k in range(16))
    exact = co.cnf_field(m)(t, torch.cat([x, torch.zeros(9, 1, dtype=torch.float64)], 1))[:, -1]
    assert torch.allclose(tr, exact, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("direction", ["forward", "reverse"])
def test_probe_ordinals_follow_torchdyns_evaluation_count(direction):
    m = _mlp(8, 16, 3)
    z = torch.cat([torch.randn(6, 8, dtype=torch.float64, generator=torch.Generator().manual_seed(4)),
                   torch.zeros(6, 1, dtype=torch.float64)], 1)
    span = torch.linspace(0, 1, 3, dtype=torch.float64)
    span = span.flip(0) if direction == "reverse" else span
    pe = ho.Probes("hutch_rademacher", 5, 6, 8)
    co.euler_any_direction(ho.hutch_field(m, pe), z, span)
    assert pe.n == span.numel() - 1
    pd = ho.Probes("hutch_gaussian", 5, 6, 8)
    _, st = co.dopri5_any_direction(ho.hutch_field(m, pd), z, span, 1e-3, 1e-3)
    assert st["rejected"] + st["accepted"] > 2
    assert pd.n == st["nfe"] == 2 + 6 * (st["accepted"] + st["rejected"])


def test_new_kernels_are_built_for_sm90a_without_spills(lib_built):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", lib_built], capture_output=True,
                         text=True).stdout
    blocks = re.findall(r"Fatbin elf code:\n=+\narch = (sm_\w+)(.*?)(?=Fatbin|\Z)", out, flags=re.S)
    found = {}
    for arch, body in blocks:
        for name, usage in re.findall(r"Function (\S+):\n\s*(REG:\d+ STACK:\d+[^\n]*)", body):
            if "cnf_tc_cu" in name:
                found[name] = (arch, usage)
    wanted = ["cnf_probe_kernel", "cnf_fold_kernel", "cnf_euler_init_kernel", "cnf_euler_step_kernel",
              "cnf_gemm_kernelINS0_12CnfPrimalEpi", "cnf_gemm_kernelINS0_13CnfTangentEpi"]
    for w in wanted:
        hits = [v for k, v in found.items() if w in k]
        assert len(hits) == 1, (w, sorted(found))
        arch, usage = hits[0]
        assert arch == "sm_90a", (w, arch)
        assert "STACK:0 " in usage and "LOCAL:0 " in usage, (w, usage)
    assert len(found) == len(wanted), sorted(found)


def test_state_struct_matches_the_header():
    assert ctypes.sizeof(_ffi.CnfTcState) == 40
    assert (_ffi.CnfTcState.n.offset, _ffi.CnfTcState.t.offset) == (24, 32)


def test_entry_points_check_arguments_before_any_cuda_call(lib_built):
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(1 << 12)
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    q = p + 4  # 4-byte aligned only
    big = 1 << 40

    def field(**kw):
        a = dict(prepared=p, x=p, x_hi=None, x_lo=None, batch=256, dim=64, w=128, act=0, est=0, t=p, seed=p, n=p,
                 off=0, f=p, div=p, ws=p, wsb=big, stream=None)
        a.update(kw)
        return lib.cfm_cnf_tc_field_f32(*a.values())

    cases = [(dict(prepared=None), "null pointer"), (dict(seed=None), "null pointer"),
             (dict(x_hi=p, x_lo=p), "either x or the pair"), (dict(x=None, x_hi=p), "either x or the pair"),
             (dict(act=7), "unknown activation"), (dict(est=2), "unknown estimator"),
             (dict(batch=127), "unsupported shape"), (dict(dim=60), "unsupported shape"),
             (dict(w=36), "unsupported shape"), (dict(wsb=16), "workspace too small"),
             (dict(x=q), "16-byte aligned"), (dict(ws=q), "16-byte aligned"), (dict(f=q + 1), "4-byte aligned")]
    for kw, text in cases:
        assert field(**kw) == ERR_ARG, kw
        assert text.encode() in lib.cfm_last_error(), (kw, lib.cfm_last_error())
    assert lib.cfm_cnf_tc_euler_init(None, p, p, p, p, p, p, p, 3, 1, 256, 64, None) == ERR_ARG
    assert lib.cfm_cnf_tc_euler_init(p, p, p, p, p, p, p, p, 1, 1, 256, 64, None) == ERR_ARG
    assert lib.cfm_cnf_tc_euler_init(p, p, q, p, p, p, p, p, 3, 1, 256, 64, None) == ERR_ARG
    assert lib.cfm_cnf_tc_euler_step(p, p, p, p, p, p, p, 256, 20, None) == ERR_ARG
    assert lib.cfm_cnf_tc_euler_step(p, p, p, q, p, p, p, 256, 64, None) == ERR_ARG
    assert lib.cfm_cnf_tc_euler_step(p, p, p, p, None, p, p, 256, 64, None) == ERR_ARG
    assert lib.cfm_cnf_tc_supported(256, 784, 256) and not lib.cfm_cnf_tc_supported(256, 2, 64)
    assert lib.cfm_cnf_tc_workspace_bytes(64, 784, 256) == 0 < lib.cfm_cnf_tc_workspace_bytes(128, 784, 256)


def test_refusals_without_a_device():
    small = cfm_b200.MLP(dim=2, w=64, time_varying=True)
    for grad in (True, False):
        with torch.set_grad_enabled(grad):
            for est in ("hutch_gaussian", "hutch_rademacher"):
                node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(small, likelihood_estimator=est), solver="euler")
                with pytest.raises(NotImplementedError, match="Hutchinson.*exact trace costs only dim tangents"):
                    node.trajectory(torch.zeros(256, 3), torch.linspace(1, 0, 3))
    wide = cfm_b200.MLP(dim=64, w=128, time_varying=True)
    node = cfm_b200.NeuralODE(cfm_b200.cnf_wrapper(wide, likelihood_estimator="hutch_gaussian"), solver="euler")
    with pytest.raises(NotImplementedError, match="B=64"):  # below the class's batch floor
        node.trajectory(torch.zeros(64, 65), torch.linspace(1, 0, 3))
    with pytest.raises(_ffi.CfmLibraryError, match="needs CUDA inputs"):  # in the class: no CPU fallback
        node.trajectory(torch.zeros(256, 65), torch.linspace(1, 0, 3))
    assert "Hutchinson" in node._cnf_backward_gap(wide, torch.zeros(256, 65))
