"""The tensor-core gradient field of wide scalar actions without a device: the float64 restatement
(tests/grad_tc_oracle.py) against autograd, the class cfm_grad_tc_supported accepts, the case table
(tests/grad_tc_cases.py) against the sources and the paths it must reach, the compiled kernels, argument errors of the
C entry points (returned before any CUDA call) and the wrapper's refusals, which launch nothing."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

import grad_tc_cases as gc
import grad_tc_oracle as go
from oracle import vector_field as vf

import cfm_b200
from cfm_b200 import _ffi

ERR_ARG = -1  # CFM_ERR_ARG
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cfm_b200", "csrc")


def _action(dim, w, seed, act="selu"):
    torch.manual_seed(seed)
    m = vf.make_mlp(dim, out_dim=1, w=w, time_varying=True, dtype=torch.float64)
    if act == "silu":
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m


@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim,w", [(32, 32), (72, 136), (784, 256)])
def test_oracle_field_is_the_autograd_gradient_of_the_action(dim, w, act):
    m = _action(dim, w, dim + w, act)
    state = {k: v.detach() for k, v in m.state_dict().items()}
    x = torch.randn(7, dim, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    t = 0.41
    v = go.field(state, t, x, act)
    xg = x.clone().requires_grad_(True)
    s = m(torch.cat([xg, torch.full((7, 1), t, dtype=torch.float64)], 1)).sum()
    (ref,) = torch.autograd.grad(s, xg)
    assert torch.allclose(v, ref, rtol=1e-12, atol=1e-14)
    M, kink = go.bounds(state, t, x, act)
    assert bool((M >= v.abs() * (1 - 1e-12)).all())  # the scale bounds its entry
    assert kink.dtype == torch.bool and (act == "silu") <= (not bool(kink.any()))


def test_oracle_bounds_cover_an_fp32_evaluation():
    """An fp32 CPU evaluation of the same chain stays far inside the gate: the gate is not below fp32 rounding."""
    dim, w, act = 72, 136, "silu"
    m = _action(dim, w, 5, act)
    state = {k: v.detach() for k, v in m.state_dict().items()}
    x = torch.randn(33, dim, dtype=torch.float64, generator=torch.Generator().manual_seed(6))
    v64 = go.field(state, 0.3, x, act)
    v32 = go.field({k: v.float().double() for k, v in state.items()}, 0.3, x.float().double(), act)
    M, _ = go.bounds(state, 0.3, x, act)
    s32 = {k: v.float() for k, v in state.items()}
    W = [s32[f"net.{li}.weight"] for li in (0, 2, 4, 6)]
    b = [s32[f"net.{li}.bias"] for li in (0, 2, 4, 6)]
    xf, t = x.float(), torch.tensor(0.3)
    pre, a, D = None, xf, []
    for li in range(3):
        pre = a @ (W[li][:, :dim] if li == 0 else W[li]).T + b[li] + (t * W[0][:, dim] if li == 0 else 0)
        s = torch.sigmoid(pre)
        D.append(s * (1 + pre * (1 - s)))
        a = torch.nn.functional.silu(pre)
    g = D[0] * ((D[1] * ((D[2] * W[3][0]) @ W[2])) @ W[1])
    vf32 = (g @ W[0][:, :dim]).double()
    assert bool(((vf32 - v32).abs() <= 0.1 * go.GRAD_K * M).all())
    assert bool(((v32 - v64).abs() <= go.GRAD_K * M).all())


def test_supported_is_exactly_the_tensor_core_class(lib_built):
    lib = _ffi.load_library(lib_built)
    table = [((128, 32, 32), 1), ((127, 32, 32), 0), ((128, 24, 32), 0), ((128, 36, 32), 0), ((128, 32, 24), 0),
             ((128, 32, 36), 0), ((256, 784, 256), 1), ((10000, 784, 256), 1), ((129, 40, 136), 1),
             ((1024, 8, 64), 0), ((1024, 2, 256), 0), ((128, 32, 40), 1)]
    for (B, dim, w), want in table:
        assert lib.cfm_grad_tc_supported(B, dim, w) == want, (B, dim, w)
        assert lib.cfm_grad_tc_supported(B, dim, w) == lib.cfm_mlp_tc_supported(B, dim, w, dim)
        assert (lib.cfm_grad_tc_workspace_bytes(B, dim, w) > 0) == bool(want)
        assert not (want and lib.cfm_ode_small_grad_supported(B, dim, w))  # the two classes are disjoint
    assert lib.cfm_grad_tc_prepared_bytes(784, 256) > 0 == lib.cfm_grad_tc_prepared_bytes(2, 64)


def test_case_table_constants_match_the_sources():
    tc = open(os.path.join(CSRC, "gemm_tc.cuh")).read()
    h3 = open(os.path.join(CSRC, "gemm_h3.cuh")).read()
    assert re.search(r"constexpr int kTM = (\d+), kTN = (\d+);", tc).groups() == (str(gc.TM), str(gc.TN))
    assert re.search(r"constexpr int kHK = (\d+);", h3).group(1) == str(gc.HK)
    assert "col0 + 32 <= n1" in open(os.path.join(CSRC, "grad_tc.cu")).read() and gc.CHUNK == 32
    src = open(os.path.join(CSRC, "grad_tc.cu")).read()
    # layers 0, 1 (one loop through cnf_tc.cu's primal GEMM), layer 2, the reverse GEMMs by W2^T and W1^T, and by
    # W0x^T: the six GEMMs of gc.gemms
    launches = re.findall(r"launch_gemm_h3<(\w+), grad_gemm_kernel<", src)
    assert launches == ["GradSeedEpi", "GradReverseEpi", "GradReverseEpi", "GradOutEpi"]
    assert re.search(r"for \(int l = 0; l < 2; \+\+l\) \{[^}]*cnf_tc_primal_hidden\(", src)
    assert len(gc.gemms(64, 128)) == 6


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_case_table_reaches_every_path(sms):
    got = gc.reached(sms)
    missing = gc.REQUIRED - set(got)
    assert not missing, (sms, sorted(missing))


def test_new_kernels_are_built_for_sm90a_without_spills(lib_built):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-res-usage", lib_built], capture_output=True,
                         text=True).stdout
    blocks = re.findall(r"Fatbin elf code:\n=+\narch = (sm_\w+)(.*?)(?=Fatbin|\Z)", out, flags=re.S)
    found = {}
    for arch, body in blocks:
        for name, usage in re.findall(r"Function (\S+):\n\s*(REG:\d+ STACK:\d+[^\n]*)", body):
            if "grad_tc_cu" in name:
                found[name] = (arch, usage)
    for name, (arch, usage) in found.items():
        assert arch == "sm_90a", (name, arch)
        assert "STACK:0 " in usage and "LOCAL:0 " in usage, (name, usage)
    assert len(found) == 7, sorted(found)


def test_kernel_instantiations_are_pinned(lib_built):
    out = subprocess.run(["/usr/local/cuda/bin/cuobjdump", "-symbols", lib_built], capture_output=True, text=True,
                         check=True).stdout
    names = sorted(set(re.findall(r"grad_tc_cu_[0-9a-f]{8}(\w+)", out)))
    want = ["16grad_gemm_kernelINS0_10GradOutEpiEEEv14CUtensorMap_stS3_S3_S3_NS_7TcShapeET_",
            "16grad_gemm_kernelINS0_11GradSeedEpiEEEv14CUtensorMap_stS3_S3_S3_NS_7TcShapeET_",
            "16grad_gemm_kernelINS0_14GradReverseEpiEEEv14CUtensorMap_stS3_S3_S3_NS_7TcShapeET_",
            "17grad_split_kernelEPK6float4P6__halfS5_l",
            "22grad_euler_init_kernelEP17cfm_grad_tc_statePK6float4PS3_P6__halfS8_S6_PKfil",
            "22grad_euler_step_kernelEP17cfm_grad_tc_stateP6float4PKS3_P6__halfS8_l",
            "27grad_transpose_split_kernelENS0_13TransposeJobsEi"]
    assert names == want, names


def test_state_struct_matches_the_header():
    assert ctypes.sizeof(_ffi.GradTcState) == 32
    assert (_ffi.GradTcState.traj.offset, _ffi.GradTcState.t_span.offset) == (0, 8)
    assert (_ffi.GradTcState.n.offset, _ffi.GradTcState.n_steps.offset) == (16, 20)
    assert (_ffi.GradTcState.t.offset, _ffi.GradTcState.ticket.offset) == (24, 28)
    hdr = open(os.path.join(os.path.dirname(CSRC), "..", "include", "cfm_b200.h")).read()
    body = re.search(r"typedef struct cfm_grad_tc_state \{(.*?)\} cfm_grad_tc_state;", hdr, re.S).group(1)
    fields = re.findall(r"^\s*[\w\s\*]*?\**(\w+);", body, re.M)
    assert fields == [f for f, _ in _ffi.GradTcState._fields_]


def test_entry_points_check_arguments_before_any_cuda_call(lib_built):
    lib = _ffi.load_library(lib_built)
    buf = ctypes.create_string_buffer(1 << 12)
    p = (ctypes.addressof(buf) + 15) // 16 * 16
    q = p + 4  # 4-byte aligned only
    big = 1 << 40

    def field(**kw):
        a = dict(blob=p, gblob=p, x=p, x_hi=None, x_lo=None, batch=256, dim=64, w=128, act=0, t=p, v=p, ws=p,
                 wsb=big, stream=None)
        a.update(kw)
        return lib.cfm_grad_tc_field_f32(*a.values())

    cases = [(dict(blob=None), "null pointer"), (dict(gblob=None), "null pointer"), (dict(t=None), "null pointer"),
             (dict(v=None), "null pointer"), (dict(x_hi=p, x_lo=p), "either x or the pair"),
             (dict(x=None, x_hi=p), "either x or the pair"), (dict(act=7), "unknown activation"),
             (dict(batch=127), "unsupported shape"), (dict(dim=60), "unsupported shape"),
             (dict(w=36), "unsupported shape"), (dict(dim=8), "unsupported shape"), (dict(wsb=16), "workspace too small"),
             (dict(x=q), "16-byte aligned"), (dict(ws=q), "16-byte aligned"), (dict(gblob=q), "16-byte aligned"),
             (dict(v=q + 1), "4-byte aligned")]
    for kw, text in cases:
        assert field(**kw) == ERR_ARG, kw
        assert text.encode() in lib.cfm_last_error(), (kw, lib.cfm_last_error())
    assert lib.cfm_grad_tc_prepare(None, 64, 128, p, big, None) == ERR_ARG
    assert lib.cfm_grad_tc_prepare(p, 64, 36, p, big, None) == ERR_ARG
    assert lib.cfm_grad_tc_prepare(p, 64, 128, p, 16, None) == ERR_ARG and b"too small" in lib.cfm_last_error()
    assert lib.cfm_grad_tc_prepare(p, 64, 128, q, big, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_init(None, p, p, p, p, p, p, 3, 256, 64, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_init(p, p, p, p, p, p, p, 1, 256, 64, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_init(p, q, p, p, p, p, p, 3, 256, 64, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_init(p, p, p, p, p, q, p, 3, 256, 64, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_step(p, p, p, p, p, 256, 20, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_step(p, p, q, p, p, 256, 64, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_step(p, p, None, p, p, 256, 64, None) == ERR_ARG
    assert lib.cfm_grad_tc_euler_step(p + 4, p, p, p, p, 256, 64, None) == ERR_ARG


def _node(action, **kw):
    return cfm_b200.NeuralODE(cfm_b200.torch_wrapper(cfm_b200.GradModel(action)), **kw)


@pytest.mark.parametrize("solver", ["euler", "dopri5"])
@pytest.mark.parametrize("B,dim,w", [(127, 64, 128), (1024, 16, 64), (1024, 64, 36), (1024, 60, 128),
                                     (1024, 2, 128)])
def test_shapes_outside_both_classes_are_refused_with_no_launch(B, dim, w, solver):
    """The refusal comes from the shapes alone, on the host: the state here is on the CPU, and the message names both
    classes."""
    L = _ffi.lib()
    action = cfm_b200.MLP(dim=dim, out_dim=1, w=w, time_varying=True)
    node = _node(action, solver=solver)
    before = L.cfm_launch_count()
    with pytest.raises(NotImplementedError, match=r"no gradient-field kernel.*w in \{32, 64\}, dim <= 8.*"
                                                  r"tensor-core class takes B >= 128, dim >= 32"):
        node._grad_trajectory_on(action, torch.zeros(B, dim), torch.linspace(0, 1, 3), torch.device("cpu"))
    assert L.cfm_launch_count() == before


def test_other_refusals_stay():
    wide = cfm_b200.MLP(dim=64, out_dim=2, w=128, time_varying=True)
    with pytest.raises(NotImplementedError, match="out_dim=2"):
        _node(wide, solver="euler").trajectory(torch.zeros(256, 64), torch.linspace(0, 1, 3))
    with pytest.raises(NotImplementedError, match="time_varying=False"):
        _node(cfm_b200.MLP(dim=64, out_dim=1, w=128), solver="euler").trajectory(torch.zeros(256, 64),
                                                                                  torch.linspace(0, 1, 3))
    with pytest.raises(TypeError, match="GradModel"):
        _node(torch.nn.Linear(65, 1), solver="euler").trajectory(torch.zeros(256, 64), torch.linspace(0, 1, 3))
    action = cfm_b200.MLP(dim=64, out_dim=1, w=128, time_varying=True)
    node = _node(action, solver="dopri5")
    node.lockstep = True
    with pytest.raises(NotImplementedError, match="lock-step"):
        node._grad_trajectory_on(action, torch.zeros(256, 64), torch.linspace(0, 1, 3), torch.device("cpu"))
    with pytest.raises(_ffi.CfmLibraryError, match="needs CUDA inputs"):  # in the class: no CPU fallback
        _node(action, solver="euler").trajectory(torch.zeros(256, 64), torch.linspace(0, 1, 3))


# ---- the scales of the prepared blobs ---------------------------------------------------------------------------------
def _scaled_state(dim, w, factors, act="selu", seed=gc.LAYER_SCALE_SEED):
    return {k: v.detach() for k, v in gc.scaled_action(dim, w, seed, factors, act).state_dict().items()}


def test_scale_rules_match_the_sources():
    """grad_tc_oracle.layer_scales restates h3_pow2_scale and the chain rule of grad_tc.cu's grad_chain_scale."""
    h3 = open(os.path.join(CSRC, "gemm_h3.cuh")).read()
    body = re.search(r"float h3_pow2_scale\(float am\) \{(.*?)\n\}", h3, re.S).group(1)
    assert "if (am > 0.f && am < 3.0e38f)" in body and "e = max(-100, min(100, 13 - e));" in body
    assert "int e = ilogbf(am);" in body and "sc = scalbnf(1.f, e);" in body
    src = open(os.path.join(CSRC, "grad_tc.cu")).read()
    A = float(re.search(r"constexpr float kActPrimeMax = ([\d.]+)f;", src).group(1))
    assert go.ACT_PRIME_MAX == go.np.float32(A)
    assert A >= go.SELU_L * go.SELU_A and A >= 1.0998  # SELU's lambda alpha and SiLU's max act'
    body = re.search(r"void grad_chain_scale\((.*?)\n\}", src, re.S).group(1)
    for line in ["s1 += fabsf(__ldg(jobs.j[1].src + (int64_t)j * jobs.j[1].lds + i));",
                 "s2 += fabsf(__ldg(jobs.j[2].src + (int64_t)j * jobs.j[2].lds + i));",
                 "float k = 0x1p-7f / __ldg(jobs.inv_ws3);",
                 "const float b2 = kActPrimeMax * m3;", "const float b1 = b2 * (kActPrimeMax * c2);",
                 "const float b0 = b1 * (kActPrimeMax * c1);", "const float peak = fmaxf(b2, fmaxf(b1, b0));",
                 "if (peak > 0.f && peak <= 3.0e38f) k = fminf(k, __int_as_float(__float_as_int(65504.f / peak) & "
                 "0x7f800000));",
                 "jobs.sc[0] = k;", "jobs.sc[1] = __ldg(jobs.j[0].inv_ws) / k;"]:
        assert line in body, line
    # the transpose scales each layer by its own s_l, and the epilogues undo layer 2's, then layer 1's
    assert "const float sc = 1.f / __ldg(J.inv_ws);" in src
    assert "if ((blockIdx.x | blockIdx.y) == 0) grad_chain_scale(jobs, w);" in src
    assert "J.inv_ws3 = W.inv_ws[3];" in src
    assert "GradReverseEpi r2{W.inv_ws[2]," in src and "GradReverseEpi r1{W.inv_ws[1]," in src
    assert "GradSeedEpi se{F(boff[2]), W.inv_ws[2]," in src and "GradOutEpi r0{sc + 1," in src


def test_pow2_scale_restatement():
    assert go.pow2_scale(0.0) == 1 and go.pow2_scale(float("inf")) == 1 and go.pow2_scale(float("nan")) == 1
    assert go.pow2_scale(1.0) == 2.0 ** 13 and go.pow2_scale(1.5) == 2.0 ** 13 and go.pow2_scale(2.0) == 2.0 ** 12
    assert go.pow2_scale(2.0 ** -110) == 2.0 ** 100 and go.pow2_scale(2.0 ** 120) == 2.0 ** -100
    assert go.pow2_scale(2.0 ** -140) == 2.0 ** 100  # a float32 subnormal


@pytest.mark.parametrize("factors", gc.LAYER_SCALE_SETS)
@pytest.mark.parametrize("B,dim,w", gc.LAYER_SCALE_SHAPES)
def test_layer_scale_sets_give_distinct_scales(B, dim, w, factors):
    s, (k, k0) = go.layer_scales(_scaled_state(dim, w, factors), dim)
    vals = [float(v) for v in s] + [float(k)]
    assert len(set(vals)) == 5, vals
    assert float(k0) == 1 / (float(s[0]) * float(k))


def test_layer_scale_sets_rank_each_hidden_layer_first_and_last():
    hidden = [f[:3] for f in gc.LAYER_SCALE_SETS]
    assert {h.index(max(h)) for h in hidden} == {0, 1, 2} and {h.index(min(h)) for h in hidden} == {0, 1, 2}
    assert all(f[3] not in f[:3] for f in gc.LAYER_SCALE_SETS)


@pytest.mark.parametrize("act,factors,frac", gc.RANGE_CASES)
def test_range_cases_reach_their_fraction(act, factors, frac):
    """Under the W3-only rule 2^k = s_3 2^-7 the chain peaks at the claimed fraction of 65504; under the chain bound no
    split passes 65504; the forward activations stay far below it."""
    B, dim, w = gc.RANGE_SHAPE
    state = _scaled_state(dim, w, factors, act, seed=7)
    x = gc.range_input(B, dim).double()
    _, (k_w3, _) = go.layer_scales(state, dim, chain_bound=False)
    got = max(go.chain_peaks(state, 0.3, x, act, sk=float(k_w3))) / go.FP16_MAX
    assert abs(got - frac) <= 0.01 * frac, (got, frac)
    assert max(go.chain_peaks(state, 0.3, x, act)) <= go.FP16_MAX
    assert go.activation_peak(state, 0.3, x, act) <= 0.1 * go.FP16_MAX


def test_chain_bound_keeps_the_default_action_and_lowers_the_scaled_ones():
    """At the default-initialised MNIST action the bound leaves 2^k = s_3 2^-7; W0..W2 x 3 and x 11 lower it by 2^3 and
    2^7."""
    dim, w = 784, 256
    for f, drop in ((1.0, 0), (3.0, 3), (11.0, 7)):
        state = _scaled_state(dim, w, (f, f, f, 1.0), seed=7)
        k_w3 = go.layer_scales(state, dim, chain_bound=False)[1][0]
        k = go.layer_scales(state, dim)[1][0]
        assert k_w3 / k == 2.0 ** drop, (f, k_w3, k)


def test_chain_factor_is_linear_in_w3():
    dim, w = 72, 136
    state = _scaled_state(dim, w, (20.0, 20.0, 20.0, 1.0))
    k = float(go.layer_scales(state, dim)[1][0])
    for p in gc.W3_POWERS:
        st = dict(state)
        st["net.6.weight"] = state["net.6.weight"] * 2.0 ** p
        assert float(go.layer_scales(st, dim)[1][0]) == k * 2.0 ** -p, p


@pytest.mark.parametrize("dim,w,factors", [(784, 256, (1.0,) * 4), (32, 40, (1.0,) * 4), (264, 264, (1.0,) * 4),
                                           (72, 136, gc.LAYER_SCALE_SETS[1])])
def test_grad_blob_matches_a_float64_transpose(dim, w, factors):
    np = go.np
    state = _scaled_state(dim, w, factors)
    blob, regions = go.grad_blob(state, dim, w)
    s, sc = go.layer_scales(state, dim)
    r = {name: (off, n) for name, off, n in regions}
    assert r["sc"] == (0, 8) and all(off % 1024 == 0 for off, _ in r.values())
    assert blob[:8].view(np.float32).tolist() == [float(sc[0]), float(sc[1])]
    W = go._weights32(state, dim)
    for li in range(3):
        ref = W[li].astype(np.float64).T * float(s[li])
        rows = dim if li == 0 else w
        got = []
        for part in ("wth", "wtl"):
            off, n = r[f"{part}{li}"]
            assert n == rows * w * 2
            got.append(blob[off:off + n].view(np.float16).astype(np.float64).reshape(rows, w))
        val = got[0] + got[1] * 2.0 ** -11
        assert np.all(np.abs(val - ref) <= 2.0 ** -22 * np.abs(ref) + 2.0 ** -35), li
