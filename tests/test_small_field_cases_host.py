"""The edge cases of the one-launch SDE and gradient-field kernels without a device (tests/small_field_cases.py): the
constants it restates are the text of csrc/ode_small.cu; the table reaches every listed path on an H100's 132 SMs and
on parts with fewer; the SDE boundary cases fall on each side of the small / tensor-core split; and the per-entry
scales of tests/small_field_oracle.py bound their entries and an fp32 evaluation on the CPU by far."""
import os
import re

import pytest
import torch

import small_field_cases as sc
import small_field_oracle as so

import cfm_b200

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "cfm_b200", "csrc")


def _src(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_restated_constants_are_the_sources():
    ode = _src("ode_small.cu")
    assert re.search(r"constexpr int RB = (\d+);", _src("mlp_small.cuh")).group(1) == str(sc.RB)
    assert re.search(r"constexpr int kSlots = (\d+);", ode).group(1) == str(sc.K_SLOTS)
    assert re.search(r"constexpr int kSdeSlots = (\d+);", ode).group(1) == str(sc.K_SDE_SLOTS)
    assert re.search(r"constexpr int kGradMaxWarps = (\d+);", ode).group(1) == str(sc.GRAD_MAX_WARPS)
    assert re.search(r"constexpr int kSdeMaxWarps = (\d+);", ode).group(1) == str(sc.SDE_MAX_WARPS)
    assert ode.count("if (gpw > (1 << 19)) return 0;") == 2 and sc.GPW_CAP == 1 << 19
    assert ode.count("> 200 * 1024") == 1 and ode.count("<= 200 * 1024") == 1 and sc.SMEM_BUDGET == 200 * 1024
    assert ode.count("if (B <= 0 || dim <= 0 || dim > 1024) return 0;") == 2 and sc.MAX_DIM == 1024
    # the layouts, in order
    assert re.search(r"s\.wt0 = take\(\(size_t\)dim \* w\);\s+s\.wtime = take\(w\);\s+s\.b0 = take\(w\);\s+"
                     r"s\.wt1 = take\(\(size_t\)w \* w\);\s+s\.b1 = take\(w\);\s+s\.wt2 = take\(\(size_t\)w \* w\);\s+"
                     r"s\.b2 = take\(w\);\s+s\.wt3 = take\(\(size_t\)w \* dim\);\s+s\.b3 = take\(dim\);\s+"
                     r"s\.hbuf = take\(\(size_t\)nwarps \* RB \* 2 \* w \* \(cnf \? 1 \+ dim : 1\)\);\s+"
                     r"s\.xin = take\(\(size_t\)nwarps \* RB \* s\.dimp\);\s+"
                     r"s\.state = take\(\(size_t\)nwarps \* rpw \* kSlots \* s\.dimp\);\s+"
                     r"s\.red = take\(2 \* 3 \* 32 \+ 8\);", ode)
    assert "(f == kGradField ? (size_t)2 * w * w * sizeof(float) : 0)" in ode
    assert re.search(r"s\.set2 = s\.net\.hbuf;\s+size_t o = 2 \* s\.set2;\s+s\.hbuf = o;\s+"
                     r"o \+= \(size_t\)nwarps \* RB \* 2 \* w;\s+s\.state = o;\s+"
                     r"o \+= \(size_t\)nwarps \* rpw \* kSdeSlots \* s\.net\.dimp;", ode)
    # the planners: 4 warps first, doubling while a warp holds 2+ groups; the gradient field's fallback halves
    assert ode.count("int nwarps = 4;") == 2
    assert "if (gpw == 1 || nwarps == max_warps) break;" in ode and "if (gpw == 1 || nwarps == kSdeMaxWarps) break;" in ode
    assert "if (f == kPlainField || nwarps == 1) return 0;\n    nwarps /= 2;" in ode
    assert "if (f != kPlainField && dim > 8) return 0;" in ode
    # the rows of a warp
    assert ode.count("return (gwarp + (int64_t)(j / RB) * wstride) * RB + (j % RB);") == 2
    # sdeint's class choice
    sde = open(os.path.join(os.path.dirname(CSRC), "sde.py")).read()
    assert "small = bool(L.cfm_sde_small_supported(B, D, drift.w))" in sde
    assert "batch >= 128 && dim >= 32 && dim % 8 == 0" in _src("sde_common.cuh")


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_the_table_reaches_every_path(sms):
    missing = sorted(sc.REQUIRED - set(sc.reached(sms)))
    assert not missing, (sms, missing)


def test_planner_edges_on_132_sms():
    """The boundaries named in DESIGN.md sections 3.10, 3.11 and 7 (restated, not measured)."""
    sms = sc.H100_SMS
    assert sc.sde_bmax(64, 64, sms) == 4224 and sc.tc_supported(4225, 64, 64)
    assert sc.sde_bmax(100, 64, sms) == 2112 and not sc.tc_supported(2113, 100, 64)
    assert (sc.sde_dmax(32, sms), sc.sde_dmax(64, sms)) == (285, 114)
    assert sc.plan_sde(1, 286, 32, sms) is None and sc.plan_sde(1, 115, 64, sms) is None
    for w in (32, 64):
        for dim in range(1, 9):
            B = sc.grad_bmax(dim, w, sms)
            assert sc.plan_grad(B, dim, w, sms)[1] == 1 and sc.plan_grad(B + 1, dim, w, sms) is None
    assert sc.grad_bmax(1, 32, sms) == 170544 and sc.plan_grad(170544, 1, 32, sms)[2] == 1292
    assert sc.grad_bmax(8, 64, sms) == 60456 and sc.plan_grad(60456, 8, 64, sms)[2] == 458
    assert [sc.plan_grad(sc.grad_fallback_batch(5, 64, n, sms), 5, 64, sms)[1] for n in (4, 2, 1)] == [4, 2, 1]
    assert sc.grad_fallback_batch(5, 64, 4, sms) == 57025
    plan = sc.plan_sde(80 * sms + 3, 3, 64, sms)
    assert plan[:3] == (132, 16, 6)
    assert sc.edge_rows(80 * sms + 3, plan) == {
        "first row of a group": 0, "second row of a group": 1, "CTA's last row in its first pass": 4223,
        "first row of a second pass": 4224, "batch's last row": 10562, "lone last row of an odd batch": 10562}


@pytest.mark.parametrize("sms", [132, 114, 78])
def test_sde_boundary_cases_fall_on_each_side_of_the_split(sms):
    """Each SDE boundary case: the small kernel plans its batch, not the next; the next goes to the tensor-core class
    exactly where that class's shape rule takes it; the dmax cases refuse the next dim in both classes."""
    sides = set()
    for w, d in sc.SDE_BMAX:
        dim = sc.resolve_dim(w, d, sms)
        B = sc.sde_bmax(dim, w, sms)
        assert sc.plan_sde(B, dim, w, sms) is not None and sc.plan_sde(B + 1, dim, w, sms) is None
        sides.add(sc.tc_supported(B + 1, dim, w))
        if d == "dmax":
            assert sc.plan_sde(1, dim + 1, w, sms) is None and not sc.tc_supported(1, dim + 1, w)
    assert sides == {True, False}


# ---- the per-entry scales -------------------------------------------------------------------------------------------
FP32_BOUND = 0.02  # an fp32 evaluation on the CPU errs by far less than the gate


def _model(dim, out_dim, w, act, seed):
    torch.manual_seed(seed)
    m = cfm_b200.MLP(dim=dim, out_dim=out_dim, w=w, time_varying=True)
    if act == "silu":
        for k in (1, 3, 5):
            m.net[k] = torch.nn.SiLU()
    return m


@pytest.mark.parametrize("scale", [1.0, 30.0])
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim,w", [(1, 32), (8, 64), (9, 32), (100, 64), (285, 32)])
def test_mlp_scales_bound_the_output_and_an_fp32_run(dim, w, act, scale):
    m = _model(dim, None, w, act, seed=dim + w)
    x = scale * torch.randn(300, dim, generator=torch.Generator().manual_seed(dim))
    f, F, gate = so.mlp_bounds(m.state_dict(), 0.37, x, act)
    with torch.no_grad():
        f32 = m.net(torch.cat([x, torch.full((300, 1), 0.37)], 1)).double()
        f64 = m.double().net(torch.cat([x.double(), torch.full((300, 1), 0.37, dtype=torch.float64)], 1))
    assert torch.allclose(f, f64, rtol=0, atol=1e-12 * float(F.max()))
    assert (f.abs() <= F).all() and (gate > 0).all() and (gate < 1e-3 * F).all()
    worst = float(((f32 - f).abs() / gate).max())
    assert 0 < worst < FP32_BOUND, worst


@pytest.mark.parametrize("scale", [1.0, 30.0])
@pytest.mark.parametrize("act", ["selu", "silu"])
@pytest.mark.parametrize("dim,w", [(1, 32), (5, 64), (8, 32), (8, 64)])
def test_grad_scales_bound_the_field_and_an_fp32_run(dim, w, act, scale):
    m = _model(dim, 1, w, act, seed=10 + dim + w)
    x = scale * torch.randn(300, dim, generator=torch.Generator().manual_seed(dim))
    f, G, gate, kink = so.grad_bounds(m.state_dict(), 0.37, x, act)

    def grad(mod, xx):
        y = xx.clone().requires_grad_(True)
        s = mod(torch.cat([y, torch.full((300, 1), 0.37, dtype=xx.dtype)], 1))
        return torch.autograd.grad(s.sum(), y)[0].double()
    g32, g64 = grad(m, x), grad(m.double(), x.double())
    assert torch.allclose(f, g64, rtol=0, atol=1e-12 * float(G.max()))
    assert (f.abs() <= G).all() and (gate > 0).all()
    assert int(kink.sum()) <= 30 and (act == "selu" or not kink.any())
    worst = float(((g32 - f).abs() / gate)[~kink].max())
    assert 0 < worst < FP32_BOUND, worst


def test_grad_scale_is_the_field_when_no_term_cancels():
    """Positive weights and inputs, SELU with every pre-activation positive: act' is the constant lambda, no term
    cancels, and the scale with its widening taken out is the field itself."""
    dim, w = 3, 32
    m = _model(dim, 1, w, "selu", seed=3)
    with torch.no_grad():
        for p in m.parameters():
            p.abs_()
    x = torch.rand(20, dim)
    f, G, gate, kink = so.grad_bounds(m.state_dict(), 0.5, x, "selu")
    assert not kink.any() and (f > 0).all()
    assert torch.allclose(G, f, rtol=1e-5, atol=0) and (G >= f).all()
