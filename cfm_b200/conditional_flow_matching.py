"""Conditional flow matchers: drop-in for ``torchcfm.conditional_flow_matching``.

API surface, class names, method names, attribute names (``sigma``, ``ot_sampler``,
``ot_method``) and error behaviour follow the reference file
(torchcfm/conditional_flow_matching.py:17-618).  The OT variants call the CUDA coupling
(``cfm_b200.optimal_transport.OTPlanSampler``); the per-element ``xt / ut`` arithmetic is a few
elementwise torch ops on the inputs' device, evaluated in the same operation order as the
reference so results are bit-identical given the same pairs, ``t`` and ``eps``.

For contiguous fp32 CUDA batches that do not require grad, the stock classes take a fused path
(SURVEY section 8 f-1, csrc/flow.cu): the pair gather ``x0[i], x1[j]``, ``xt`` and ``ut`` are produced
by ONE kernel pass whose element arithmetic is unfused round-to-nearest fp32 in the reference's
association order, so the tensors equal the unfused ones bit for bit (tests/test_gpu_parity.py,
tests/test_gpu_flow_gather.py).  Subclasses that override ``compute_*``, inputs that need autograd
and strided inputs (whose ``randn_like`` noise is laid out differently) use the plain torch expressions.
"""
import math
import warnings
from typing import Union

import torch

from . import _ffi
from .optimal_transport import OTPlanSampler


def pad_t_like_x(t, x):
    """Reshape the time vector ``t`` (bs,) to (bs, 1, ..., 1) so it broadcasts against ``x``;
    scalars pass through (reference :17-38)."""
    if isinstance(t, (float, int)):
        return t
    return t.reshape(-1, *([1] * (x.dim() - 1)))


class ConditionalFlowMatcher:
    """Independent CFM (reference :41-217): path N(t*x1 + (1-t)*x0, sigma), field x1 - x0."""

    def __init__(self, sigma: Union[float, int] = 0.0):
        self.sigma = sigma

    def compute_mu_t(self, x0, x1, t):
        """mean of the path: t*x1 + (1-t)*x0 (reference :62-83)."""
        t = pad_t_like_x(t, x0)
        return t * x1 + (1 - t) * x0

    def compute_sigma_t(self, t):
        """std of the path: the constant sigma (reference :85-102)."""
        del t
        return self.sigma

    def sample_xt(self, x0, x1, t, epsilon):
        """xt = mu_t + sigma_t * eps (reference :104-129)."""
        mu_t = self.compute_mu_t(x0, x1, t)
        sigma_t = pad_t_like_x(self.compute_sigma_t(t), x0)
        return mu_t + sigma_t * epsilon

    def compute_conditional_flow(self, x0, x1, t, xt):
        """ut = x1 - x0 (reference :131-154)."""
        del t, xt
        return x1 - x0

    def sample_noise_like(self, x):
        return torch.randn_like(x)

    def sample_location_and_conditional_flow(self, x0, x1, t=None, return_noise=False):
        """(t, xt, ut[, eps]) for a batch of pairs (reference :159-199).  ``t`` defaults to
        ``torch.rand(bs)`` drawn on the CPU generator and cast like x0, as in the reference."""
        return self._sample_flow(x0, x1, None, None, t, return_noise)

    # -- fused device path -----------------------------------------------------------------
    _FUSED_KIND = _ffi.FLOW_ICFM  # which closed form csrc/flow.cu evaluates for this class

    def _fused_ok(self, x0, x1):
        # Contiguous inputs only: the kernel's eps is drawn contiguous, while the reference's randn_like(x0) keeps
        # a transposed or channels_last layout and fills it in memory order, i.e. puts other normals on each element.
        stock = _STOCK.get(type(self).__name__)
        return (stock is type(self) and x0.is_cuda and x1.is_cuda and x0.dtype == torch.float32
                and x1.dtype == torch.float32 and x0.shape == x1.shape and x0.dim() >= 2
                and x0.is_contiguous() and x1.is_contiguous()
                and not x0.requires_grad and not x1.requires_grad
                and isinstance(self.sigma, (int, float)))

    def _row_coefficients(self, t):
        """Per-row scalars of the closed form, computed with the reference's own expressions:
        (row_a, row_b, row_sigma | None, row_c | None, sigma scalar, constant)."""
        return t, 1 - t, None, None, float(self.sigma), 0.0

    def _sample_flow(self, x0, x1, i, j, t, return_noise):
        """Common tail of every matcher: draw t and eps in the reference's order, then xt / ut either
        by the fused kernel (pairs given by device index tensors i, j or identity) or by torch ops."""
        n = x0.shape[0] if i is None else i.shape[0]
        # a caller-supplied t of another dtype (float64 ...) promotes xt / ut in the reference: torch-op path
        t_ok = t is None or (torch.is_tensor(t) and t.dtype == x0.dtype)
        if not (t_ok and self._fused_ok(x0, x1)):
            if i is not None:
                x0, x1 = x0[i], x1[j]
            if t is None:
                t = torch.rand(x0.shape[0]).type_as(x0)
            assert len(t) == x0.shape[0], "t has to have batch size dimension"
            eps = self.sample_noise_like(x0)
            xt = self.sample_xt(x0, x1, t, eps)
            ut = self.compute_conditional_flow(x0, x1, t, xt)
            return (t, xt, ut, eps) if return_noise else (t, xt, ut)
        if t is None:
            t = torch.rand(n).type_as(x0)
        assert len(t) == n, "t has to have batch size dimension"
        shape = (n,) + tuple(x0.shape[1:])
        eps = torch.randn(shape, dtype=x0.dtype, device=x0.device)  # == randn_like(x0[i]): x0 is contiguous
        ra, rb, rs, rc, sig, kon = self._row_coefficients(t.to(x0.device))
        vec = lambda v: None if v is None else v.to(torch.float32).contiguous()  # noqa: E731
        ra, rb, rs, rc = vec(ra), vec(rb), vec(rs), vec(rc)
        xt = torch.empty(shape, dtype=torch.float32, device=x0.device)
        ut = torch.empty(shape, dtype=torch.float32, device=x0.device)
        row = 1
        for dsz in shape[1:]:
            row *= dsz
        with torch.cuda.device(x0.device):
            _ffi.check(_ffi.lib().cfm_flow_pairs_f32(
                self._FUSED_KIND, _ffi.ptr(x0), _ffi.ptr(x1), _ffi.ptr(i), _ffi.ptr(j), _ffi.ptr(eps),
                _ffi.ptr(ra), _ffi.ptr(rb), _ffi.ptr(rs), _ffi.ptr(rc), sig, kon, _ffi.ptr(xt), _ffi.ptr(ut),
                n, row, _ffi.stream_ptr(x0.device)), "cfm_flow_pairs_f32")
        return (t, xt, ut, eps) if return_noise else (t, xt, ut)

    def compute_lambda(self, t):
        """score weighting 2*sigma_t / (sigma^2 + 1e-8) (reference :201-217)."""
        sigma_t = self.compute_sigma_t(t)
        return 2 * sigma_t / (self.sigma**2 + 1e-8)


class _CoupledMixin:
    """OT-coupled variants re-pair the minibatch through ``self.ot_sampler`` first."""

    def sample_location_and_conditional_flow(self, x0, x1, t=None, return_noise=False):
        if self._fused_ok(x0, x1) and isinstance(self.ot_sampler, OTPlanSampler):
            i, j = self.ot_sampler.sample_pairs(x0, x1)  # device indices; x0[i], x1[j] never stored
            return self._sample_flow(x0, x1, i, j, t, return_noise)
        x0, x1 = self.ot_sampler.sample_plan(x0, x1)
        return super().sample_location_and_conditional_flow(x0, x1, t, return_noise)

    def guided_sample_location_and_conditional_flow(self, x0, x1, y0=None, y1=None, t=None,
                                                    return_noise=False):
        if self._fused_ok(x0, x1) and isinstance(self.ot_sampler, OTPlanSampler):
            i, j = self.ot_sampler.sample_pairs(x0, x1)
            g = self.ot_sampler._gather
            y0 = g(y0, i) if y0 is not None else None
            y1 = g(y1, j) if y1 is not None else None
            out = self._sample_flow(x0, x1, i, j, t, return_noise)
        else:
            x0, x1, y0, y1 = self.ot_sampler.sample_plan_with_labels(x0, x1, y0, y1)
            out = super().sample_location_and_conditional_flow(x0, x1, t, return_noise)
        if return_noise:
            t, xt, ut, eps = out
            return t, xt, ut, y0, y1, eps
        t, xt, ut = out
        return t, xt, ut, y0, y1


class ExactOptimalTransportConditionalFlowMatcher(_CoupledMixin, ConditionalFlowMatcher):
    """OT-CFM (reference :220-316): pairs drawn from the exact minibatch OT plan."""

    def __init__(self, sigma: Union[float, int] = 0.0):
        super().__init__(sigma)
        self.ot_sampler = OTPlanSampler(method="exact")


class TargetConditionalFlowMatcher(ConditionalFlowMatcher):
    """Lipman et al. target CFM (reference :319-394)."""

    def compute_mu_t(self, x0, x1, t):
        del x0
        return pad_t_like_x(t, x1) * x1

    def compute_sigma_t(self, t):
        return 1 - (1 - self.sigma) * t

    def compute_conditional_flow(self, x0, x1, t, xt):
        del x0
        t = pad_t_like_x(t, x1)
        return (x1 - (1 - self.sigma) * xt) / (1 - (1 - self.sigma) * t)

    _FUSED_KIND = _ffi.FLOW_TARGET

    def _row_coefficients(self, t):
        st = 1 - (1 - self.sigma) * t
        return t, None, st, st, 0.0, float(1 - self.sigma)


class SchrodingerBridgeConditionalFlowMatcher(_CoupledMixin, ConditionalFlowMatcher):
    """SB-CFM (reference :397-556): entropic coupling with reg = 2 sigma^2, Brownian-bridge
    std sigma*sqrt(t(1-t)) and the matching drift correction."""

    def __init__(self, sigma: Union[float, int] = 1.0, ot_method="exact"):
        if sigma <= 0:
            raise ValueError(f"Sigma must be strictly positive, got {sigma}.")
        elif sigma < 1e-3:
            warnings.warn("Small sigma values may lead to numerical instability.")
        super().__init__(sigma)
        self.ot_method = ot_method
        self.ot_sampler = OTPlanSampler(method=ot_method, reg=2 * self.sigma**2)

    def compute_sigma_t(self, t):
        return self.sigma * torch.sqrt(t * (1 - t))

    def compute_conditional_flow(self, x0, x1, t, xt):
        t = pad_t_like_x(t, x0)
        mu_t = self.compute_mu_t(x0, x1, t)
        sigma_t_prime_over_sigma_t = (1 - 2 * t) / (2 * t * (1 - t) + 1e-8)
        return sigma_t_prime_over_sigma_t * (xt - mu_t) + x1 - x0

    _FUSED_KIND = _ffi.FLOW_SB

    def _row_coefficients(self, t):
        return t, 1 - t, self.sigma * torch.sqrt(t * (1 - t)), (1 - 2 * t) / (2 * t * (1 - t) + 1e-8), 0.0, 0.0


class VariancePreservingConditionalFlowMatcher(ConditionalFlowMatcher):
    """Albergo et al. trigonometric interpolant (reference :559-618)."""

    def compute_mu_t(self, x0, x1, t):
        t = pad_t_like_x(t, x0)
        return torch.cos(math.pi / 2 * t) * x0 + torch.sin(math.pi / 2 * t) * x1

    def compute_conditional_flow(self, x0, x1, t, xt):
        del xt
        t = pad_t_like_x(t, x0)
        return math.pi / 2 * (torch.cos(math.pi / 2 * t) * x1 - torch.sin(math.pi / 2 * t) * x0)

    _FUSED_KIND = _ffi.FLOW_VP

    def _row_coefficients(self, t):
        return torch.cos(math.pi / 2 * t), torch.sin(math.pi / 2 * t), None, None, float(self.sigma), math.pi / 2


# the stock classes: only exactly these (no user subclass overriding compute_*) take the fused path
_STOCK = {c.__name__: c for c in (ConditionalFlowMatcher, ExactOptimalTransportConditionalFlowMatcher,
                                  TargetConditionalFlowMatcher, SchrodingerBridgeConditionalFlowMatcher,
                                  VariancePreservingConditionalFlowMatcher)}
