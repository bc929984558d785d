"""Vector-field MLP: drop-in for ``torchcfm.models.MLP`` and ``torchcfm.utils.torch_wrapper``.

``MLP`` keeps the reference architecture and parameter names (torchcfm/models/models.py:4-21:
``net.0 / net.2 / net.4 / net.6`` Linear layers with SELU between them), so reference
checkpoints load unchanged.  Under ``torch.no_grad()`` on a CUDA device -- the regime of the ODE
sampling loop, where torchdyn calls ``forward(t, x)`` six times per step
(examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb:332-338) -- the forward runs
in libcfm_b200's kernels (cfm_mlp_forward_f32).  With autograd enabled the module is an ordinary
``torch.nn.Sequential`` on any device; the tutorials' training step (forward, regression loss and backward of a small
``MLP(time_varying=True)``) runs in one kernel through ``cfm_b200.flow_matching_loss`` instead (cfm_b200/train.py).
"""
import torch

from . import _ffi


class MLP(torch.nn.Module):
    def __init__(self, dim, out_dim=None, w=64, time_varying=False):
        super().__init__()
        self.time_varying = time_varying
        if out_dim is None:
            out_dim = dim
        self.dim, self.out_dim, self.w = dim, out_dim, w
        self.net = torch.nn.Sequential(
            torch.nn.Linear(dim + (1 if time_varying else 0), w),
            torch.nn.SELU(),
            torch.nn.Linear(w, w),
            torch.nn.SELU(),
            torch.nn.Linear(w, w),
            torch.nn.SELU(),
            torch.nn.Linear(w, out_dim),
        )
        self.act = _ffi.ACT_SELU
        self.mlp_algo = 0  # 0 auto, 1 SIMT fp32, 2 tensor cores (fp16x3 scheme: fused kernel for w = 256, per-layer otherwise)
        self._blobs = {}   # (split_t, device) -> (version key, prepared blob tensor)
        self._reversed = None  # (version key, time-reversed MLP); a tuple, so it is not registered as a submodule

    # -- prepared weights (rebuilt when any parameter changes in place or is replaced) ------
    def _linears(self):
        return [self.net[0], self.net[2], self.net[4], self.net[6]]

    def _weights_key(self):
        return tuple((p.data_ptr(), p._version) for lin in self._linears()
                     for p in (lin.weight, lin.bias))

    def _device_params(self, device):
        """The eight parameters (weight and bias of each Linear in order), detached and contiguous, for the kernels."""
        ps = []
        for lin in self._linears():
            for p in (lin.weight, lin.bias):
                if p.device != device or p.dtype != torch.float32:
                    raise _ffi.CfmLibraryError("MLP parameters must be fp32 on the input's CUDA device")
                ps.append(p.detach().contiguous())
        return ps

    def _prepared(self, split_t, device):
        """Device blob for the kernels.  ``split_t``: treat the last input column as the shared
        scalar time (torch_wrapper path) instead of a data column."""
        key = (bool(split_t), device)
        ver = self._weights_key()
        hit = self._blobs.get(key)
        if hit is not None and hit[0] == ver:
            return hit[1]
        L = _ffi.lib()
        in0 = self.net[0].in_features
        dim = in0 - 1 if split_t else in0
        tv = 1 if split_t else 0
        nbytes = L.cfm_mlp_prepared_bytes(dim, self.w, self.out_dim, tv)
        blob = torch.empty(nbytes, dtype=torch.uint8, device=device)
        ps = self._device_params(device)
        with torch.cuda.device(device):
            _ffi.check(L.cfm_mlp_prepare(*[_ffi.ptr(p) for p in ps], dim, self.w, self.out_dim, tv,
                                         _ffi.ptr(blob), nbytes, _ffi.stream_ptr(device)),
                       "cfm_mlp_prepare")
        self._blobs[key] = (ver, blob)
        return blob

    def _grad_prepared(self, device):
        """(forward blob, gradient blob) of a scalar action for the tensor-core gradient field (csrc/grad_tc.cu): the
        gradient blob holds the transposed weight pairs of the reverse pass, built from the forward blob once per
        weight version."""
        fwd = self._prepared(True, device)
        key = ("grad", device)
        ver = (self._weights_key(), fwd.data_ptr())
        hit = self._blobs.get(key)
        if hit is not None and hit[0] == ver:
            return fwd, hit[1]
        L = _ffi.lib()
        nbytes = L.cfm_grad_tc_prepared_bytes(self.dim, self.w)
        blob = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            _ffi.check(L.cfm_grad_tc_prepare(_ffi.ptr(fwd), self.dim, self.w, _ffi.ptr(blob), nbytes,
                                             _ffi.stream_ptr(device)), "cfm_grad_tc_prepare")
        self._blobs[key] = (ver, blob)
        return fwd, blob

    def _time_reversed(self):
        """The field f_(s, x) = -f(-s, x) as an MLP: W3, b3 and the time column of W0 negated.  A decreasing
        ``t_span`` is integrated as this field over ``-t_span`` (torchdyn's reparametrisation); negation is exact
        and fmaf(-s, -w, b) == fmaf(s, w, b), so the time input keeps its bits.  Built once per weight version."""
        if not self.time_varying:
            raise RuntimeError("a time-reversed field needs an MLP built with time_varying=True")
        ver = self._weights_key()
        hit = getattr(self, "_reversed", None)  # absent on modules pickled before the cache existed
        if hit is not None and hit[0] == ver:
            m = hit[1]
        else:
            w0 = self.net[0].weight
            m = MLP(self.dim, self.out_dim, self.w, self.time_varying).to(device=w0.device, dtype=w0.dtype)
            with torch.no_grad():
                for dst, src in zip(m._linears(), self._linears()):
                    dst.weight.copy_(src.weight)
                    dst.bias.copy_(src.bias)
                m.net[0].weight[:, -1].neg_()
                m.net[6].weight.neg_()
                m.net[6].bias.neg_()
            self._reversed = (ver, m)
        m.act, m.mlp_algo = self.act, self.mlp_algo
        return m

    def _kernel_forward(self, x, t_dev, t_host, split_t, out=None):
        L = _ffi.lib()
        dev = x.device
        x = x.contiguous()
        in0 = self.net[0].in_features
        dim = in0 - 1 if split_t else in0
        if x.dim() != 2 or x.shape[1] != dim:
            raise RuntimeError(f"MLP: expected input of shape (B, {dim}), got {tuple(x.shape)}")
        B = x.shape[0]
        blob = self._prepared(split_t, dev)
        y = out if out is not None else torch.empty((B, self.out_dim), dtype=torch.float32, device=dev)
        ws = _ffi.workspace(L.cfm_mlp_workspace_bytes(B, dim, self.w, self.out_dim, self.mlp_algo), dev)
        with torch.cuda.device(dev):  # kernels launch on the current device: make it the tensors' one
            _ffi.check(L.cfm_mlp_forward_f32(
                _ffi.ptr(blob), _ffi.ptr(x), B, dim, self.w, self.out_dim, 1 if split_t else 0,
                _ffi.ptr(t_dev), float(t_host), self.act, _ffi.ptr(y), self.mlp_algo, _ffi.ptr(ws),
                ws.numel(), _ffi.stream_ptr(dev)), "cfm_mlp_forward_f32")
        return y

    def _use_kernels(self, x):
        """Sampling regime (no autograd): the kernels, or nothing -- a CPU tensor under ``torch.no_grad()`` raises
        instead of silently running ``torch.nn.Sequential`` (north_star: no CPU fallback).  With autograd enabled the
        module is plain PyTorch on any device (the device training step is ``cfm_b200.flow_matching_loss``)."""
        if torch.is_grad_enabled():
            return False
        if not x.is_cuda:
            raise _ffi.CfmLibraryError(
                "cfm_b200.MLP under torch.no_grad() runs in libcfm_b200's CUDA kernels; the input is a CPU tensor and "
                "there is no CPU fallback (enable grad for the plain-PyTorch training path)")
        return x.dtype == torch.float32

    def forward(self, x):
        """net(x) (reference models.py:20-21).  x already carries t as a column if time_varying."""
        if self._use_kernels(x):
            lead = x.shape[:-1]
            y = self._kernel_forward(x.reshape(-1, x.shape[-1]), None, 0.0, split_t=False)
            return y.reshape(*lead, self.out_dim)
        return self.net(x)

    def vector_field(self, t, x, out=None):
        """f(t, x) = net(cat([x, t*1], 1)) with ONE scalar t for the batch (utils.py:51-52), t
        folded into the first-layer bias so the concatenation never exists.  ``t`` may be a
        Python float, a 0-d/1-element tensor on any device (a CUDA tensor is read on the device,
        no sync)."""
        if not self.time_varying:
            raise RuntimeError("vector_field(t, x) needs an MLP built with time_varying=True")
        if not self._use_kernels(x):
            tt = torch.as_tensor(t, dtype=x.dtype, device=x.device)
            return self.net(torch.cat([x, tt.reshape(-1)[:1].repeat(x.shape[0])[:, None]], 1))
        if torch.is_tensor(t) and t.is_cuda:
            return self._kernel_forward(x, t.reshape(-1)[:1].float().contiguous(), 0.0, True, out)
        return self._kernel_forward(x, None, float(t), True, out)


    def tc_path(self, batch):
        """True when vector_field(t, x) for this batch runs on the tensor-core kernels."""
        if self.mlp_algo == 1 or not self.time_varying:
            return False
        return bool(_ffi.lib().cfm_mlp_tc_supported(batch, self.net[0].in_features - 1, self.w, self.out_dim))

    def vector_field_split(self, t_dev, x_hi, x_lo, out, skip_flag=None):
        """vector_field for an input already stored as its fp16x3 tensor-core operand pair (x_hi, x_lo fp16), as
        the dopri5 stage-input kernel writes it; ``t_dev`` is a 1-element CUDA tensor.  ``skip_flag``: optional
        1-element int32 CUDA tensor; the fused kernel returns at once when it is non-zero."""
        L = _ffi.lib()
        dev = x_hi.device
        dim = self.net[0].in_features - 1
        B = x_hi.shape[0]
        blob = self._prepared(True, dev)
        ws = _ffi.workspace(L.cfm_mlp_workspace_bytes(B, dim, self.w, self.out_dim, 2), dev)
        _ffi.check(L.cfm_mlp_forward_split_gated_f32(
            _ffi.ptr(blob), _ffi.ptr(x_hi), _ffi.ptr(x_lo), B, dim, self.w, self.out_dim, 1, _ffi.ptr(t_dev), 0.0,
            self.act, _ffi.ptr(out), _ffi.ptr(skip_flag), _ffi.ptr(ws), ws.numel(), _ffi.stream_ptr(dev)),
            "cfm_mlp_forward_split_gated_f32")
        return out


class GradModel(torch.nn.Module):
    """Velocity field v(x) = grad_x s(x) of a scalar action network, as action matching trains it (reference
    torchcfm/models/models.py ``GradModel``; examples/2D_tutorials/tutorial_training_8_gaussians_to_moons.ipynb
    cells 10-11).  The input carries t as its last column and v drops that column's derivative.

    ``forward`` is plain PyTorch with ``create_graph=True``, so the action-matching loss backpropagates through it on
    any device; it needs autograd and fails under ``torch.no_grad()`` as the reference does.  Sampling
    ``torch_wrapper(GradModel(MLP(dim, out_dim=1, time_varying=True)))`` with ``cfm_b200.NeuralODE`` runs the forward
    and reverse pass of the action in one kernel instead (csrc/ode_small.cu, gradient variant) for w in {32, 64} and
    dim <= 8, and on the tensor cores (csrc/grad_tc.cu: six GEMM launches per evaluation) for actions in the
    tensor-core class (B >= 128, dim >= 32, dim and w multiples of 8, w >= 32; e.g. the MNIST shape), and
    ``cfm_b200.action_matching_loss(action, xt, t, x0, x1)`` computes the notebook's training loss and all parameter
    gradients of such an action in one kernel (csrc/action_train.cu) without this double backward."""

    def __init__(self, action):
        super().__init__()
        self.action = action

    def forward(self, x):
        x = x.requires_grad_(True)
        (dsdx,) = torch.autograd.grad(torch.sum(self.action(x)), x, create_graph=True)
        return dsdx[:, :-1]


class torch_wrapper(torch.nn.Module):
    """Wraps model to torchdyn compatible format (reference torchcfm/utils.py:44-52)."""

    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, t, x, *args, **kwargs):
        if isinstance(self.model, MLP) and self.model.time_varying and self.model._use_kernels(x):
            return self.model.vector_field(t, x)
        return self.model(torch.cat([x, t.repeat(x.shape[0])[:, None]], 1))


def exact_div_fn(u):
    """div u = tr(du/dy) of a map u: R^D -> R^D at one point, from its full Jacobian (torch.func.jacrev)."""
    jac = torch.func.jacrev(u)

    def div(y, *args):
        return torch.trace(jac(y))

    return div


def div_fn_hutch_trace(u):
    """Hutchinson's estimate eps . (du/dy)^T eps of div u at one point, from one vector-Jacobian product."""
    def div(y, eps):
        _, pullback = torch.func.vjp(u, y)
        return (pullback(eps)[0] * eps).sum()

    return div


def _rademacher_like(x):
    return torch.randint_like(x, low=0, high=2).float() * 2 - 1.0


class SDE(torch.nn.Module):
    """Schrodinger-bridge SDE of the SF2M examples (examples/2D_tutorials/SF2M_tutorial.ipynb cell 5,
    examples/single_cell/single-cell_example.ipynb cell 16): dy = [drift(t, y) + score(t, y)] dt + sigma dW, Ito, with
    diagonal noise of constant scale sigma.

    ``f`` and ``g`` are the notebooks' plain-PyTorch bodies, so they run on any device and under autograd.  Under
    ``torch.no_grad()`` on CUDA, ``cfm_b200.sdeint`` integrates an SDE whose two nets are ``MLP(time_varying=True)``
    of one shape on the device instead (cfm_b200/sde.py): small nets in a single kernel, wide nets in the tensor-core
    class with one launch of both nets' forward and one step kernel per step."""
    noise_type = "diagonal"
    sde_type = "ito"

    def __init__(self, ode_drift, score, input_size=(3, 32, 32), sigma=1.0):
        super().__init__()
        self.drift = ode_drift
        self.score = score
        self.input_size = input_size
        self.sigma = sigma

    def f(self, t, y):
        """Drift: drift(t, y) + score(t, y), with t appended as the last input column."""
        y = y.view(-1, *self.input_size)
        if len(t.shape) == len(y.shape):
            x = torch.cat([y, t], 1)
        else:
            x = torch.cat([y, t.repeat(y.shape[0])[:, None]], 1)
        return self.drift(x).flatten(start_dim=1) + self.score(x).flatten(start_dim=1)

    def g(self, t, y):
        """Diffusion: sigma in every component."""
        return torch.ones_like(y) * self.sigma


class cnf_wrapper(torch.nn.Module):
    """Continuous-normalising-flow field of the maximum-likelihood tutorial
    (examples/2D_tutorials/Maximum_likelihood_CNF_tutorial.ipynb): the state is [x, ll] with the log-density change
    as its LAST column, and d/dt [x, ll] = [f(t, x), div f(t, x)].  Integrating [x1, 0] from t = 1 to t = 0 gives
    log p(x1) = prior.log_prob(x0) + ll.

    ``forward(t, x)`` is plain PyTorch (torch.func per row), so maximum-likelihood training backpropagates through it
    on any device.  On CUDA, ``cfm_b200.NeuralODE`` integrates a wrapped ``MLP(time_varying=True)`` with
    ``likelihood_estimator="exact"`` in one kernel instead (cfm_b200/ode.py).  Under autograd, with
    ``solver="euler"``, w in {32, 64}, dim <= 8 and out_dim == dim, that trajectory is differentiable: ``backward()``
    gives the exact gradient of the computed fp32 Euler trajectory for the MLP's parameters and the initial state in
    one more kernel (csrc/cnf_train.cu); for dopri5 and other shapes it raises ``NotImplementedError``.  The Hutchinson
    estimators run on the device for models in the tensor-core class (csrc/cnf_tc.cu), with probes the kernels draw."""

    def __init__(self, model, likelihood_estimator="exact"):
        super().__init__()
        self.model = model
        self.likelihood_estimator = likelihood_estimator
        self.div_fn, self.eps_fn = self.get_div_and_eps(likelihood_estimator)

    def get_div_and_eps(self, likelihood_estimator):
        """(divergence-function factory, probe-vector sampler or None) for an estimator name."""
        if likelihood_estimator == "exact":
            return exact_div_fn, None
        if likelihood_estimator == "hutch_gaussian":
            return div_fn_hutch_trace, torch.randn_like
        if likelihood_estimator == "hutch_rademacher":
            return div_fn_hutch_trace, _rademacher_like
        raise NotImplementedError(f"likelihood estimator {likelihood_estimator} is not implemented")

    def forward(self, t, x, *args, **kwargs):
        t = t.squeeze()
        x = x[..., :-1]

        def field(y):  # one row: u(y) = model([y, t])
            return self.model(torch.cat([y, t[None]]))

        div_fn = self.div_fn(field)
        if self.eps_fn is None:
            div = torch.vmap(div_fn)(x)
        else:
            div = torch.vmap(div_fn)(x, self.eps_fn(x))
        dx = self.model(torch.cat([x, t.repeat(x.shape[0])[:, None]], 1))
        return torch.cat([dx, div[:, None]], dim=-1)
