"""cfm_b200 -- H100-native (sm_90a) implementation of torchcfm's two numeric hot paths:

(A) the minibatch optimal-transport coupling behind ``OTPlanSampler`` (cost matrix, log-domain
    Sinkhorn or exact assignment, pair draw, gather), and
(B) the batched MLP vector-field forward evaluated at every ODE step during sampling,

behind the reference's own Python API (torchcfm 1.0.7).  Host code is Python/PyTorch; all
arithmetic of the two paths runs in hand-written CUDA behind the C ABI in include/cfm_b200.h.
Importing this package does not need a GPU; calling into the hot path without libcfm_b200.so or
an sm_90 device raises (there is no CPU fallback).
"""
from .conditional_flow_matching import *  # noqa: F401,F403
from .conditional_flow_matching import (ConditionalFlowMatcher,  # noqa: F401
                                        ExactOptimalTransportConditionalFlowMatcher,
                                        SchrodingerBridgeConditionalFlowMatcher,
                                        TargetConditionalFlowMatcher,
                                        VariancePreservingConditionalFlowMatcher, pad_t_like_x)
from .models import MLP, SDE, cnf_wrapper, torch_wrapper  # noqa: F401
from .ode import NeuralODE  # noqa: F401
from .optimal_transport import CouplingStream, OTPlanSampler, wasserstein  # noqa: F401
from .sde import sdeint  # noqa: F401

__version__ = "0.1.0"
