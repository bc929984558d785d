"""ctypes binding of libcfm_b200.so (the C ABI declared in include/cfm_b200.h).

No pybind / ATen coupling: tensors cross the boundary as raw ``data_ptr()`` + sizes and
the current torch CUDA stream as a ``void*``.  There is NO fallback: if the library is
missing or the device is not sm_90 every entry point raises.
"""
import ctypes as C
import os
import threading

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcfm_b200.so")

FLAG_NONFINITE, FLAG_ZERO_MASS, FLAG_NOT_CONVERGED, FLAG_INFEASIBLE = 1, 2, 4, 8
ACT_SELU, ACT_SILU = 0, 1
HUTCH_GAUSSIAN, HUTCH_RADEMACHER = 0, 1
FLOW_ICFM, FLOW_TARGET, FLOW_SB, FLOW_VP = 0, 1, 2, 3


class CfmLibraryError(RuntimeError):
    pass


class RkState(C.Structure):
    """Mirror of ``cfm_rk_state`` (include/cfm_b200.h)."""
    _fields_ = [("t", C.c_float), ("dt", C.c_float), ("t_end", C.c_float), ("atol", C.c_float),
                ("rtol", C.c_float), ("dt_old", C.c_float), ("ratio", C.c_float),
                ("ckpt_flag", C.c_int32), ("ckpt", C.c_int32), ("n_span", C.c_int32),
                ("commit", C.c_int32), ("done", C.c_int32), ("save_slot", C.c_int32),
                ("accepted", C.c_int32), ("rejected", C.c_int32), ("nfe", C.c_int32),
                ("err_acc", C.c_double)]


class SdeState(C.Structure):
    """Mirror of ``cfm_sde_state`` (include/cfm_b200.h)."""
    _fields_ = [("seed", C.c_uint64), ("traj", C.c_void_p), ("increments", C.c_void_p), ("n", C.c_int32),
                ("n_steps", C.c_int32), ("t", C.c_float), ("ticket", C.c_uint32)]


class CnfTcState(C.Structure):
    """Mirror of ``cfm_cnf_tc_state`` (include/cfm_b200.h)."""
    _fields_ = [("seed", C.c_uint64), ("traj", C.c_void_p), ("t_span", C.c_void_p), ("n", C.c_int32),
                ("n_steps", C.c_int32), ("t", C.c_float), ("ticket", C.c_uint32)]


class GradTcState(C.Structure):
    """Mirror of ``cfm_grad_tc_state`` (include/cfm_b200.h)."""
    _fields_ = [("traj", C.c_void_p), ("t_span", C.c_void_p), ("n", C.c_int32), ("n_steps", C.c_int32),
                ("t", C.c_float), ("ticket", C.c_uint32)]


_p, _i, _i64, _f, _d, _sz =C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_double, C.c_size_t

# name -> (restype, argtypes); must list every symbol include/cfm_b200.h declares
SIGNATURES = {
    "cfm_abi_version": (_i, []),
    "cfm_last_error": (C.c_char_p, []),
    "cfm_device_info": (_i, [C.POINTER(_i), C.POINTER(_i)]),
    "cfm_launch_count": (C.c_longlong, []),
    "cfm_sqdist_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "cfm_sqdist_f32": (_i, [_p, _p, _p, _i, _i, _i, _i64, _i, _p, _i, _p, _sz, _p]),
    "cfm_sinkhorn_workspace_bytes": (_sz, [_i, _i]),
    "cfm_sinkhorn_log_f32": (_i, [_p, _i, _i, _i64, _f, _p, _i, _i, _d, _i, _i, _d, _p, _p, _p, _p,
                                  _p, _sz, _p]),
    "cfm_plan_materialize_f64": (_i, [_p, _i, _i, _i64, _f, _p, _i, _p, _p, _p, _p, _p, _p]),
    "cfm_plan_dot_cost": (_i, [_p, _i, _i, _i64, _f, _p, _i, _p, _p, _p, _p]),
    "cfm_plan_sample_workspace_bytes": (_sz, [_i]),
    "cfm_plan_sample": (_i, [_p, _i, _i, _i64, _f, _p, _i, _p, _p, _i, _p, _i, _p, _p, _p, _p, _sz, _p]),
    "cfm_plan_sample_rows": (_i, [_p, _i, _i, _i64, _f, _p, _i, _p, _p, _p, _p, _i, _p, _p, _p]),
    "cfm_dense_plan_sample_f64": (_i, [_p, _i, _i, _p, _i, _p, _p, _p, _sz, _p]),
    "cfm_perm_plan_sample": (_i, [_p, _p, _i, _p, _i, _p, _p, _p]),
    "cfm_assign_workspace_bytes": (_sz, [_i]),
    "cfm_assign_exact_f32": (_i, [_p, _i, _i64, _p, _i, _p, _p, _p, _p, _sz, _p]),
    "cfm_gather_rows": (_i, [_p, _i64, _i, _p, _i64, _p, _p]),
    "cfm_flow_pairs_f32": (_i, [_i, _p, _p, _p, _p, _p, _p, _p, _p, _p, _f, _f, _p, _p, _i64, _i64, _p]),
    "cfm_mlp_prepared_bytes": (_sz, [_i, _i, _i, _i]),
    "cfm_mlp_prepare": (_i, [_p] * 8 + [_i, _i, _i, _i, _p, _sz, _p]),
    "cfm_mlp_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "cfm_mlp_forward_f32": (_i, [_p, _p, _i, _i, _i, _i, _i, _p, _f, _i, _p, _i, _p, _sz, _p]),
    "cfm_mlp_tc_supported": (_i, [_i, _i, _i, _i]),
    "cfm_mlp_forward_split_gated_f32": (_i, [_p, _p, _p, _i, _i, _i, _i, _i, _p, _f, _i, _p, _p, _p, _sz, _p]),
    "cfm_rk_stage_input": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _i64, _i, _p]),
    "cfm_rk_error_norm": (_i, [_p, _p, _p, _p, _p, _i64, _p]),
    "cfm_rk_control": (_i, [_p, _p, _i64, _p]),
    "cfm_rk_commit": (_i, [_p, _p, _p, _p, _p, _i64, _p]),
    "cfm_rk_init_sums": (_i, [_p, _p, _p, _p, _p, _i64, _i, _p]),
    "cfm_rk_init_probe": (_i, [_p, _p, _p, _p, _p, _p, _i64, _i64, _p]),
    "cfm_rk_init_finish": (_i, [_p, _p, _p, _i64, _p]),
    "cfm_axpy_f32": (_i, [_p, _p, _f, _p, _i64, _p]),
    "cfm_ode_small_supported": (_i, [_i64, _i, _i, _i]),
    "cfm_ode_small_workspace_bytes": (_sz, [_i64, _i, _i]),
    "cfm_ode_small_trajectory_f32": (_i, [_p] * 8 + [_i, _i, _i, _i, _p, _i64, _p, _i, _f, _f, _i, _p, _p, _p, _sz, _p]),
    "cfm_ode_small_cnf_supported": (_i, [_i64, _i, _i]),
    "cfm_ode_small_cnf_trajectory_f32": (_i, [_p] * 8 + [_i, _i, _i, _i, _p, _i64, _p, _i, _f, _f, _i, _p, _p, _p, _sz,
                                                          _p]),
    "cfm_ode_small_cnf_backward_supported": (_i, [_i64, _i, _i]),
    "cfm_ode_small_cnf_backward_workspace_bytes": (_sz, [_i64, _i, _i, _i]),
    "cfm_ode_small_cnf_euler_backward_f32": (_i, [_p] * 8 + [_i, _i, _i, _p, _i64, _p, _i, _p, _p, _p, _p, _sz, _p]),
    "cfm_ode_small_grad_supported": (_i, [_i64, _i, _i]),
    "cfm_ode_small_grad_trajectory_f32": (_i, [_p] * 8 + [_i, _i, _i, _i, _p, _i64, _p, _i, _f, _f, _i, _p, _p, _p,
                                                           _sz, _p]),
    "cfm_sde_small_supported": (_i, [_i64, _i, _i]),
    "cfm_sde_small_euler_f32": (_i, [_p, _p, _i, _i, _i, _f, _p, _i64, _p, _i, _p, _p, _p, _i, C.c_uint64, _p, _p,
                                     _p]),
    "cfm_sde_tc_supported": (_i, [_i, _i, _i]),
    "cfm_mlp_pair_forward_split_f32": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _f, _i, _p, _p, _p, _sz, _p]),
    "cfm_sde_tc_init": (_i, [_p, _p, _p, _p, _p, _p, _p, C.c_uint64, _p, _i, _i, _i, _p]),
    "cfm_sde_tc_euler_step": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _f, _i, _i, _p]),
    "cfm_cnf_tc_supported": (_i, [_i, _i, _i]),
    "cfm_cnf_tc_workspace_bytes": (_sz, [_i, _i, _i]),
    "cfm_cnf_tc_field_f32": (_i, [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p, _p, _p, _i, _p, _p, _p, _sz, _p]),
    "cfm_cnf_tc_euler_init": (_i, [_p, _p, _p, _p, _p, _p, _p, _p, _i, C.c_uint64, _i, _i, _p]),
    "cfm_cnf_tc_euler_step": (_i, [_p, _p, _p, _p, _p, _p, _p, _i, _i, _p]),
    "cfm_grad_tc_supported": (_i, [_i, _i, _i]),
    "cfm_grad_tc_prepared_bytes": (_sz, [_i, _i]),
    "cfm_grad_tc_prepare": (_i, [_p, _i, _i, _p, _sz, _p]),
    "cfm_grad_tc_workspace_bytes": (_sz, [_i, _i, _i]),
    "cfm_grad_tc_field_f32": (_i, [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p, _p, _p, _sz, _p]),
    "cfm_grad_tc_euler_init": (_i, [_p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p]),
    "cfm_grad_tc_euler_step": (_i, [_p, _p, _p, _p, _p, _i, _i, _p]),
    "cfm_mlp_small_train_supported":(_i, [_i64, _i, _i, _i]),
    "cfm_mlp_small_train_workspace_bytes": (_sz, [_i64, _i, _i, _i]),
    "cfm_mlp_small_mse_grad_f32": (_i, [_p] * 8 + [_i, _i, _i, _i, _p, _p, _p, _p, _i64, _i, _p, _p, _p, _sz, _p]),
    "cfm_mlp_small_action_grad_f32": (_i, [_p] * 8 + [_i, _i, _i, _p, _p, _p, _p, _i64, _i, _p, _p, _p, _sz, _p]),
    "cfm_mlp_tc_train_supported": (_i, [_i64, _i, _i, _i]),
    "cfm_mlp_tc_train_workspace_bytes": (_sz, [_i64, _i, _i, _i]),
    "cfm_mlp_tc_mse_grad_f32": (_i, [_p] * 8 + [_i, _i, _i, _i, _p, _p, _p, _p, _i64, _i, _p, _p, _p, _sz, _p]),
}

_lock = threading.Lock()
_lib = None


def load_library(path=LIB_PATH):
    """dlopen the library and bind every declared symbol (no CUDA call is made)."""
    if not os.path.exists(path):
        raise CfmLibraryError(
            f"{path} not found: build it with `python -m cfm_b200.build` "
            "(cfm_b200 has no CPU / PyTorch fallback path)")
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


def lib():
    global _lib
    if _lib is None:
        with _lock:
            if _lib is None:
                _lib = load_library()
    return _lib


def last_error():
    return lib().cfm_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise CfmLibraryError(f"{what} failed (code {rc}): {last_error()}")


def require_device():
    """Raise unless a CUDA sm_90 device is usable; returns (sm_count, cc)."""
    if not torch.cuda.is_available():
        raise CfmLibraryError("cfm_b200 needs a CUDA device (sm_90a); none is available and "
                              "there is no CPU fallback")
    sms, cc = C.c_int(0), C.c_int(0)
    check(lib().cfm_device_info(C.byref(sms), C.byref(cc)), "cfm_device_info")
    return sms.value, cc.value


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def stream_ptr(device=None):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def workspace(nbytes, device):
    """Scratch bytes from torch's caching allocator (the library never allocates)."""
    return torch.empty(max(int(nbytes), 16), dtype=torch.uint8, device=device)


def replay_steps(plan, step, n_steps, graph):
    """Enqueue ``n_steps`` calls of ``step``, which launches one step on the current stream and reads everything that
    changes from step to step from device memory.  With ``graph``, the first call of a plan runs step 0 eagerly (which
    loads every kernel), captures one step into ``plan["graph"]`` when more steps follow, and replays it for the rest;
    later calls replay it for every step.  Without ``graph`` every step is enqueued eagerly."""
    first = 0
    if not graph or plan["graph"] is None:
        step()
        first = 1
        if graph and n_steps > 1:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                step()
            plan["graph"] = g
    for _ in range(first, n_steps):
        if graph:
            plan["graph"].replay()
        else:
            step()
