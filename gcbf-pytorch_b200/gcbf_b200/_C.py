"""ctypes binding of libgcbf_b200.so (C ABI declared in include/gcbf_b200.h).

The library is loaded lazily on first use.  There is NO fallback: if the shared object is missing or a
call fails, a RuntimeError is raised (the product path must never silently run on the CPU).
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_longlong, c_size_t, c_ulonglong, c_void_p

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('GCBF_B200_LIB') or os.path.join(_HERE, 'libgcbf_b200.so')   # (override: kernel experiments)
_lib = None


class EnvCfg(ctypes.Structure):
    """mirror of `gcbf_env_cfg`"""
    _fields_ = [('env', c_int32), ('num_graphs', c_int32), ('nodes_per_graph', c_int32), ('num_agents', c_int32),
                ('agent_radius', c_double), ('speed_limit', c_double), ('dist2goal', c_double), ('dt', c_double)]


class SnLayer(ctypes.Structure):
    """mirror of `gcbf_sn_layer`"""
    _fields_ = [('W', c_void_p), ('ldw', c_int32), ('N', c_int32), ('K', c_int32), ('pad_', c_int32), ('u', c_void_p),
                ('v', c_void_p), ('inv_sigma', c_void_p)]


class SplitDesc(ctypes.Structure):
    """mirror of `gcbf_split_desc`"""
    _fields_ = [('src', c_void_p), ('ld', c_int32), ('rows', c_int32), ('cols', c_int32), ('ld_h', c_int32),
                ('amax_slot', c_void_p), ('dst', c_void_p)]


class ResetDesc(ctypes.Structure):
    """mirror of `gcbf_reset_desc`"""
    _fields_ = [('seed', c_ulonglong), ('states', c_void_p), ('goals', c_void_p), ('step_count', c_void_p), ('episode', c_void_p),
                ('failed', c_void_p), ('reach', c_void_p), ('env', c_int32), ('num_envs', c_int32), ('num_agents', c_int32),
                ('num_obs', c_int32), ('ld_state', c_int32), ('ld_goal', c_int32), ('goal_dim', c_int32), ('max_steps', c_int32),
                ('max_tries', c_int32), ('first_env', c_int32), ('area', c_float), ('agent_dist2', c_float), ('goal_dist2', c_float),
                ('clear2', c_float), ('obs_speed_limit', c_float), ('pad_', c_float)]


P = c_void_p  # every device pointer travels as void*
_SIGS = {
    'gcbf_last_error': (c_char_p, []),
    'gcbf_abi_version': (c_int, []),
    'gcbf_abi_struct_size': (c_size_t, [c_int]),
    'gcbf_launch_count': (c_longlong, [c_int]),
    'gcbf_has_wgmma': (c_int, []),
    'gcbf_last_gemm_impl': (c_int, []),
    'gcbf_radius_graph_count': (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, P, P]),
    'gcbf_radius_graph_fill': (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, P, P, c_int64, P]),
    'gcbf_rowptr_from_targets': (c_int, [P, c_int64, c_int, P, P, P]),
    'gcbf_edge_attr_fwd': (c_int, [c_int, P, c_int, P, c_int64, P, P]),
    'gcbf_edge_attr_bwd': (c_int, [c_int, P, c_int, P, c_int64, P, P, P]),
    'gcbf_edge_input_fwd': (c_int, [P, c_int, P, c_int, P, c_int64, P, c_int, P]),
    'gcbf_linear_fwd': (c_int, [P, c_int, P, c_int, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, P, P]),
    'gcbf_linear_bwd_data': (c_int, [P, c_int, P, c_int, P, P, c_int, P, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'gcbf_linear_bwd_weight': (c_int, [P, c_int, P, c_int, P, P, c_int, P, c_int, c_int, c_int, c_int, c_int, P]),
    'gcbf_amax_f32': (c_int, [P, c_int, c_int, c_int, P, c_int, P]),
    'gcbf_split_f16': (c_int, [P, c_int, c_int, c_int, P, P, c_int, P, c_int, P]),
    'gcbf_amax_split_batched': (c_int, [POINTER(SplitDesc), c_int, P]),
    'gcbf_linear_h_supported': (c_int, [c_int, c_int, c_int]),
    'gcbf_linear_fwd_h': (c_int, [P, c_int, P, P, c_int, P, P, P, P, c_int, c_int, c_int, c_int, c_int, P, P]),
    'gcbf_linear_bwd_data_h': (c_int, [P, c_int, P, P, c_int, P, P, P, c_int, P, c_int, c_int, c_int, c_int, c_int, P, P]),
    'gcbf_linear_bwd_weight_h': (c_int, [P, c_int, P, P, c_int, P, P, P, c_int, c_int, c_int, c_int, c_int, P]),
    'gcbf_act_bwd': (c_int, [P, P, P, c_int64, c_int, P]),
    'gcbf_attn_aggr_fwd': (c_int, [P, c_int, P, P, c_int, c_int, P, P, c_int, P]),
    'gcbf_attn_aggr_bwd': (c_int, [P, c_int, P, P, c_int, c_int, P, c_int, P, c_int, P, c_int, P]),
    'gcbf_rows_gather': (c_int, [P, c_int, P, P, c_int, c_int64, c_int, P]),
    'gcbf_rows_scatter': (c_int, [P, c_int, P, P, c_int, c_int64, c_int, P]),
    'gcbf_copy2d': (c_int, [P, c_int, P, c_int, c_int64, c_int, P]),
    'gcbf_u_ref': (c_int, [POINTER(EnvCfg), P, c_int, P, c_int, P, P, P]),
    'gcbf_step_fwd': (c_int, [POINTER(EnvCfg), P, c_int, P, P, c_int, P, c_int, P, P, P]),
    'gcbf_step_bwd': (c_int, [POINTER(EnvCfg), P, c_int, P, P, P]),
    'gcbf_u_ref_multi': (c_int, [POINTER(EnvCfg), P, c_int, P, c_int, P, P, P]),
    'gcbf_step_fwd_multi': (c_int, [POINTER(EnvCfg), P, c_int, P, P, c_int, P, c_int, P, P, P]),
    'gcbf_masks': (c_int, [POINTER(EnvCfg), P, c_int, P, P, P, P]),
    'gcbf_loss_partials': (c_int, [P, P, P, P, c_int, P, P, c_int64, c_float, c_float, c_float, P, P, P]),
    'gcbf_loss_grads': (c_int, [P, P, P, P, c_int, P, P, c_int64, c_float, c_float, c_float, c_float, c_float, c_float,
                                c_float, P, P, P, P, P, P]),
    'gcbf_pair_count': (c_int, [P, c_int64, P, c_int64, c_float, P, P]),
    'gcbf_sn_workspace_floats': (c_size_t, [c_int, c_int]),
    'gcbf_sn_power_iter': (c_int, [P, c_int, c_int, c_int, P, P, P, P, P]),
    'gcbf_sn_power_iter_batched': (c_int, [POINTER(SnLayer), c_int, P, c_size_t, P]),
    'gcbf_sn_grad_fixup': (c_int, [P, c_int, P, c_int, c_int, c_int, P, P, P, P, P, c_int, P]),
    'gcbf_grad_sumsq': (c_int, [P, c_int64, P, P]),
    'gcbf_clip_adam': (c_int, [P, P, P, P, c_int64, P, c_double, c_double, c_double, c_double, c_double, c_int, P]),
    # MACBF baseline (csrc/macbf.cu)
    'gcbf_radius_graph_topk_count': (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_int, P, P]),
    'gcbf_radius_graph_topk_fill': (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_int, P, P, c_int64, P]),
    'gcbf_edge_masks': (c_int, [P, c_int, c_int, c_int64, c_double, P, P, P]),
    'gcbf_seg_max_fwd': (c_int, [P, c_int, P, c_int, c_int, P, c_int, P, P]),
    'gcbf_seg_max_bwd': (c_int, [P, c_int, P, c_int, c_int, P, c_int, c_int64, P]),
    'gcbf_macbf_loss_partials': (c_int, [P, P, P, P, c_int64, P, c_int, c_int64, c_float, c_float, c_float, P, P]),
    # analytic h_dot (csrc/jvp.cu)
    'gcbf_state_dot': (c_int, [POINTER(EnvCfg), P, c_int, P, P, P, c_int, c_int, c_int, P, c_int, P]),
    'gcbf_edge_attr_tangent': (c_int, [c_int, P, c_int, P, c_int, P, c_int64, P, P]),
    'gcbf_attn_aggr_tangent': (c_int, [P, c_int, P, c_int, P, P, P, c_int, c_int, P, c_int, P]),
    # backward of the analytic h_dot pass (csrc/jvp.cu, csrc/loss.cu)
    'gcbf_attn_aggr_tangent_bwd': (c_int, [P, c_int, P, c_int, P, P, P, c_int, c_int, P, c_int, P, c_int, P, P, c_int, P, c_int, P]),
    'gcbf_act_tangent_bwd': (c_int, [P, P, P, P, c_int64, c_int, P, P, P]),
    'gcbf_state_dot_bwd': (c_int, [POINTER(EnvCfg), P, c_int, P, P, P, c_int, c_int, c_int, P, c_int, P, c_int, P]),
    'gcbf_edge_attr_bwd_ordered': (c_int, [c_int, P, c_int, P, c_int64, c_int, P, P, P]),
    'gcbf_loss_partials_hdot': (c_int, [P, P, P, c_int, P, P, c_int64, c_float, c_float, P, P]),
    'gcbf_loss_grads_hdot': (c_int, [P, P, P, c_int, P, P, c_int64, c_float, c_float, c_float, c_float, c_float, c_float, P, P, P, P, P, P]),
    'gcbf_macbf_loss_grads': (c_int, [P, P, P, P, c_int64, P, c_int, c_int64, c_float, c_float, c_float, c_float, c_float, c_float,
                                      c_float, P, P, P, P, P, P]),
    # batched episode reset (csrc/reset.cu)
    'gcbf_env_reset_batch': (c_int, [POINTER(ResetDesc), P]),
}
EXPORTED_SYMBOLS = tuple(_SIGS)


def library_available() -> bool:
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f'{LIB_PATH} not found: build it with `python gcbf-pytorch_b200/csrc/build.py` '
                '(gcbf_b200 has no CPU / eager fallback)')
        _lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(_lib, name)
            fn.restype = res
            fn.argtypes = args
    return _lib


def register(sigs: dict):
    """Add entry-point signatures (the chain-level ABI is declared next to its ctypes structures in native.py)."""
    global EXPORTED_SYMBOLS
    _SIGS.update(sigs)
    EXPORTED_SYMBOLS = tuple(_SIGS)
    if _lib is not None:
        for name, (res, args) in sigs.items():
            f = getattr(_lib, name)
            f.restype = res
            f.argtypes = args


def ptr(t):
    """device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


_raw_stream = getattr(torch._C, '_cuda_getCurrentRawStream', None)
_get_device = getattr(torch._C, '_cuda_getDevice', None)


def stream():
    """cudaStream_t of torch's current stream on the current device (raw C accessors: this sits on the launch path of
    every kernel, and torch.cuda.current_stream() costs ~14 us of Python per call)."""
    if _raw_stream is not None and _get_device is not None:
        return _raw_stream(_get_device())
    return torch.cuda.current_stream().cuda_stream


def check(rc, what):
    if rc != 0:
        msg = lib().gcbf_last_error()
        raise RuntimeError(f'{what} failed (code {rc}): {msg.decode() if msg else ""}')


# kernels launched by one call of each entry point (for bench.py's `gpu_launches`; memsets are not counted)
_KERNELS_PER_CALL = {'gcbf_radius_graph_count': 2, 'gcbf_radius_graph_topk_count': 2, 'gcbf_sn_power_iter': 4, 'gcbf_sn_power_iter_batched': 4, 'gcbf_sn_grad_fixup': 2, 'gcbf_linear_bwd_weight': 2,
                     'gcbf_linear_h_supported': 0, 'gcbf_amax_split_batched': 2}
KERNEL_LAUNCHES = 0
ABI_CALLS = 0


def reset_counters():
    global KERNEL_LAUNCHES, ABI_CALLS
    KERNEL_LAUNCHES = 0
    ABI_CALLS = 0
    lib().gcbf_launch_count(1)


def kernel_launches() -> int:
    """Kernels launched since reset_counters(): by per-kernel entry points called from Python (counted here) and by the
    chain-level entry points (counted inside the library, csrc/net.cu)."""
    return KERNEL_LAUNCHES + int(lib().gcbf_launch_count(0))


_FN = {}


def call(name, *args):
    """Invoke a status-returning entry point on the current CUDA stream and raise on error."""
    global KERNEL_LAUNCHES, ABI_CALLS
    fn = _FN.get(name)
    if fn is None:
        fn = _FN[name] = getattr(lib(), name)
    rc = fn(*args, stream())
    if rc != 0:
        check(rc, name)
    ABI_CALLS += 1
    KERNEL_LAUNCHES += _KERNELS_PER_CALL.get(name, 1)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError('gcbf_b200 ops need CUDA tensors: there is no CPU fallback '
                               '(build the library with __graft_entry__.build() and run on a GPU)')
