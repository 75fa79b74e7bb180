"""ctypes binding of libdisvae_b200.so (C ABI in include/disvae_b200.h).

The library is the only compute backend of this package: there is NO PyTorch/CPU fallback.
If the shared object is missing, or a tensor is not a CUDA fp32 tensor, the call raises.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_ulonglong, c_void_p

import torch

_PKG_DIR = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB_PATH = os.path.join(_PKG_DIR, "libdisvae_b200.so")

ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_LEAKY = 0, 1, 2, 3
DIST = {"bernoulli": 0, "gaussian": 1, "laplace": 2}

P, I, LL, F, SZ, ULL, DBL = c_void_p, c_int, c_longlong, c_float, c_size_t, c_ulonglong, c_double

# name -> (restype, argtypes); mirrors include/disvae_b200.h one to one
SIGNATURES = {
    "dv_version": (I, []),
    "dv_built_arch": (I, []),
    "dv_status_string": (c_char_p, [I]),
    "dv_last_cuda_error": (I, []),
    "dv_device_check": (I, []),
    "dv_launch_count": (LL, []),
    "dv_conv_packed_floats": (SZ, [I]),
    "dv_conv_pack_weights": (I, [P, P, I, P]),
    "dv_conv_pack_multi": (I, [I, P, P, P, P]),
    "dv_conv_down": (I, [P, P, P, P, P, I, I, I, I, I, I, P, P, P, P, P]),
    "dv_conv_up": (I, [P, P, P, P, P, I, I, I, I, I, I, P, P, P]),
    "dv_conv_wgrad_workspace_bytes": (SZ, [I, I, I, I]),
    "dv_conv_wgrad": (I, [P, P, P, P, P, SZ, I, I, I, I, I, P]),
    "dv_channel_sum_workspace_bytes": (SZ, []),
    "dv_channel_sum": (I, [P, P, LL, I, I, I, P, P]),
    "dv_flat_transpose": (I, [P, P, I, I, I, I, P]),
    "dv_act_bwd": (I, [P, P, P, LL, I, F, P]),
    "dv_linear_fwd_workspace_bytes": (SZ, [I, I, I]),
    "dv_linear_dgrad_workspace_bytes": (SZ, [I, I, I]),
    "dv_linear_fwd": (I, [P, P, P, P, I, I, I, I, F, P, P]),
    "dv_linear_dgrad": (I, [P, P, P, P, I, I, I, I, F, P, P]),
    "dv_linear_packed_floats": (SZ, [I, I]),
    "dv_linear_pack_multi": (I, [I, P, P, P, P, P]),
    "dv_linear_fwd_packed": (I, [P, P, P, P, P, I, I, I, I, F, P]),
    "dv_linear_dgrad_packed": (I, [P, P, P, P, P, I, I, I, I, F, P]),
    "dv_linear_wgrad_workspace_bytes": (SZ, [I, I, I]),
    "dv_linear_wgrad": (I, [P, P, P, P, I, I, I, P, P]),
    "dv_reparam_fwd": (I, [P, P, I, I, P, ULL, P, P, P, I, I, P]),
    "dv_reparam_bwd": (I, [P, P, I, I, P, P, P, I, I, P]),
    "dv_vae_loss_workspace_bytes": (SZ, [I, LL]),
    "dv_vae_loss_fwd": (I, [P, P, LL, I, I, P, P, I, I, I, P, P, P]),
    "dv_vae_loss_bwd": (I, [P, P, LL, I, I, P, P, I, I, I, P, P, P, P, P, P]),
    "dv_btcvae_workspace_bytes": (SZ, [I, I]),
    "dv_btcvae_fwd": (I, [P, P, P, I, I, I, I, LL, I, P, P, P, P]),
    "dv_btcvae_bwd": (I, [I, I, LL, I, P, P, P, P, P, P, P]),
    "dv_btcvae_fwd_rows": (I, [P, P, P, I, I, I, I, I, I, LL, I, P, P, P, P]),
    "dv_btcvae_bwd_rows": (I, [I, I, I, I, LL, I, P, P, P, P, P, P, P]),
    "dv_u8_to_f32": (I, [P, P, LL, P]),
    "dv_gather_u8_to_f32": (I, [P, P, I, I, P, P]),
    "dv_loss_combine_fwd": (I, [P, P, I, P, P, I, P, P]),
    "dv_loss_combine_bwd": (I, [P, P, I, I, P, I, P, P, P]),
    "dv_loss_combine_sched_fwd": (I, [P, I, P, I, P, I, DBL, DBL, LL, I, P, P, P, P, P]),
    "dv_loss_combine_sched_bwd": (I, [P, P, I, I, I, P, P, P]),
    "dv_betab_loss_fwd": (I, [P, DBL, DBL, DBL, LL, I, P, P, P, P, P]),
    "dv_betab_loss_bwd": (I, [P, P, P, I, P, P]),
    "dv_loss_record": (I, [P, P, P]),
    "dv_act_bwd_chansum": (I, [P, P, P, I, I, I, I, F, P, P, P]),
    "dv_latent_entropy_workspace_bytes": (SZ, [I, I, I]),
    "dv_latent_entropy": (I, [P, P, P, I, I, I, I, I, P, P, P, P]),
    "dv_permute_dims": (I, [P, P, ULL, P, P, I, I, P]),
    "dv_permute_dims_workspace_bytes": (SZ, [I, I]),
    "dv_permute_dims_rows": (I, [P, P, ULL, P, P, I, I, I, I, P, P]),
    "dv_index_permutation_workspace_bytes": (SZ, [I]),
    "dv_index_permutation": (I, [I, ULL, P, P, P, P]),
    "dv_factor_tc_fwd": (I, [P, I, P, P]),
    "dv_factor_tc_bwd": (I, [P, I, P, P]),
    "dv_factor_ce_fwd": (I, [P, P, I, P, P]),
    "dv_factor_ce_bwd": (I, [P, P, P, I, P, P, P]),
    "dv_adam_step": (I, [P, P, P, P, P, LL, F, DBL, DBL, F, F, P]),
    "dv_adam_multi_max_tensors": (I, []),
    "dv_adam_multi": (I, [I, P, P, P, P, P, P, F, DBL, DBL, F, F, P]),
}

LOSS_LOG_MAX_SRC = 8


class LossLog(ctypes.Structure):
    """dv_loss_log: where a recording step's scalars go (device ring [cap][ncols]) and where they come from."""
    _fields_ = [("ring", c_void_p), ("cap", c_int), ("ncols", c_int), ("every", c_int), ("nsrc", c_int),
                ("src", c_void_p * LOSS_LOG_MAX_SRC), ("len", c_int * LOSS_LOG_MAX_SRC)]


_lib = None
GRAPH_LAUNCHES = 0       # kernels launched through CUDA-graph replays (dv_launch_count() only sees direct launches)


class NativeLibraryMissing(RuntimeError):
    pass


def lib():
    """Load (once) and return the ctypes handle.  Raises if the .so has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryMissing(
                "libdisvae_b200.so not found at %s -- build it with "
                "`python disentangling-vae_b200/build.py` (or __graft_entry__.build()). "
                "This package has no CPU/PyTorch fallback." % LIB_PATH)
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def ptr(t):
    """Device pointer of a CUDA fp32 (or int64) tensor, None -> NULL."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("disvae_b200: expected a CUDA tensor, got a %s tensor (no CPU fallback exists)" % t.device)
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def check(status, what):
    if status != 0:
        L = lib()
        msg = L.dv_status_string(status).decode()
        extra = ""
        if status == -4:
            extra = " (cudaError %d)" % L.dv_last_cuda_error()
        raise RuntimeError("disvae_b200.%s failed: %s%s" % (what, msg, extra))


# ---- optional per-entry-point device timing (bench.py roofline pass) ----------------------
_prof_events = None      # list of (name, start_event, end_event) while profiling is enabled
PROFILE_ONLY = None      # restrict to one entry point


def enable_profiling():
    """Bracket every C-ABI call with CUDA events on the launching (current) stream."""
    global _prof_events
    _prof_events = []
    return _prof_events


def disable_profiling():
    """Stop profiling; returns {entry point: (total ms, calls)}."""
    global _prof_events
    ev, _prof_events = _prof_events, None
    torch.cuda.synchronize()
    table = {}
    for name, e0, e1 in ev or []:
        t, n = table.get(name, (0.0, 0))
        table[name] = (t + e0.elapsed_time(e1), n + 1)
    return table


def call(name, *args, tag=None):
    """Invoke a C-ABI entry point.  `tag` (e.g. the layer geometry) only labels profiling records."""
    if _prof_events is not None and (PROFILE_ONLY is None or PROFILE_ONLY == name):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        check(getattr(lib(), name)(*args), name)
        e1.record()
        _prof_events.append((name if tag is None else "%s%s" % (name, tag), e0, e1))
        return
    check(getattr(lib(), name)(*args), name)


def launch_count():
    """Kernels of this library launched so far, including those replayed inside CUDA graphs."""
    return lib().dv_launch_count() + GRAPH_LAUNCHES


def require_cuda_f32(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("disvae_b200 runs on CUDA only: got a tensor on %s. Move the model and data to a "
                               "GPU (`.to('cuda')`); there is no CPU path." % t.device)
        if t.dtype != torch.float32:
            raise RuntimeError("disvae_b200 computes in fp32; got %s" % t.dtype)
