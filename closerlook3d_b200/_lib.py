"""ctypes binding of libcl3d.so (include/cl3d.h).  No fallback: if the library is missing or a call fails,
a RuntimeError / ImportError is raised (the reference's TORCH_CHECK -> RuntimeError convention,
_ext_src/include/utils.h:9-30)."""
import ctypes
import os

import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(_PKG, "libcl3d.so")
_lib = None

_vp = ctypes.c_void_p
_i = ctypes.c_int
_f = ctypes.c_float
_sz = ctypes.c_size_t
_ll = ctypes.c_longlong

# name -> (restype, argtypes); must list every symbol include/cl3d.h declares (tests check this)
SIGNATURES = {
    "cl3d_version": (_i, []),
    "cl3d_last_error": (ctypes.c_char_p, []),
    "cl3d_padded_channels": (_i, [_i]),
    "cl3d_sm_count": (_i, []),
    "cl3d_launch_count": (_ll, []),
    "cl3d_ball_query_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "cl3d_ball_query_algo": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _i, _vp, _vp, _vp, _vp, _sz, _i, _vp]),
    "cl3d_ball_query_csr_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "cl3d_ball_query_csr": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _sz, _i, _i, _i, _vp]),
    "cl3d_nearest_query_workspace_bytes": (_sz, [_i, _i, _i]),
    "cl3d_nearest_query": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "cl3d_csr_workspace_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "cl3d_build_csr": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _i, _vp]),
    "cl3d_group_points": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp]),
    "cl3d_group_points_grad": (_i, [_vp, _i, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "cl3d_grid_subsample_workspace_bytes": (_sz, [_i, _i, _i]),
    "cl3d_grid_subsample": (_i, [_vp, _vp, _i, _i, _i, _f, _vp, _vp, _vp, _sz, _vp]),
    "cl3d_gather_max_fwd": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _i, _vp, _vp]),
    "cl3d_gather_max_bwd": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "cl3d_to_point_major": (_i, [_vp, _i, _i, _i, _i, _vp, _vp]),
    "cl3d_to_channel_major": (_i, [_vp, _i, _i, _i, _vp, _i, _vp]),
    "cl3d_agg_num_tiles": (_i, [_i, _i]),
    "cl3d_agg_num_params": (_i, [_i, _i, _i, _i]),
    "cl3d_agg_bwd_num_blocks": (_i, [_i, _i]),
    "cl3d_agg_fwd": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _i, _i, _f, _i, _vp,
                          _vp, _vp, _vp]),
    "cl3d_agg_bwd": (_i, [_i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _i, _i, _i,
                          _f, _i, _vp, _i, _vp, _vp, _vp]),
    "cl3d_reduce_partials": (_i, [_vp, _i, _i, _vp, _vp]),
    "cl3d_bn_finalize": (_i, [_vp, _i, _i, _ll, _f, _f, _i, _vp, _vp, _vp, _vp]),
    "cl3d_bn_relu_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp, _i, _vp]),
    "cl3d_bn_relu_bwd": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp]),
    "cl3d_bn_relu_bwd_stats": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "cl3d_bn_relu_bwd_apply": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "cl3d_bn_rank_moments": (_i, [_vp, _i, _i, _ll, _vp, _vp]),
    "cl3d_bn_finalize_ranks": (_i, [_vp, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _vp]),
    "cl3d_sgemm_workspace_bytes": (_sz, [_i, _i, _i]),
    "cl3d_sgemm_algo": (_i, [_vp, _ll, _ll, _vp, _ll, _ll, _i, _i, _i, _vp, _ll, _i, _vp, _sz, _i, _vp]),
    "cl3d_pwmlp_prep_weights": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "cl3d_pwmlp_weight_grad": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp]),
    "cl3d_to_point_major_aug": (_i, [_vp, _i, _vp, _i, _i, _i, _f, _vp, _vp]),
    "cl3d_pwmlp_fwd_stats": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cl3d_pwmlp_bwd_scratch_floats": (_sz, [_i, _i, _i, _i, _i]),
    "cl3d_pwmlp_bwd": (_i, [_vp, _i] + [_vp] * 15 + [_i, _i, _i, _i, _i, _f, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "cl3d_pwmlp_bwd_stats": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _vp, _vp]),
    "cl3d_pwmlp_bwd_apply": (_i, [_vp, _i] + [_vp] * 15 + [_i, _i, _i, _i, _i, _f, _i, _i] + [_vp] * 7),
    "cl3d_mhead_save_floats": (_sz, [_i, _i]),
    "cl3d_mhead_fwd_workspace_bytes": (_sz, [_vp, _i, _i]),
    "cl3d_mhead_bwd_workspace_bytes": (_sz, [_vp, _i, _i]),
    "cl3d_mhead_fwd": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _f, _f, _i, _vp, _vp, _vp, _sz, _vp]),
    "cl3d_mhead_bwd": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
}

MHEAD_MAX_HEADS = 32       # CL3D_MHEAD_MAX_HEADS
MHEAD_MAX_PARTS = 64       # CL3D_MHEAD_MAX_PARTS
MHEAD_MAX_CHANNELS = 128   # CL3D_MHEAD_MAX_CHANNELS (padded)


class MHeadDesc(ctypes.Structure):
    """struct cl3d_mhead_desc (passed by host pointer, copied into the kernels' arguments)"""
    _fields_ = [("S", _i), ("C", _i), ("num_parts", _i * MHEAD_MAX_HEADS),
                ("running_mean", _vp * MHEAD_MAX_HEADS), ("running_var", _vp * MHEAD_MAX_HEADS),
                ("num_batches_tracked", _vp * MHEAD_MAX_HEADS), ("grad_logits", _vp * MHEAD_MAX_HEADS)]


class _Profiler:
    """optional per-entry-point CUDA-event timing (bench.py): events are recorded on torch's current stream,
    the stream every kernel of the call is launched on."""

    def __init__(self):
        self.enabled = False
        self.records = []  # (name, start_event, end_event)

    def start(self):
        self.records = []
        self.enabled = True

    def stop(self):
        """-> {entry point: (calls, total_ms)}; synchronises"""
        self.enabled = False
        torch.cuda.synchronize()
        out = {}
        for name, e0, e1 in self.records:
            c, t = out.get(name, (0, 0.0))
            out[name] = (c + 1, t + e0.elapsed_time(e1))
        self.records = []
        return out


profiler = _Profiler()


class _Lib:
    pass


def _wrap(name, fn):
    def call(*args):
        if profiler.enabled and name not in _UNTIMED:
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            rc = fn(*args)
            e1.record()
            profiler.records.append((name, e0, e1))
            return rc
        return fn(*args)
    return call


_UNTIMED = {"cl3d_version", "cl3d_last_error", "cl3d_padded_channels", "cl3d_sm_count", "cl3d_launch_count",
            "cl3d_ball_query_workspace_bytes", "cl3d_ball_query_csr_workspace_bytes", "cl3d_csr_workspace_bytes", "cl3d_grid_subsample_workspace_bytes",
            "cl3d_agg_num_tiles", "cl3d_agg_bwd_num_blocks", "cl3d_agg_num_params", "cl3d_sgemm_workspace_bytes", "cl3d_pwmlp_bwd_scratch_floats",
            "cl3d_mhead_save_floats", "cl3d_mhead_fwd_workspace_bytes", "cl3d_mhead_bwd_workspace_bytes"}


def lib():
    """Load libcl3d.so (built in-tree by closerlook3d_b200/build.py).  Raises ImportError if absent."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ImportError(
                f"{SO_PATH} not found: build it with `python -m closerlook3d_b200.build` "
                "(or __graft_entry__.build()).  There is no CPU / PyTorch fallback.")
        cdll = ctypes.CDLL(SO_PATH)
        L = _Lib()
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(cdll, name)  # AttributeError if the symbol is missing -> loud
            fn.restype = res
            fn.argtypes = args
            setattr(L, name, _wrap(name, fn))
        L._cdll = cdll
        _lib = L
    return _lib


def ptr(t):
    """device pointer of a tensor (None -> NULL)"""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc, what=""):
    if rc != 0:
        msg = lib().cl3d_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"libcl3d {what} failed (code {rc}): {msg}")


def require_cuda(t, name, dtype):
    """the reference's CHECK_CUDA / CHECK_CONTIGUOUS / CHECK_IS_FLOAT / CHECK_IS_INT (utils.h:9-30)"""
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (CPU not supported)")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be a contiguous tensor")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must be a{'n int' if dtype == torch.int32 else ' float'} tensor")
