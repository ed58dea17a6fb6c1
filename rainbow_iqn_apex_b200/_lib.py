"""ctypes binding of libriqn_b200.so (the C-ABI declared in include/riqn_b200.h).

There is deliberately NO fallback: if the CUDA library is missing or a call fails, this raises.
"""
import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libriqn_b200.so")

c_f32p = C.c_void_p
_P = C.c_void_p


class ConvGeom(C.Structure):
    _fields_ = [("B", C.c_int), ("Cin", C.c_int), ("H", C.c_int), ("W", C.c_int), ("Cout", C.c_int),
                ("KH", C.c_int), ("KW", C.c_int), ("stride", C.c_int), ("pad", C.c_int), ("OH", C.c_int),
                ("OW", C.c_int), ("in_bstride", C.c_long)]


class NoisyLayer(C.Structure):
    """riqn_noisy_layer (include/riqn_b200.h)"""
    _fields_ = [("out_features", C.c_int), ("in_features", C.c_int), ("weight_mu", _P), ("weight_sigma", _P),
                ("weight_epsilon", _P), ("bias_mu", _P), ("bias_sigma", _P), ("bias_epsilon", _P), ("eps_in", _P),
                ("eps_out", _P), ("w_eff", _P), ("b_eff", _P), ("stream_in", C.c_ulonglong),
                ("stream_out", C.c_ulonglong), ("w_hi", _P), ("w_lo", _P), ("w_fp16", C.c_int)]


class ResetSegment(C.Structure):
    """riqn_reset_segment (include/riqn_b200.h)"""
    _fields_ = [("begin", C.c_longlong), ("end", C.c_longlong), ("kind", C.c_int), ("value", C.c_float),
                ("alpha", C.c_float)]


class SplitJob(C.Structure):
    """riqn_split_job (include/riqn_b200.h)"""
    _fields_ = [("src", _P), ("perm", _P), ("rows", C.c_int), ("cols", C.c_int), ("div", C.c_float), ("hi", _P),
                ("lo", _P), ("hi_t", _P)]


# name -> argtypes (everything returns int).  Must list every symbol of include/riqn_b200.h.
SIGNATURES = {
    "riqn_version": [],
    "riqn_device_ok": [],
    "riqn_launch_count": [],
    "riqn_conv_fwd": [C.POINTER(ConvGeom), _P, C.c_int, _P, _P, _P, _P, _P],
    "riqn_conv_bwd": [C.POINTER(ConvGeom), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "riqn_im2col_f32": [C.POINTER(ConvGeom), _P, C.c_int, _P, _P],
    "riqn_conv_fwd_tc": [C.POINTER(ConvGeom), _P, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P],
    "riqn_conv_bwd_tc": [C.POINTER(ConvGeom), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_float, _P],
    "riqn_s2d_u8": [C.POINTER(ConvGeom), _P, _P, _P],
    "riqn_conv_fwd_strip": [C.POINTER(ConvGeom), _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, C.c_int, _P],
    "riqn_conv_bwd_strip": [C.POINTER(ConvGeom), _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_float, _P],
    "riqn_split_bf16_scaled": [C.c_long, C.c_int, _P, C.c_float, _P, _P, _P],
    "riqn_fill_uniform": [C.c_long, C.c_ulonglong, C.c_ulonglong, _P, _P, _P],
    "riqn_fill_tau_distorted": [C.c_long, C.c_ulonglong, C.c_ulonglong, C.c_int, C.c_float, _P, _P, _P],
    "riqn_noisy_sample": [C.c_long, C.c_ulonglong, C.c_ulonglong, _P, _P, _P],
    "riqn_fill_shifts": [C.c_long, C.c_int, C.c_ulonglong, C.c_ulonglong, _P, _P, _P],
    "riqn_random_shift": [C.c_int] * 4 + [_P, C.c_long, _P, C.c_long, C.c_int, _P, _P, _P],
    "riqn_noisy_compose": [C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, C.c_int, _P],
    "riqn_noisy_reset_net": [C.c_int, C.POINTER(NoisyLayer), C.c_ulonglong, C.c_int, C.c_int, _P, _P],
    "riqn_noisy_linear_fwd": [C.c_long, C.c_int, C.c_int, _P, _P, _P, _P, _P],
    "riqn_noisy_linear_dgrad": [C.c_long, C.c_int, C.c_int, _P, _P, _P, _P],
    "riqn_noisy_linear_wgrad": [C.c_long, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "riqn_noisy_bias_grad": [C.c_long, C.c_int, _P, _P, _P, _P, _P, _P],
    "riqn_quantile_embed_fwd": [C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P],
    "riqn_quantile_embed_fwd_tc": [C.c_int, C.c_int, C.c_int, C.c_int] + [_P] * 13 + [C.c_int, _P],
    "riqn_quantile_embed_bwd_tc": [C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_int, _P, _P, _P, _P, _P],
    "riqn_quantile_embed_bwd": [C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P],
    "riqn_dueling_fwd": [C.c_long, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P],
    "riqn_dueling_bwd": [C.c_long, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, C.c_float, _P, _P, _P, _P, _P],
    "riqn_dueling_bwd_bf16": [C.c_long, C.c_int, C.c_int, C.c_int] + [_P] * 5 + [C.c_float] + [_P] * 7,
    "riqn_dueling_bwd_dense": [C.c_long, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P],
    "riqn_dueling_bwd_dense_bf16": [C.c_long, C.c_int, C.c_int, C.c_int] + [_P] * 10,
    "riqn_z_wgrad": [C.c_long, C.c_int, C.c_int] + [_P] * 17,
    "riqn_z_wgrad_tc": [C.c_long, C.c_int, C.c_int] + [_P] * 18,
    "riqn_argmax_mean": [C.c_int, C.c_int, C.c_int, _P, _P, _P],
    "riqn_iqn_loss_fwd_bwd": [C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, C.c_float, C.c_float,
                              _P, _P, _P, _P, _P],
    "riqn_miqn_loss_fwd_bwd": [C.c_int] * 4 + [_P] * 6 + [C.c_float] * 5 + [_P] * 6,
    "riqn_cql_loss_fwd_bwd": [C.c_int] * 4 + [_P] * 7 + [C.c_float] * 3 + [_P] * 8,
    "riqn_cql_loss_fwd_bwd_h": [C.c_int] * 4 + [_P] * 7 + [C.c_float] * 4 + [_P] * 8,
    "riqn_cql_dense_grad": [C.c_int] * 3 + [_P] * 4 + [C.c_float] * 2 + [_P, _P],
    "riqn_dqfd_loss_fwd_bwd": [C.c_int] * 4 + [_P] * 8 + [C.c_float] * 4 + [_P] * 8,
    "riqn_dqfd_loss_fwd_bwd_h": [C.c_int] * 4 + [_P] * 8 + [C.c_float] * 5 + [_P] * 8,
    "riqn_dqfd_dense_grad": [C.c_int] * 3 + [_P] * 5 + [C.c_float] * 2 + [_P, _P],
    "riqn_fqf_fractions": [C.c_int, C.c_int] + [_P] * 6,
    "riqn_fqf_fraction_bwd": [C.c_int] * 3 + [_P] * 6 + [C.c_float] * 2 + [_P] * 3,
    "riqn_fqf_fraction_wgrad": [C.c_int] * 3 + [_P] * 5,
    "riqn_linear_wgrad": [C.c_int] * 3 + [_P] * 5,
    "riqn_curl_infonce_fwd_bwd": [C.c_int, C.c_int, _P, _P, _P, C.c_float] + [_P] * 5,
    "riqn_layernorm_fwd": [C.c_long, C.c_int, _P, _P, C.c_int, _P, _P],
    "riqn_layernorm_bwd": [C.c_long, C.c_int, _P, _P, _P, C.c_int, _P, _P],
    "riqn_colsum_add": [C.c_long, C.c_int, _P, _P, _P],
    "riqn_ema_f32": [C.c_long, _P, _P, C.c_float, _P],
    "riqn_add_f32": [C.c_long, _P, _P, _P, _P],
    "riqn_spr_pack": [C.c_int, C.c_int, _P, _P, C.c_int, C.c_int, _P, _P, _P],
    "riqn_spr_unpack_grad": [C.c_int, C.c_int, _P, _P, _P, _P],
    "riqn_spr_weight_images": [C.c_int] * 3 + [_P] * 5,
    "riqn_spr_weight_grad_add": [C.c_int] * 3 + [_P] * 3,
    "riqn_spr_cosine_fwd_bwd": [C.c_int] * 3 + [_P] * 3 + [C.c_float, _P, _P, _P],
    "riqn_sequence_gather": [C.c_int] * 4 + [_P] * 10,
    "riqn_arena_reset": [C.c_long, _P, _P, _P, C.c_int, C.POINTER(ResetSegment), C.c_ulonglong, C.c_ulonglong, _P],
    "riqn_argmax_weighted": [C.c_int] * 3 + [_P] * 4,
    "riqn_c51_head_fwd":[C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P],
    "riqn_c51_loss_fwd_bwd": [C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, C.c_float, C.c_float, C.c_float,
                              C.c_float, _P, _P, _P, _P],
    "riqn_value_rescale": [C.c_long, _P, C.c_float, C.c_int, _P, _P],
    "riqn_iqn_loss_fwd_bwd_h": [C.c_int] * 4 + [_P] * 7 + [C.c_float] * 3 + [_P] * 5,
    "riqn_argmax_expected_h": [C.c_int] * 3 + [_P, _P, C.c_float, _P, _P, _P],
    "riqn_c51_loss_fwd_bwd_h": [C.c_int] * 3 + [_P] * 7 + [C.c_float] * 5 + [_P] * 4,
    "riqn_c51_head_bwd": [C.c_int, C.c_int, C.c_int, _P, _P, C.c_float, _P, _P, _P, _P],
    "riqn_c51_head_bwd_dense": [C.c_int, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P, _P],
    "riqn_qr_head_fwd": [C.c_int] * 3 + [_P] * 4,
    "riqn_qr_head_bwd": [C.c_int] * 3 + [_P, _P, C.c_float, _P, _P, _P, _P],
    "riqn_qr_head_bwd_dense": [C.c_int] * 3 + [_P] * 4,
    "riqn_mmd_loss_fwd_bwd": [C.c_int] * 3 + [_P] * 6 + [C.c_float, C.c_int, _P] + [_P] * 5,
    "riqn_mmd_loss_fwd_bwd_h": [C.c_int] * 3 + [_P] * 6 + [C.c_float, C.c_int, _P, C.c_float] + [_P] * 5,
    "riqn_hl_gauss_loss_fwd_bwd": [C.c_int] * 3 + [_P] * 7 + [C.c_float] * 4 + [_P] * 5,
    "riqn_hl_gauss_loss_fwd_bwd_h": [C.c_int] * 3 + [_P] * 7 + [C.c_float] * 5 + [_P] * 5,
    "riqn_zero_f32": [_P, C.c_long, _P],
    "riqn_relu_mask": [C.c_long, _P, _P, _P],
    "riqn_linear_fwd_ld": [C.c_long, C.c_int, C.c_int, _P, C.c_long, _P, _P, _P, C.c_long, C.c_int, _P],
    "riqn_linear_dgrad_ld": [C.c_long, C.c_int, C.c_int, _P, C.c_long, _P, _P, C.c_long, _P],
    "riqn_noisy_wgrad_ld": [C.c_long, C.c_int, C.c_int, _P, C.c_long, _P, C.c_long, _P, _P, _P, _P],
    "riqn_adam_step": [C.c_long, _P, _P, _P, _P, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, _P, _P],
    "riqn_adamw_step": [C.c_long, _P, _P, _P, _P, C.c_int] + [C.c_float] * 6 + [_P, _P],
    "riqn_sumtree_stratified": [C.c_int, C.c_ulonglong, C.c_ulonglong, _P, _P, _P, _P],
    "riqn_sumtree_sample": [C.c_int, C.c_long, C.c_int, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P],
    "riqn_sumtree_is_weights": [C.c_int, _P, _P, C.c_double, C.c_double, _P, _P, _P, _P, _P],
    "riqn_sumtree_update": [C.c_int, C.c_long, _P, _P, _P, C.c_float, C.c_int, _P, _P, _P, _P],
    "riqn_sumtree_update_demo": [C.c_int, C.c_long, _P, _P, _P, C.c_float, C.c_int, _P, _P, _P, C.c_longlong, C.c_float,
                                 _P],
    "riqn_replay_append": [C.c_int, C.c_int, C.c_int, C.c_int] + [_P] * 11,
    "riqn_frame_gather": [C.c_int, C.c_int, C.c_int, C.c_int] + [_P] * 12,
    "riqn_split_bf16_multi": [C.c_int, C.POINTER(SplitJob), _P],
    "riqn_split_bf16": [C.c_long, C.c_int, _P, _P, _P, _P, _P, C.c_int, _P],
    "riqn_gemm_bf16_tc": [C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P, C.c_long, C.c_int, _P, _P, _P, C.c_int, _P, _P, C.c_int, _P],
    "riqn_gemm_bf16_tc_mn": [C.c_int, C.c_int, C.c_int, _P, _P, C.c_int, _P, C.c_long, C.c_int, _P, _P, C.c_float, C.c_int, _P, C.c_int, _P],
    "riqn_gemm_f32": [C.c_int, C.c_int, C.c_int, _P, C.c_long, C.c_long, _P, C.c_long, C.c_long, _P, C.c_long, _P],
}

_lib = None


class RiqnError(RuntimeError):
    pass


def load():
    """dlopen the in-tree library and attach prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RiqnError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                        "(the product has no CPU or PyTorch fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.argtypes = argtypes
        fn.restype = C.c_longlong if name == "riqn_launch_count" else C.c_int
    if lib.riqn_version() != 1:
        raise RiqnError("ABI version mismatch between _lib.py and libriqn_b200.so")
    _lib = lib
    return lib


def stream():
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


_timers = None  # {entry point name: [(start_event, end_event), ...]} while bench.py profiles a region


def time_entry_points(names):
    """Record CUDA events (on the launching stream) around every call of the named entry points."""
    global _timers
    _timers = {n: [] for n in names} if names else None
    return _timers


def call(name, *args):
    """Invoke a C-ABI entry point on torch's current stream; raise on a non-zero return."""
    lib = load()
    if _timers is not None and name in _timers:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args, stream())
        e1.record()
        _timers[name].append((e0, e1, args))
    else:
        rc = getattr(lib, name)(*args, stream())
    if rc != 0:
        raise RiqnError(f"{name} failed with cudaError {rc}")


def launch_count():
    return int(load().riqn_launch_count())


def require_device():
    """Fail loudly unless a CUDA device of compute capability 9.x is current."""
    if not torch.cuda.is_available():
        raise RiqnError("rainbow_iqn_apex_b200 needs a CUDA device (H100, sm_90a); there is no CPU path")
    lib = load()
    ok = lib.riqn_device_ok()
    if ok != 1:
        raise RiqnError(f"libriqn_b200.so holds sm_90a code only; riqn_device_ok() returned {ok}")
