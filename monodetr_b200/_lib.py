"""ctypes loader for libmonodetr_b200.so (the C-ABI product library).

There is NO fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmonodetr_b200.so")
_lib = None

c_int, c_void_p, c_float = ctypes.c_int, ctypes.c_void_p, ctypes.c_float

# name -> argtypes (restype is always int unless listed in _RESTYPES)
_PTR = c_void_p
SIGNATURES = {
    "mdb_abi_version": [],
    "mdb_error_string": [c_int],
    "mdb_msda_forward_f32": [_PTR] * 5 + [c_int] * 7 + [_PTR, _PTR],
    "mdb_msda_forward_f64": [_PTR] * 5 + [c_int] * 7 + [_PTR, _PTR],
    "mdb_msda_backward_f32": [_PTR] * 6 + [c_int] * 7 + [_PTR] * 4,
    "mdb_msda_backward_f64": [_PTR] * 6 + [c_int] * 7 + [_PTR] * 4,
    "mdb_msda_fused_forward_f32": [_PTR] * 6 + [c_int] * 8 + [_PTR, _PTR],
    "mdb_msda_fused_backward_f32": [_PTR] * 7 + [c_int] * 8 + [_PTR] * 4,
    "mdb_msda_fused_backward_ref_f32": [_PTR] * 7 + [c_int] * 8 + [_PTR] * 5,
    "mdb_msda_prep_forward_f32": [_PTR] * 4 + [c_int] * 6 + [_PTR] * 3,
    "mdb_msda_prep_backward_f32": [_PTR] * 5 + [c_int] * 6 + [_PTR] * 3,
    "mdb_set_deterministic": [c_int],
    "mdb_get_deterministic": [],
    "mdb_set_precision": [c_int],
    "mdb_get_precision": [],
    "mdb_conv2d_forward_f32": [_PTR] * 5 + [c_int] * 10 + [_PTR],
    "mdb_conv2d_forward_bf16x3": [_PTR] * 5 + [c_int] * 10 + [_PTR],
    "mdb_conv2d_dgrad_bf16x3": [_PTR] * 5 + [c_int] * 10 + [_PTR],
    "mdb_conv2d_forward_workspace_bytes": [c_int] * 12,
    "mdb_conv2d_forward_dilated_f32": [_PTR] * 5 + [c_int] * 11 + [_PTR],
    "mdb_conv2d_forward_dilated_bf16x3": [_PTR] * 5 + [c_int] * 11 + [_PTR],
    "mdb_conv2d_dgrad_dilated_f32": [_PTR] * 5 + [c_int] * 11 + [_PTR],
    "mdb_conv2d_dgrad_dilated_bf16x3": [_PTR] * 5 + [c_int] * 11 + [_PTR],
    "mdb_conv2d_wgrad_bias_dilated_f32": [_PTR] * 5 + [c_int] * 11 + [_PTR],
    "mdb_conv2d_forward_workspace_bytes_dilated": [c_int] * 13,
    "mdb_set_workspace": [_PTR, ctypes.c_ulonglong],
    "mdb_pack_gemm_weights_bf16x3": [c_int] + [_PTR] * 7 + [c_int, _PTR],
    "mdb_conv2d_dgrad_f32": [_PTR] * 5 + [c_int] * 10 + [_PTR],
    "mdb_conv2d_wgrad_f32": [_PTR] * 4 + [c_int] * 10 + [_PTR],
    "mdb_conv2d_wgrad_bias_f32": [_PTR] * 5 + [c_int] * 10 + [_PTR],
    "mdb_pack_conv_weight_f32": [_PTR] * 3 + [c_int] * 3 + [_PTR],
    "mdb_unpack_conv_wgrad_f32": [_PTR] * 2 + [c_int] * 4 + [_PTR],
    "mdb_pack_conv_weights_multi_f32": [c_int] + [_PTR] * 6 + [_PTR],
    "mdb_unpack_conv_wgrads_multi_f32": [c_int] + [_PTR] * 5 + [_PTR],
    "mdb_colsum_f32": [_PTR] * 2 + [ctypes.c_longlong, c_int, c_int, _PTR],
    "mdb_attention_forward_f32": [_PTR] * 6 + [c_int] * 9 + [c_float, _PTR, ctypes.c_ulonglong, _PTR],
    "mdb_attention_backward_f32": [_PTR] * 11 + [c_int] * 12 + [c_float, _PTR, ctypes.c_ulonglong, _PTR],
    "mdb_add_layernorm_forward_f32": [_PTR] * 7 + [ctypes.c_longlong, c_int, c_float, c_float, _PTR, ctypes.c_ulonglong, _PTR],
    "mdb_add_layernorm_backward_f32": [_PTR] * 10 + [ctypes.c_longlong, c_int, c_float, _PTR, ctypes.c_ulonglong, c_int, _PTR],
    "mdb_groupnorm_forward_f32": [_PTR] * 7 + [c_int] * 4 + [c_float, c_int, _PTR],
    "mdb_groupnorm_backward_f32": [_PTR] * 10 + [c_int] * 5 + [_PTR],
    "mdb_relu_backward_f32": [_PTR] * 3 + [ctypes.c_longlong, c_float, _PTR],
    "mdb_dropout_f32": [_PTR] * 2 + [ctypes.c_longlong, c_float, _PTR, ctypes.c_ulonglong, _PTR],
    "mdb_round_tf32_f32": [_PTR] * 2 + [ctypes.c_longlong, _PTR],
    "mdb_stem_conv7x7_bn_relu_f32": [_PTR] * 5 + [c_int] * 3 + [_PTR],
    "mdb_maxpool3x3s2_nhwc_f32": [_PTR] * 2 + [c_int] * 4 + [_PTR],
    "mdb_depth_sample_forward_f32": [_PTR] * 3 + [c_int] * 4 + [_PTR],
    "mdb_depth_sample_backward_f32": [_PTR] * 3 + [c_int] * 4 + [_PTR],
    "mdb_box_refine_forward_f32": [_PTR] * 3 + [ctypes.c_longlong, c_int, _PTR],
    "mdb_box_refine_backward_f32": [_PTR] * 5 + [ctypes.c_longlong, c_int, _PTR],
    "mdb_dab_sine_embed_forward_f32": [_PTR] * 2 + [ctypes.c_longlong, _PTR],
    "mdb_dab_sine_embed_backward_f32": [_PTR] * 3 + [ctypes.c_longlong, _PTR],
    "mdb_dab_query_pos_forward_f32": [_PTR] * 3 + [c_int, ctypes.c_longlong, c_int, c_int, _PTR],
    "mdb_dab_query_pos_backward_f32": [_PTR] * 5 + [c_int, ctypes.c_longlong, c_int, c_int, _PTR],
    "mdb_msda_ref_grad_f32": [_PTR] * 2 + [c_int] * 6 + [_PTR, _PTR],
    "mdb_msda_ref_partials_reduce_f32": [_PTR] + [c_int] * 6 + [_PTR, _PTR],
    "mdb_dab_anchor_forward_f32": [_PTR] * 4 + [c_int, ctypes.c_longlong, _PTR],
    "mdb_dab_anchor_backward_f32": [_PTR] * 4 + [c_int, ctypes.c_longlong, _PTR, _PTR],
    "mdb_pos_learned_forward_f32": [_PTR] * 2 + [c_int] * 2 + [_PTR, _PTR],
    "mdb_pos_learned_backward_f32": [_PTR] + [c_int] * 2 + [_PTR] * 3,
    "mdb_head_depth_forward_f32": [_PTR] * 7 + [c_int] * 4 + [_PTR],
    "mdb_head_depth_backward_f32": [_PTR] * 10 + [c_int] * 4 + [_PTR],
    "mdb_depth_tail_forward_f32": [_PTR] * 5 + [ctypes.c_longlong, c_int, c_int, c_int, c_float, _PTR],
    "mdb_depth_tail_backward_f32": [_PTR] * 7 + [ctypes.c_longlong, c_int, c_int, c_int, c_float, _PTR],
    "mdb_upsample_bilinear_nhwc_forward_f32": [_PTR] * 2 + [c_int] * 6 + [_PTR],
    "mdb_upsample_bilinear_nhwc_backward_f32": [_PTR] * 2 + [c_int] * 6 + [_PTR],
    "mdb_mean3_f32": [_PTR] * 4 + [ctypes.c_longlong, _PTR],
    "mdb_scale_f32": [_PTR] * 2 + [ctypes.c_longlong, c_float, _PTR],
    "mdb_sum_mean_squares_forward_f32": [c_int, _PTR, _PTR, _PTR, _PTR],
    "mdb_sum_mean_squares_backward_f32": [c_int, _PTR, _PTR, _PTR, _PTR, _PTR],
    "mdb_adamw_step_f32": [_PTR] * 4 + [ctypes.c_longlong] * 2 + [c_float] * 7 + [_PTR, _PTR],
    "mdb_adamw_advance": [_PTR, _PTR],
    "mdb_trainlog_push_f32": [_PTR, _PTR, c_int, _PTR, c_int, _PTR, _PTR],
    "mdb_criterion_prepare": [_PTR, c_int, c_int, _PTR, _PTR, _PTR, _PTR],
    "mdb_criterion_match_f32": [c_int] + [_PTR] * 6 + [c_int] * 5 + [c_float] * 4 + [_PTR] * 3,
    "mdb_criterion_depth_map_f32": [_PTR] + [ctypes.c_longlong] * 3 + [_PTR] * 4 + [c_int] * 5 + [c_float] * 7 + [_PTR] * 4,
    "mdb_criterion_losses_f32": [c_int] + [_PTR] * 17 + [c_int] * 6 + [c_float] * 2 + [_PTR, _PTR, _PTR],
    "mdb_criterion_losses_backward_f32": [c_int] + [_PTR] * 16 + [c_int] * 5 + [c_float] * 2 + [_PTR] * 8,
    "mdb_warp_affine_normalize_u8": [_PTR] * 5 + [c_int] * 3 + [_PTR] * 4,
    "mdb_photometric_distort_u8": [_PTR] * 6 + [c_int, _PTR],
    "mdb_kitti_encode_targets": [_PTR] * 3 + [c_int, _PTR, c_int] + [_PTR] * 14,
    "mdb_extract_dets_f32": [_PTR] * 5 + [c_int] * 4 + [_PTR, _PTR],
    "mdb_decode_dets_f32": [_PTR] * 4 + [c_int] * 3 + [c_float, _PTR, _PTR, _PTR],
    "mdb_kitti_overlaps": [_PTR] * 3 + [c_int] * 3 + [ctypes.c_longlong] + [_PTR] * 4,
    "mdb_kitti_eval_workspace_bytes": [c_int] * 5,
    "mdb_kitti_eval": [_PTR] * 3 + [c_int] * 5 + [ctypes.c_longlong] + [_PTR] * 7 + [c_int] * 2 + [_PTR, ctypes.c_longlong]
                      + [_PTR, _PTR],
    "mdb_kitti_eval_distance": [_PTR] * 3 + [c_int] * 5 + [ctypes.c_longlong] + [_PTR] * 7 + [c_int] * 2
                               + [_PTR, ctypes.c_longlong] + [_PTR, _PTR],
    "mdb_kitti_collect_dets_f32": [_PTR] * 3 + [c_int] * 3 + [_PTR, c_int] + [_PTR] * 4,
    "mdb_kitti_compact_dets": [_PTR] * 3 + [c_int] * 2 + [_PTR] * 3,
}
_RESTYPES = {"mdb_error_string": ctypes.c_char_p, "mdb_conv2d_forward_workspace_bytes": ctypes.c_longlong,
             "mdb_conv2d_forward_workspace_bytes_dilated": ctypes.c_longlong,
             "mdb_kitti_eval_workspace_bytes": ctypes.c_longlong}


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} not found: build it with `python -m monodetr_b200.build` "
                "(there is no CPU / PyTorch fallback for the hot path)")
        L = ctypes.CDLL(LIB_PATH)
        for name, argtypes in SIGNATURES.items():
            fn = getattr(L, name)  # AttributeError if the symbol is missing
            fn.argtypes = argtypes
            fn.restype = _RESTYPES.get(name, c_int)
        _lib = L
        # MDB_DETERMINISTIC=1: the process starts in reproducible mode (mdb_set_deterministic), so that a program that never calls
        # set_deterministic -- bench.py, a training script -- can be run twice and compared bit for bit; set_deterministic overrides it
        if os.environ.get("MDB_DETERMINISTIC") == "1":
            check(L.mdb_set_deterministic(1), "mdb_set_deterministic")
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().mdb_error_string(rc)
        raise RuntimeError(f"monodetr_b200 {what} failed (code {rc}): {msg.decode() if msg else '?'}")


# number of kernels of THIS library launched so far in this process (bench.py reports the per-step delta)
_launches = 0


def _device_ptr(t, name):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError(f"monodetr_b200 {name}: CUDA tensors required (there is no CPU path)")
    return t.data_ptr()


def call(name: str, *args, launches: int = 1):
    """Run the entry point `name` on the current CUDA stream (appended as the last argument) and count `launches` kernels.

    A tensor argument becomes its device pointer, None becomes NULL and a list / tuple of tensors (entries may be None)
    becomes a host array of device pointers; anything else is passed as it is.  A tensor that is not on the GPU raises
    RuntimeError before anything is launched; a non-zero status raises RuntimeError naming the entry point."""
    conv = []
    for a in args:
        if isinstance(a, torch.Tensor) or a is None:
            a = _device_ptr(a, name)
        elif isinstance(a, (list, tuple)):
            a = (c_void_p * len(a))(*[_device_ptr(t, name) for t in a])
        conv.append(a)
    check(getattr(lib(), name)(*conv, torch.cuda.current_stream().cuda_stream), name)
    count(launches)


def deterministic() -> bool:
    """Whether the library is in reproducible mode (mdb_set_deterministic); some entry points then launch a different number of
    kernels."""
    return bool(lib().mdb_get_deterministic())


def count(n: int = 1):
    global _launches
    _launches += n


def launch_count() -> int:
    return _launches
