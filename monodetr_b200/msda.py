"""Host side of the MSDeformAttn extension boundary (B1 in SURVEY.md 8b).

Mirrors the reference's pybind module `MultiScaleDeformableAttention`
(lib/models/monodetr/ops/src/vision.cpp:13-16) and autograd glue
(lib/models/monodetr/ops/functions/ms_deform_attn_func.py:21-38) on top of the C ABI in
include/monodetr_b200.h.  Same argument order, same contiguity / device checks as
ms_deform_attn_cuda.cu:28-38, same error behaviour for CPU tensors (ms_deform_attn.h:38,60).
"""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib


PROBE = None    # set to a list by bench.py to collect (start_event, stop_event, B, Lq) per forward launch


def _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, extra=()):
    tensors = [("value", value), ("spatial_shapes", spatial_shapes), ("level_start_index", level_start_index),
               ("sampling_loc", sampling_loc), ("attn_weight", attn_weight), *extra]
    for name, t in tensors:
        if not t.is_cuda:
            raise RuntimeError("Not implemented on the CPU" if name == "value" else f"{name} must be a CUDA tensor")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} tensor has to be contiguous")
    if value.dtype not in (torch.float32, torch.float64):
        raise RuntimeError(f"ms_deform_attn: unsupported dtype {value.dtype}")
    for name, t in (("sampling_loc", sampling_loc), ("attn_weight", attn_weight), *extra):
        if t.dtype != value.dtype:
            raise RuntimeError(f"{name} dtype {t.dtype} != value dtype {value.dtype}")
    if spatial_shapes.dtype != torch.int64 or level_start_index.dtype != torch.int64:
        raise RuntimeError("spatial_shapes / level_start_index must be int64")
    if value.dim() != 4 or sampling_loc.dim() != 6 or attn_weight.dim() != 5:
        raise RuntimeError("ms_deform_attn: bad tensor rank")
    B, S, M, D = value.shape
    _, Lq, M2, L, P, two = sampling_loc.shape
    if sampling_loc.shape[0] != B or M2 != M or two != 2 or tuple(attn_weight.shape) != (B, Lq, M, L, P):
        raise RuntimeError("ms_deform_attn: inconsistent shapes")
    if spatial_shapes.shape != (L, 2) or level_start_index.shape != (L,):
        raise RuntimeError("ms_deform_attn: spatial_shapes must be (L,2) and level_start_index (L,)")
    if max(B * S * M * D, B * Lq * M * D) >= 2 ** 31:
        raise RuntimeError("ms_deform_attn: tensor too large for 32-bit unit indexing")
    return B, S, M, D, L, Lq, P


def ms_deform_attn_forward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, im2col_step):
    """Same contract as the reference pybind function (vision.cpp:14).  `im2col_step` is accepted and ignored."""
    B, S, M, D, L, Lq, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight)
    out = torch.empty((B, Lq, M * D), dtype=value.dtype, device=value.device)
    name = "mdb_msda_forward_f32" if value.dtype == torch.float32 else "mdb_msda_forward_f64"
    with torch.cuda.device(value.device):
        if PROBE is not None:       # bench.py: CUDA events tight around the launch (nothing else between them)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        _lib.call(name, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, B, S, M, D, L, Lq, P, out)
        if PROBE is not None:
            e1.record()
            PROBE.append((e0, e1, B, Lq))
    return out


def ms_deform_attn_backward(value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output,
                            im2col_step):
    """Same contract as the reference pybind function (vision.cpp:15): returns [grad_value, grad_loc, grad_attn]."""
    B, S, M, D, L, Lq, P = _check_inputs(value, spatial_shapes, level_start_index, sampling_loc, attn_weight,
                                         extra=(("grad_output", grad_output),))
    if grad_output.numel() != B * Lq * M * D:
        raise RuntimeError("ms_deform_attn: grad_output has the wrong size")
    grad_value = torch.empty_like(value)          # zero-filled inside the C call
    grad_loc = torch.empty_like(sampling_loc)
    grad_attn = torch.empty_like(attn_weight)
    name = "mdb_msda_backward_f32" if value.dtype == torch.float32 else "mdb_msda_backward_f64"
    with torch.cuda.device(value.device):
        _lib.call(name, value, spatial_shapes, level_start_index, sampling_loc, attn_weight, grad_output, B, S, M, D, L, Lq, P,
                  grad_value, grad_loc, grad_attn)
    return [grad_value, grad_loc, grad_attn]


class MSDeformAttnFunction(Function):
    """Drop-in for the reference class of the same name (ms_deform_attn_func.py:21-38)."""

    @staticmethod
    def forward(ctx, value, value_spatial_shapes, value_level_start_index, sampling_locations, attention_weights,
                im2col_step):
        ctx.im2col_step = im2col_step
        value = value.contiguous()
        sampling_locations = sampling_locations.contiguous()
        attention_weights = attention_weights.contiguous()
        output = ms_deform_attn_forward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                                        attention_weights, im2col_step)
        ctx.save_for_backward(value, value_spatial_shapes, value_level_start_index, sampling_locations,
                              attention_weights)
        return output

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        value, shapes, lsi, loc, attn = ctx.saved_tensors
        gv, gl, ga = ms_deform_attn_backward(value, shapes, lsi, loc, attn, grad_output.contiguous(), ctx.im2col_step)
        return gv, None, None, gl, ga, None
