"""Host wrappers of the tensor-core convolution / linear C ABI (include/monodetr_b200.h, "Tensor-core
convolution / linear family").  Tensors are fp32 CUDA, activations NHWC, weights packed [tap][Cout][Cin].
No fallback: a missing library or a failing launch raises RuntimeError.
"""
import ctypes

import torch

from . import _lib


def _chk(*ts):
    for t in ts:
        if t is None:
            continue
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise RuntimeError("monodetr_b200.tc: contiguous float32 tensors required")


def out_size(n, k, s, p, d=1):
    return (n + 2 * p - d * (k - 1) - 1) // s + 1


def pack_weight(w_oihw, scale=None):
    """(O, I, kh, kw) -> (kh*kw, O, I), optionally multiplied by scale[O] (FrozenBatchNorm fold)."""
    _chk(w_oihw, scale)
    O, I, kh, kw = w_oihw.shape
    out = torch.empty((kh * kw, O, I), dtype=torch.float32, device=w_oihw.device)
    _lib.call("mdb_pack_conv_weight_f32", w_oihw, scale, out, O, I, kh * kw)
    return out


def _int_array(vals):
    return (ctypes.c_int * len(vals))(*vals)


# ---- precision mode 2: weights pre-split into bf16 (hi, lo) pairs ------------------------------------------------------
class SplitW:
    """A GEMM weight in the layout of the bf16x3 kernels (include/monodetr_b200.h, mdb_pack_gemm_weights_bf16x3):
    wf (taps, O, ceil(I/32), 64) bf16 for the forward, wd (taps, I, ceil(O/32), 64) for the data gradient (or None)."""
    __slots__ = ("wf", "wd", "taps", "O", "I")

    def __init__(self, wf, wd, taps, O, I):
        self.wf, self.wd, self.taps, self.O, self.I = wf, wd, taps, O, I

    @property
    def shape(self):
        return (self.taps, self.O, self.I)


def split_weights(weights, scales=None, need_dgrad=True, packed_src=False):
    """[(O, I, kh, kw) or (O, I)] (packed_src: [(taps, O, I)]) -> [SplitW], ONE launch per 64 tensors; all outputs are views
    of one allocation.  scales[j] (O,) folds FrozenBatchNorm (backbone.py:54-64) before the split."""
    n = len(weights)
    if n == 0:
        return []
    scales = list(scales) if scales is not None else [None] * n
    weights = [w if w.is_contiguous() else w.contiguous() for w in weights]
    _chk(*weights, *[s for s in scales if s is not None])
    dims = []
    for w in weights:
        if packed_src:
            taps, O, I = w.shape
        else:
            O, I = w.shape[0], w.shape[1]
            taps = w.numel() // (O * I)
        dims.append((taps, O, I))
    nf = [t * O * ((I + 31) // 32) * 64 for t, O, I in dims]
    nd = [t * I * ((O + 31) // 32) * 64 if need_dgrad else 0 for t, O, I in dims]
    flat = torch.empty((sum(nf) + sum(nd),), dtype=torch.bfloat16, device=weights[0].device)
    outs, wfs, wds, off = [], [], [], 0
    for (t, O, I), a, b in zip(dims, nf, nd):
        wf = flat[off:off + a].view(t, O, (I + 31) // 32, 64)
        off += a
        wd = flat[off:off + b].view(t, I, (O + 31) // 32, 64) if need_dgrad else None
        off += b
        outs.append(SplitW(wf, wd, t, O, I))
        wfs.append(wf)
        wds.append(wd)
    _lib.call("mdb_pack_gemm_weights_bf16x3", n, weights, scales, wfs, wds, _int_array([d[1] for d in dims]),
              _int_array([d[2] for d in dims]), _int_array([d[0] for d in dims]), int(packed_src), launches=(n + 63) // 64)
    return outs


# Weights split once per model forward (MonoDETR.forward enters `prepacked`): lookups are valid only inside the context,
# so a stale split can never outlive the parameters it was made from; backward uses the SplitW objects saved in ctx.
_PREPACK = None


class prepacked:
    def __init__(self, tensors):
        self.tensors = tensors

    def __enter__(self):
        global _PREPACK
        self._prev = _PREPACK
        _PREPACK = {}
        if get_precision() == "bf16x3" and self.tensors:
            with torch.no_grad():
                uniq = {}
                for t in self.tensors:
                    uniq.setdefault((t.data_ptr(), tuple(t.shape)), t)
                keys = list(uniq)
                for k, sw in zip(keys, split_weights([uniq[k].detach() for k in keys])):
                    _PREPACK[k] = sw
        return self

    def __exit__(self, *a):
        global _PREPACK
        _PREPACK = self._prev


def lookup_split(w):
    """SplitW of a weight tensor: the pre-packed one inside a `prepacked` context, else split now (one launch)."""
    if _PREPACK is not None:
        sw = _PREPACK.get((w.data_ptr(), tuple(w.shape)))
        if sw is not None:
            return sw
    return split_weights([w.detach()])[0]


_WORKSPACE = {}


def _ensure_workspace(dev, need):
    """Split-K scratch of the forward kernels: taken from torch's allocator and registered with the library per device;
    grown buffers keep their predecessors alive (a captured CUDA graph may still reference them)."""
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    bufs = _WORKSPACE.setdefault(idx, [])
    if not bufs or bufs[-1].numel() < need:
        bufs.append(torch.empty((max(need, 1 << 20),), dtype=torch.uint8, device=dev))
    _lib.check(_lib.lib().mdb_set_workspace(bufs[-1].data_ptr(), bufs[-1].numel()), "set_workspace")


def pack_weights_multi(weights, scales=None):
    """[(O, I, kh, kw)] -> [(kh*kw, O, I)] in ONE launch per 64 tensors (views of one flat allocation)."""
    n = len(weights)
    if n == 0:
        return []
    scales = list(scales) if scales is not None else [None] * n
    weights = [w.contiguous() for w in weights]
    _chk(*weights, *scales)
    sizes = [w.numel() for w in weights]
    flat = torch.empty((sum(sizes),), dtype=torch.float32, device=weights[0].device)
    outs, off = [], 0
    for w, sz in zip(weights, sizes):
        O, I, kh, kw = w.shape
        outs.append(flat[off:off + sz].view(kh * kw, O, I))
        off += sz
    _lib.call("mdb_pack_conv_weights_multi_f32", n, weights, scales, outs, _int_array([w.shape[0] for w in weights]),
              _int_array([w.shape[1] for w in weights]), _int_array([w.shape[2] * w.shape[3] for w in weights]),
              launches=(n + 63) // 64)
    return outs


def unpack_wgrads_multi(dw_packed_list, khw_list):
    """[(taps, O, I)] -> [(O, I, kh, kw)] in ONE launch per 64 tensors."""
    n = len(dw_packed_list)
    if n == 0:
        return []
    _chk(*dw_packed_list)
    outs = [torch.empty((d.shape[1], d.shape[2], kh, kw), dtype=torch.float32, device=d.device)
            for d, (kh, kw) in zip(dw_packed_list, khw_list)]
    _lib.call("mdb_unpack_conv_wgrads_multi_f32", n, dw_packed_list, outs, _int_array([d.shape[1] for d in dw_packed_list]),
              _int_array([d.shape[2] for d in dw_packed_list]), _int_array([d.shape[0] for d in dw_packed_list]),
              launches=(n + 63) // 64)
    return outs


def unpack_wgrad(dw_packed, kh, kw):
    _chk(dw_packed)
    taps, O, I = dw_packed.shape
    out = torch.empty((O, I, kh, kw), dtype=torch.float32, device=dw_packed.device)
    _lib.call("mdb_unpack_conv_wgrad_f32", dw_packed, out, O, I, taps, 0)
    return out


# ---- grouped 3x3 convolutions (ResNeXt's conv2): band-local weights ------------------------------------------------------
class GroupedW:
    """A grouped 3x3 weight (C, C/groups, 3, 3) in the band-local layout of the grouped entry points (include/monodetr_b200.h,
    "Grouped convolutions"): wf (9, C, 128) for the forward and wd (9, C, 128) for the data gradient (or None), fp32, or
    bf16 (9, C, 4, 64) pre-split (hi, lo) rows in precision mode 'bf16x3'."""
    __slots__ = ("wf", "wd", "C", "groups")

    def __init__(self, wf, wd, C, groups):
        self.wf, self.wd, self.C, self.groups = wf, wd, C, groups

    @property
    def split(self):
        return self.wf.dtype == torch.bfloat16


def pack_grouped_multi(weights, scales=None, groups=None, need_dgrad=True):
    """[(C, C/g, 3, 3)] -> [GroupedW] in the precision mode's format, ONE launch per 64 tensors; all outputs are views of one
    allocation.  scales[j] (C,) folds FrozenBatchNorm (backbone.py:54-64) first; groups[j] = g."""
    n = len(weights)
    if n == 0:
        return []
    scales = list(scales) if scales is not None else [None] * n
    weights = [w if w.is_contiguous() else w.contiguous() for w in weights]
    _chk(*weights, *[s for s in scales if s is not None])
    split = get_precision() == "bf16x3"
    row = 256 if split else 128                         # elements per (tap, channel) row: 4 x [hi 32 | lo 32] bf16, or 128 fp32
    Cs = [w.shape[0] for w in weights]
    sizes = [9 * C * row for C in Cs]
    flat = torch.empty(((2 if need_dgrad else 1) * sum(sizes),), dtype=torch.bfloat16 if split else torch.float32,
                       device=weights[0].device)
    outs, wfs, wds, off = [], [], [], 0
    for C, g, sz in zip(Cs, groups, sizes):
        shape = (9, C, 4, 64) if split else (9, C, 128)
        wf = flat[off:off + sz].view(shape)
        off += sz
        wd = flat[off:off + sz].view(shape) if need_dgrad else None
        off += sz if need_dgrad else 0
        outs.append(GroupedW(wf, wd, C, g))
        wfs.append(wf)
        wds.append(wd)
    _lib.call("mdb_pack_conv_weights_grouped_multi_bf16x3" if split else "mdb_pack_conv_weights_grouped_multi_f32", n, weights,
              scales, wfs, wds, _int_array(Cs), _int_array(list(groups)), launches=(n + 63) // 64)
    return outs


def lookup_grouped(w, groups):
    """GroupedW of a (C, C/g, 3, 3) weight tensor: the one packed earlier in the enclosing `prepacked` context, else packed
    now (one launch)."""
    key = ("grouped", w.data_ptr(), tuple(w.shape), groups, get_precision())
    if _PREPACK is not None and key in _PREPACK:
        return _PREPACK[key]
    gw = pack_grouped_multi([w.detach()], groups=[groups])[0]
    if _PREPACK is not None:
        _PREPACK[key] = gw
    return gw


def unpack_grouped_wgrads_multi(dw_band_list, groups_list):
    """[(9, C, 128)] band-local weight gradients -> [(C, C/g, 3, 3)] in ONE launch per 64 tensors."""
    n = len(dw_band_list)
    if n == 0:
        return []
    _chk(*dw_band_list)
    outs = [torch.empty((d.shape[1], d.shape[1] // g, 3, 3), dtype=torch.float32, device=d.device)
            for d, g in zip(dw_band_list, groups_list)]
    _lib.call("mdb_unpack_conv_wgrads_grouped_multi_f32", n, dw_band_list, outs, _int_array([d.shape[1] for d in dw_band_list]),
              _int_array(list(groups_list)), launches=(n + 63) // 64)
    return outs


def _as_grouped(w, groups):
    if isinstance(w, GroupedW):
        assert w.groups == groups
        return w
    return lookup_grouped(w, groups)


def _grouped_forward(x, w, bias, residual, stride, pad, relu, round_out, dilation, groups):
    w = _as_grouped(w, groups)
    _chk(x, None if w.split else w.wf, bias, residual)
    B, H, W, C = x.shape
    assert C == w.C
    Ho, Wo = out_size(H, 3, stride, pad, dilation), out_size(W, 3, stride, pad, dilation)
    y = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.shape == y.shape
    _lib.call("mdb_conv2d_forward_grouped_bf16x3" if w.split else "mdb_conv2d_forward_grouped_f32", x, w.wf, bias, residual, y,
              B, H, W, C, C, 3, 3, stride, pad, dilation, groups, int(relu) | (int(round_out) << 1))
    return y


def _grouped_dgrad(dy, w, x_shape, residual, relu_mask, stride, pad, round_out, dilation, groups):
    w = _as_grouped(w, groups)
    _chk(dy, None if w.split else w.wd, residual, relu_mask)
    B, H, W, C = x_shape
    assert C == w.C and dy.shape[-1] == C and w.wd is not None
    dx = torch.empty((B, H, W, C), dtype=torch.float32, device=dy.device)
    _lib.call("mdb_conv2d_dgrad_grouped_bf16x3" if w.split else "mdb_conv2d_dgrad_grouped_f32", dy, w.wd, residual, relu_mask, dx,
              B, H, W, C, C, 3, 3, stride, pad, dilation, groups, int(round_out) << 1, launches=stride * stride)
    return dx


def colsum(x2d):
    _chk(x2d)
    M, N = x2d.shape
    out = torch.empty((N,), dtype=torch.float32, device=x2d.device)
    _lib.call("mdb_colsum_f32", x2d, out, M, N, 0)
    return out


def _as_operand(w_packed):
    """fp32 packed weights are split on the fly in bf16x3 mode (tests, rare paths); model code passes SplitW."""
    if isinstance(w_packed, SplitW) or _lib.lib().mdb_get_precision() != 2:
        return w_packed
    return split_weights([w_packed], packed_src=True)[0]


def conv2d_forward(x, w_packed, bias=None, residual=None, kh=1, kw=1, stride=1, pad=0, relu=False, round_out=False, dilation=1,
                   groups=1):
    """w_packed: fp32 (taps, Cout, Cin) or a SplitW (precision mode 'bf16x3').  dilation > 1 (3x3, stride 1) runs the _dilated
    entry points; dilation 1 the plain ones.  groups > 1: a grouped 3x3 through the _grouped entry points, w_packed = a GroupedW
    or the (C, C/groups, 3, 3) weight (packed on the spot, or once per `prepacked` context)."""
    if groups != 1:
        assert kh == kw == 3
        return _grouped_forward(x, w_packed, bias, residual, stride, pad, relu, round_out, dilation, groups)
    w_packed = _as_operand(w_packed)
    split = isinstance(w_packed, SplitW)
    _chk(x, None if split else w_packed, bias, residual)
    B, H, W, Cin = x.shape
    taps, Cout, Cin2 = w_packed.shape
    assert taps == kh * kw and Cin2 == Cin
    Ho, Wo = out_size(H, kh, stride, pad, dilation), out_size(W, kw, stride, pad, dilation)
    y = torch.empty((B, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.shape == y.shape
    flags = int(relu) | (int(round_out) << 1)
    if dilation == 1:
        need = _lib.lib().mdb_conv2d_forward_workspace_bytes(B, H, W, Cin, Cout, kh, kw, stride, pad, flags,
                                                             int(residual is not None), int(split))
    else:
        need = _lib.lib().mdb_conv2d_forward_workspace_bytes_dilated(B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, flags,
                                                                     int(residual is not None), int(split))
    if need < 0:
        _lib.check(int(need), "conv2d_forward_workspace_bytes")
    if need > 0:
        _ensure_workspace(x.device, need)
    if dilation == 1:
        name = "mdb_conv2d_forward_bf16x3" if split else "mdb_conv2d_forward_f32"
    else:
        name = "mdb_conv2d_forward_dilated_bf16x3" if split else "mdb_conv2d_forward_dilated_f32"
    geom = (B, H, W, Cin, Cout, kh, kw, stride, pad) + ((dilation,) if dilation != 1 else ())
    _lib.call(name, x, w_packed.wf if split else w_packed, bias, residual, y, *geom, flags, launches=2 if need > 0 else 1)
    return y


def conv2d_dgrad(dy, w_packed, x_shape, residual=None, relu_mask=None, kh=1, kw=1, stride=1, pad=0, round_out=False, dilation=1,
                 groups=1):
    """w_packed: fp32 (taps, Cout, Cin) or a SplitW with .wd; dy may carry more (zero-padded) channels than a SplitW's O
    as long as both round up to the same number of 32-wide k-blocks.  groups > 1: as conv2d_forward."""
    if groups != 1:
        assert kh == kw == 3
        return _grouped_dgrad(dy, w_packed, x_shape, residual, relu_mask, stride, pad, round_out, dilation, groups)
    w_packed = _as_operand(w_packed)
    split = isinstance(w_packed, SplitW)
    _chk(dy, None if split else w_packed, residual, relu_mask)
    B, H, W, Cin = x_shape
    taps, Cout, Cin2 = w_packed.shape
    assert Cin2 == Cin
    if split:
        assert w_packed.wd is not None and (dy.shape[-1] + 31) // 32 == (Cout + 31) // 32
        Cout = dy.shape[-1]
    else:
        assert dy.shape[-1] == Cout
    dx = torch.empty((B, H, W, Cin), dtype=torch.float32, device=dy.device)
    if dilation == 1:
        name = "mdb_conv2d_dgrad_bf16x3" if split else "mdb_conv2d_dgrad_f32"
    else:
        name = "mdb_conv2d_dgrad_dilated_bf16x3" if split else "mdb_conv2d_dgrad_dilated_f32"
    geom = (B, H, W, Cin, Cout, kh, kw, stride, pad) + ((dilation,) if dilation != 1 else ())
    _lib.call(name, dy, w_packed.wd if split else w_packed, residual, relu_mask, dx, *geom, int(round_out) << 1,
              launches=stride * stride)
    return dx


def conv2d_wgrad(dy, x, rowscale=None, kh=1, kw=1, stride=1, pad=0, with_bias_grad=False, dilation=1, groups=1):
    """dw_packed (taps, Cout, Cin); with_bias_grad=True also returns db (Cout,) = dy summed over pixels, produced by the
    same launch (both live in one allocation so a single memset zero-fills them).  groups > 1 (a grouped 3x3, no bias): the
    band-local (9, C, 128) gradient, for unpack_grouped_wgrads_multi."""
    if groups != 1:
        assert kh == kw == 3 and not with_bias_grad
        _chk(dy, x, rowscale)
        B, H, W, C = x.shape
        dwb = torch.empty((9, C, 128), dtype=torch.float32, device=x.device)
        _lib.call("mdb_conv2d_wgrad_grouped_f32", dy, x, rowscale, dwb, B, H, W, C, dy.shape[-1], 3, 3, stride, pad, dilation,
                  groups, 0, launches=dilation * dilation)
        return dwb
    _chk(dy, x, rowscale)
    B, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    n = kh * kw * Cout * Cin
    buf = torch.empty((n + (Cout if with_bias_grad else 0),), dtype=torch.float32, device=x.device)
    dwp = buf[:n].view(kh * kw, Cout, Cin)
    db = buf[n:] if with_bias_grad else None
    geom = (B, H, W, Cin, Cout, kh, kw, stride, pad) + ((dilation,) if dilation != 1 else ())
    _lib.call("mdb_conv2d_wgrad_bias_f32" if dilation == 1 else "mdb_conv2d_wgrad_bias_dilated_f32", dy, x, rowscale, dwp, db,
              *geom, 0, launches=1 if (not with_bias_grad or get_precision() != "tf32") else 2)
    return (dwp, db) if with_bias_grad else dwp


# ---- linear layers = 1x1 convolution over a 1-row "image" of M pixels ---------------------------------
def set_precision(mode: str):
    """'bf16x3' (default: error-compensated BF16 for forward / dgrad with weights split once per step, and for wgrad with both
    operands split in the kernel),
    'tf32x3' (error-compensated TF32 everywhere, ~fp32 accuracy) or 'tf32' (single pass, operands rounded to nearest)."""
    _lib.check(_lib.lib().mdb_set_precision({"tf32": 0, "tf32x3": 1, "bf16x3": 2}[mode]), "set_precision")


def get_precision() -> str:
    return ("tf32", "tf32x3", "bf16x3")[_lib.lib().mdb_get_precision()]


def round_tf32(x):
    """Round-to-nearest TF32 copy of x (weights of linear layers before they become tensor-core operands);
    identity in the default 'tf32x3' mode, where operands keep all fp32 bits."""
    _chk(x)
    if _lib.lib().mdb_get_precision() != 0:
        return x
    out = torch.empty_like(x)
    _lib.call("mdb_round_tf32_f32", x, out, x.numel())
    return out


def linear_forward(x2d, w, bias=None, residual=None, relu=False, round_out=False):
    """w: fp32 (N, K) or a SplitW (taps == 1)."""
    M, K = x2d.shape
    N = w.O if isinstance(w, SplitW) else w.shape[0]
    y = conv2d_forward(x2d.view(1, 1, M, K), w if isinstance(w, SplitW) else w.view(1, N, K), bias,
                       None if residual is None else residual.view(1, 1, M, N), relu=relu, round_out=round_out)
    return y.view(M, N)


def linear_dgrad(dy2d, w, residual=None, relu_mask=None):
    M, N = dy2d.shape
    K = w.I if isinstance(w, SplitW) else w.shape[1]
    dx = conv2d_dgrad(dy2d.view(1, 1, M, N), w if isinstance(w, SplitW) else w.view(1, N, K), (1, 1, M, K),
                      None if residual is None else residual.view(1, 1, M, K),
                      None if relu_mask is None else relu_mask.view(1, 1, M, K))
    return dx.view(M, K)


def linear_wgrad(dy2d, x2d, with_bias_grad=False):
    M, N = dy2d.shape
    K = x2d.shape[1]
    if with_bias_grad:
        dw, db = conv2d_wgrad(dy2d.view(1, 1, M, N), x2d.view(1, 1, M, K), with_bias_grad=True)
        return dw.view(N, K), db
    return conv2d_wgrad(dy2d.view(1, 1, M, N), x2d.view(1, 1, M, K)).view(N, K)
