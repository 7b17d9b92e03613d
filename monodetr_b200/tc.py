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


def out_size(n, k, s, p):
    return (n + 2 * p - k) // s + 1


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


def conv2d_forward(x, w_packed, bias=None, residual=None, kh=1, kw=1, stride=1, pad=0, relu=False, round_out=False):
    """w_packed: fp32 (taps, Cout, Cin) or a SplitW (precision mode 'bf16x3')."""
    w_packed = _as_operand(w_packed)
    split = isinstance(w_packed, SplitW)
    _chk(x, None if split else w_packed, bias, residual)
    B, H, W, Cin = x.shape
    taps, Cout, Cin2 = w_packed.shape
    assert taps == kh * kw and Cin2 == Cin
    Ho, Wo = out_size(H, kh, stride, pad), out_size(W, kw, stride, pad)
    y = torch.empty((B, Ho, Wo, Cout), dtype=torch.float32, device=x.device)
    if residual is not None:
        assert residual.shape == y.shape
    flags = int(relu) | (int(round_out) << 1)
    need = _lib.lib().mdb_conv2d_forward_workspace_bytes(B, H, W, Cin, Cout, kh, kw, stride, pad, flags, int(residual is not None),
                                                         int(split))
    if need < 0:
        _lib.check(int(need), "conv2d_forward_workspace_bytes")
    if need > 0:
        _ensure_workspace(x.device, need)
    _lib.call("mdb_conv2d_forward_bf16x3" if split else "mdb_conv2d_forward_f32", x, w_packed.wf if split else w_packed, bias,
              residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, launches=2 if need > 0 else 1)
    return y


def conv2d_dgrad(dy, w_packed, x_shape, residual=None, relu_mask=None, kh=1, kw=1, stride=1, pad=0, round_out=False):
    """w_packed: fp32 (taps, Cout, Cin) or a SplitW with .wd; dy may carry more (zero-padded) channels than a SplitW's O
    as long as both round up to the same number of 32-wide k-blocks."""
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
    _lib.call("mdb_conv2d_dgrad_bf16x3" if split else "mdb_conv2d_dgrad_f32", dy, w_packed.wd if split else w_packed, residual,
              relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, int(round_out) << 1, launches=stride * stride)
    return dx


def conv2d_wgrad(dy, x, rowscale=None, kh=1, kw=1, stride=1, pad=0, with_bias_grad=False):
    """dw_packed (taps, Cout, Cin); with_bias_grad=True also returns db (Cout,) = dy summed over pixels, produced by the
    same launch (both live in one allocation so a single memset zero-fills them)."""
    _chk(dy, x, rowscale)
    B, H, W, Cin = x.shape
    Cout = dy.shape[-1]
    n = kh * kw * Cout * Cin
    buf = torch.empty((n + (Cout if with_bias_grad else 0),), dtype=torch.float32, device=x.device)
    dwp = buf[:n].view(kh * kw, Cout, Cin)
    db = buf[n:] if with_bias_grad else None
    _lib.call("mdb_conv2d_wgrad_bias_f32", dy, x, rowscale, dwp, db, B, H, W, Cin, Cout, kh, kw, stride, pad, 0,
              launches=1 if (not with_bias_grad or get_precision() != "tf32") else 2)
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
