"""Autograd glue over the C-ABI kernels (forward AND backward run on the sm_90a library; there is no
PyTorch/CPU fallback).  Activations are channels-last: images NHWC, token tensors (B, L, C).

Dropout sites are identified by an integer `site`; masks are regenerated in backward from the device seed
(kernels.seed_tensor), so nothing but the seed is kept.
"""
import os

import torch
import torch.nn.functional as F
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib, kernels as K, tc
from .msda import MSDeformAttnFunction


def _pad4(n):
    return (n + 3) // 4 * 4


# ---- fork/join onto a side stream for small, mutually independent launches --------------------------------------
# The data-gradient and the weight-gradient GEMM of a small linear layer (decoder / heads: 4400 rows) occupy 30-70 of the
# 132 SMs for ~10 us each and do not depend on each other: the weight gradient runs on a side stream while the main
# stream computes the data gradient, and the main stream waits for it before the function returns (so autograd and the
# caching allocator only ever see completed results; under CUDA-graph capture this is the ordinary fork/join pattern).
_SIDE_STREAMS = {}
_SIDE_MAX_ROWS = 0 if os.environ.get("MDB_NO_SIDE_STREAM") else 8192


class _Fork:
    def __init__(self):
        dev = torch.cuda.current_device()
        self.main = torch.cuda.current_stream()
        self.side = _SIDE_STREAMS.get(dev)
        if self.side is None:
            self.side = _SIDE_STREAMS[dev] = torch.cuda.Stream(dev)
        self.side.wait_stream(self.main)

    def join(self, *tensors):
        self.main.wait_stream(self.side)
        for t in tensors:                     # allocated on the side stream, consumed (and freed) on the main stream
            if t is not None:
                t.record_stream(self.main)


_BRANCH_STREAMS = {}
_BRANCHES = not os.environ.get("MDB_NO_BRANCH_STREAMS")
# level 1: depth predictor beside the encoder, the three levels' prediction heads beside each other; level 2 (default): also the
# decoder's independent chains (k / v projections, box / size heads off the critical path, hoisted key-value and value projections)
BRANCH_LEVEL = 0 if not _BRANCHES else int(os.environ.get("MDB_BRANCH_LEVEL", "2"))


class Branch:
    """Run an independent part of the forward graph on its own stream (`with Branch(i): ...`, then `.join(*outputs)` on the
    consumer side).  Autograd replays every node's backward on the stream its forward ran on, so the backward of the branch
    overlaps too; inside a CUDA-graph capture this is the ordinary fork / join.  `MDB_NO_BRANCH_STREAMS=1` makes it a no-op."""

    def __init__(self, index, level=1):
        self.main = torch.cuda.current_stream()
        self.side = None
        if BRANCH_LEVEL >= level:
            key = (torch.cuda.current_device(), index)
            self.side = _BRANCH_STREAMS.get(key)
            if self.side is None:
                self.side = _BRANCH_STREAMS[key] = torch.cuda.Stream(key[0])
        self._ctx = None

    def __enter__(self):
        if self.side is not None:
            self.side.wait_stream(self.main)
            self._ctx = torch.cuda.stream(self.side)
            self._ctx.__enter__()
        return self

    def __exit__(self, *exc):
        if self._ctx is not None:
            self._ctx.__exit__(*exc)
        return False

    def join(self, *tensors):
        if self.side is not None:
            self.main.wait_stream(self.side)
            for t in tensors:                  # allocated on the branch stream, consumed (and possibly freed) on the main one
                if t is not None:
                    t.record_stream(self.main)


# ---- small raw wrappers ---------------------------------------------------------------------------------
def relu_backward(dy, y, scale=1.0):
    dy = dy.contiguous()
    out = torch.empty_like(dy)
    _lib.call("mdb_relu_backward_f32", dy, y, out, dy.numel(), float(scale))
    return out


def dropout_raw(x, p, site, seed=None):
    x = x.contiguous()
    out = torch.empty_like(x)
    seed = seed if seed is not None else K.seed_tensor(x.device)
    _lib.call("mdb_dropout_f32", x, out, x.numel(), float(p), seed, site)
    return out


class _Dropout(Function):
    @staticmethod
    def forward(ctx, x, p, site):
        ctx.p, ctx.site = p, site
        ctx.seed = K.seed_tensor(x.device)          # this forward's snapshot: backward regenerates the SAME mask
        return dropout_raw(x, p, site, ctx.seed)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        return dropout_raw(dy, ctx.p, ctx.site, ctx.seed), None, None


def dropout(x, p, training, site):
    if not training or p <= 0.0:
        return x
    return _Dropout.apply(x, p, site)


# ---- linear ----------------------------------------------------------------------------------------------
class _Linear(Function):
    """y = act(x W^T + b + residual); W (N, K) as stored by nn.Linear.  N is padded to a multiple of 4 internally."""

    @staticmethod
    def forward(ctx, x, w, b, residual, relu):
        K_ = x.shape[-1]
        N = w.shape[0]
        Np = _pad4(N)
        x2 = x.reshape(-1, K_)
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        split = tc.get_precision() == "bf16x3"
        # bf16x3: the weight as (hi, lo) bf16 pairs in both operand layouts, split once per model forward (tc.prepacked)
        wr = tc.lookup_split(w) if split else tc.round_tf32(w.contiguous())
        r2 = None
        if residual is not None:
            r2 = residual.reshape(-1, N).contiguous()
        # the forward kernel takes any N (ragged right edge handled in its epilogue); only the backward operands need
        # 16-byte row pitches, so padding to a multiple of 4 happens there
        y = tc.linear_forward(x2, wr, None if b is None else b.contiguous(), r2, relu=relu)
        ctx.save_for_backward(x2, None if split else wr, y if relu else None)
        ctx.split_w = wr if split else None
        ctx.meta = (x.shape, N, Np, b is not None, residual is not None, relu)
        return y.view(*x.shape[:-1], N)

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x2, wr, y = ctx.saved_tensors
        if ctx.split_w is not None:
            wr = ctx.split_w
        xshape, N, Np, has_b, has_res, relu = ctx.meta
        dy2 = dy.reshape(-1, N).contiguous()
        if relu:
            dy2 = relu_backward(dy2, y) if N % 4 == 0 else dy2 * (y > 0)
        dres_src = dy2
        if Np != N:
            dy2 = F.pad(dy2, (0, Np - N))
            if ctx.split_w is None:                 # (a SplitW's k-blocks are zero-padded to 32 already)
                wr = F.pad(wr, (0, 0, 0, Np - N))
        dx = dw = db = dres = None
        want_db = has_b and ctx.needs_input_grad[2]
        fork = None
        if ctx.needs_input_grad[0] and ctx.needs_input_grad[1] and dy2.shape[0] <= _SIDE_MAX_ROWS:
            fork = _Fork()                    # small layer: weight gradient on the side stream, data gradient on this one
        if ctx.needs_input_grad[1]:
            with torch.cuda.stream(fork.side if fork else torch.cuda.current_stream()):
                if want_db:                   # bias gradient = by-product of the weight-gradient launch
                    dw, db = tc.linear_wgrad(dy2, x2, with_bias_grad=True)
                else:
                    dw = tc.linear_wgrad(dy2, x2)
        elif want_db:
            db = tc.colsum(dy2)
        if ctx.needs_input_grad[0]:
            dx = tc.linear_dgrad(dy2, wr).view(xshape)
        if fork:
            fork.join(dw, db)
        if dw is not None and Np != N:
            dw = dw[:N]
        if db is not None and Np != N:
            db = db[:N]
        if has_res and ctx.needs_input_grad[3]:
            dres = dres_src.view(*xshape[:-1], N)
        return dx, dw, db, dres, None


def linear(x, w, b=None, residual=None, relu=False):
    return _Linear.apply(x, w, b, residual, relu)


# ---- generic NHWC convolution with bias (neck / depth predictor; the ResNet body has its own schedule) ----
class _Conv2d(Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, pad):
        O, I, kh, kw = w.shape
        Op = _pad4(O)
        if tc.get_precision() == "bf16x3":
            # split (hi, lo) bf16 operands straight from the OIHW parameter; the forward writes a ragged Cout itself
            sw = tc.lookup_split(w)
            y = tc.conv2d_forward(x, sw, None if b is None else b.contiguous(), None, kh, kw, stride, pad)
            ctx.save_for_backward(x)
            ctx.split_w = sw
            ctx.meta = (O, Op, kh, kw, stride, pad, b is not None)
            return y
        wp = tc.pack_weight(w.contiguous())                      # (taps, O, I), rounded to TF32
        bp = b
        if Op != O:
            wp = F.pad(wp, (0, 0, 0, Op - O))
            bp = None if b is None else F.pad(b, (0, Op - O))
        y = tc.conv2d_forward(x, wp, None if bp is None else bp.contiguous(), None, kh, kw, stride, pad)
        ctx.save_for_backward(x, wp)
        ctx.split_w = None
        ctx.meta = (O, Op, kh, kw, stride, pad, b is not None)
        return y if Op == O else y[..., :O].contiguous()

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        if ctx.split_w is not None:
            (x,), wp = ctx.saved_tensors, ctx.split_w
        else:
            x, wp = ctx.saved_tensors
        O, Op, kh, kw, stride, pad, has_b = ctx.meta
        if Op != O:
            dy = F.pad(dy, (0, Op - O))
        dy = dy.contiguous()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = tc.conv2d_dgrad(dy, wp, x.shape, None, None, kh, kw, stride, pad)
        want_db = has_b and ctx.needs_input_grad[2]
        if ctx.needs_input_grad[1]:
            if want_db:
                dwp, db = tc.conv2d_wgrad(dy, x, None, kh, kw, stride, pad, with_bias_grad=True)
            else:
                dwp = tc.conv2d_wgrad(dy, x, None, kh, kw, stride, pad)
            dw = tc.unpack_wgrad(dwp, kh, kw)
            if Op != O:
                dw = dw[:O]
        elif want_db:
            db = tc.colsum(dy.view(-1, Op))
        if db is not None and Op != O:
            db = db[:O]
        return dx, dw, db, None, None


def conv2d_nhwc(x, w, b=None, stride=1, pad=0):
    return _Conv2d.apply(x.contiguous(), w, b, stride, pad)


# ---- normalisation -----------------------------------------------------------------------------------------
class _AddLayerNorm(Function):
    @staticmethod
    def forward(ctx, x, res, gamma, beta, eps, drop_p, site):
        x = x.contiguous()
        res = None if res is None else res.contiguous()
        ctx.seed = K.seed_tensor(x.device) if drop_p > 0 else None
        y, mean, rstd = K.add_layernorm_forward(x, res, gamma, beta, eps, drop_p, site, ctx.seed)
        ctx.save_for_backward(x, res, gamma, mean, rstd)
        ctx.meta = (drop_p, site)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, res, gamma, mean, rstd = ctx.saved_tensors
        drop_p, site = ctx.meta
        dx, dres, dg, db = K.add_layernorm_backward(dy, x, res, gamma, mean, rstd, drop_p, site, ctx.seed)
        return dx, (dres if res is not None else None), dg, db, None, None, None


def add_layernorm(x, res, gamma, beta, eps=1e-5, drop_p=0.0, training=False, site=0):
    """LayerNorm(x + dropout(res)) -- the residual/dropout/norm pattern of every transformer sub-block."""
    return _AddLayerNorm.apply(x, res, gamma, beta, eps, drop_p if training else 0.0, site)


class _GroupNorm(Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, G, eps, relu):
        x = x.contiguous()
        y, mean, rstd = K.groupnorm_forward(x, gamma, beta, G, eps, relu)
        ctx.save_for_backward(x, y if relu else None, gamma, mean, rstd)
        ctx.meta = (G, relu)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        x, y, gamma, mean, rstd = ctx.saved_tensors
        G, relu = ctx.meta
        dx, dg, db = K.groupnorm_backward(dy, x, y, gamma, mean, rstd, G, relu)
        return dx, dg, db, None, None, None


def groupnorm_nhwc(x, gamma, beta, G=32, eps=1e-5, relu=False):
    return _GroupNorm.apply(x, gamma, beta, G, eps, relu)


# ---- attention core -----------------------------------------------------------------------------------------
class _Attention(Function):
    @staticmethod
    def forward(ctx, q, k, v, kpm, drop_p, site):
        ctx.seed = K.seed_tensor(q.device) if drop_p > 0 else None
        out, lse, kp = K.attention_forward(q, k, v, kpm, drop_p, site, ctx.seed)
        ctx.save_for_backward(q, k, v, kp, out, lse)
        ctx.meta = (drop_p, site)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        q, k, v, kp, out, lse = ctx.saved_tensors
        drop_p, site = ctx.meta
        dq, dk, dv = K.attention_backward(q, k, v, kp, out, lse, dout, drop_p, site, ctx.seed)
        return dq, dk, dv, None, None, None


def attention(q, k, v, key_padding_mask=None, drop_p=0.0, training=False, site=0):
    """softmax(q k^T / sqrt(32)) v per head; q (B, Lq, 256), k/v (B, Lk, 256) (strided views allowed)."""
    return _Attention.apply(q, k, v, key_padding_mask, drop_p if training else 0.0, site)


def msda(value, spatial_shapes, level_start_index, sampling_locations, attention_weights):
    return MSDeformAttnFunction.apply(value, spatial_shapes, level_start_index, sampling_locations, attention_weights, 64)


class _MsdaPrep(Function):
    """(off, logits, ref) -> (sampling_locations, softmax attention weights); see csrc/msda.cu "Fused pre-processing"."""

    @staticmethod
    def forward(ctx, off, logits, ref, shapes, M, L, P):
        B, Lq = off.shape[0], off.shape[1]
        off = off.contiguous()
        logits = logits.contiguous()
        refc = ref.contiguous()
        rd = refc.shape[-1]
        loc = torch.empty((B, Lq, M, L, P, 2), dtype=torch.float32, device=off.device)
        attn = torch.empty((B, Lq, M, L, P), dtype=torch.float32, device=off.device)
        _lib.call("mdb_msda_prep_forward_f32", off, logits, refc, shapes, B, Lq, M, L, P, rd, loc, attn)
        # 6-d reference boxes that require grad (not on the model path, where they are detached -- depthaware_transformer.py
        # :613 -- but a custom decoder may pass them): keep the offsets for the box gradient
        keep_off = rd == 6 and ref.requires_grad
        ctx.save_for_backward(attn, refc, shapes, off if keep_off else None)
        ctx.meta = (B, Lq, M, L, P, rd, off.shape, logits.shape)
        return loc, attn

    @staticmethod
    @once_differentiable
    def backward(ctx, dloc, dattn):
        attn, refc, shapes, off = ctx.saved_tensors
        B, Lq, M, L, P, rd, oshape, lshape = ctx.meta
        dloc = dloc.contiguous()
        dattn = dattn.contiguous()
        doff = torch.empty(oshape, dtype=torch.float32, device=dloc.device)
        dlogits = torch.empty(lshape, dtype=torch.float32, device=dloc.device)
        _lib.call("mdb_msda_prep_backward_f32", dloc, dattn, attn, refc, shapes, B, Lq, M, L, P, rd, doff, dlogits)
        dref = None
        if ctx.needs_input_grad[2]:
            if rd == 2:
                dref = dloc.sum(dim=(2, 4))                               # (B, Lq, L, 2)
            else:
                # loc = ref_xy + off / P * (l + r, t + b) / 2 (ms_deform_attn.py:154-155; 2::2 -> (l, t), 3::2 -> (r, b)):
                # d/d(cx, cy) = sum dloc ; d/dl = d/dr = sum dloc_x off_x / (2P) ; d/dt = d/db = sum dloc_y off_y / (2P).
                # Small reductions in plain torch: this branch is never taken by the model (boxes are detached there).
                dxy = dloc.sum(dim=(2, 4))
                dwh = (dloc * off.view(B, Lq, M, L, P, 2)).sum(dim=(2, 4)) * (0.5 / P)   # (B, Lq, L, 2) = (d(l+r), d(t+b))
                dref = torch.stack((dxy[..., 0], dxy[..., 1], dwh[..., 0], dwh[..., 0], dwh[..., 1], dwh[..., 1]), -1)
        return doff, dlogits, dref, None, None, None, None


def msda_prep(off, logits, ref, spatial_shapes, M, L, P):
    return _MsdaPrep.apply(off, logits, ref, spatial_shapes, M, L, P)


def msda_fused_forward_raw(value, shapes, lsi, off, logits, refc):
    """mdb_msda_fused_forward_f32 on contiguous tensors (value (B,S,M,32), raw offsets / logits, constant reference points)."""
    B, S, M, D = value.shape
    Lq, rd = off.shape[1], refc.shape[-1]
    out = torch.empty((B, Lq, M * D), dtype=torch.float32, device=value.device)
    from . import msda as _m
    if _m.PROBE is not None:        # bench.py: CUDA events tight around the launch (nothing else between them)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    _lib.call("mdb_msda_fused_forward_f32", value, shapes, lsi, off, logits, refc, B, S, M, D, 4, Lq, 4, rd, out)
    if _m.PROBE is not None:
        e1.record()
        _m.PROBE.append((e0, e1, B, Lq))
    return out


def msda_fused_backward_raw(value, shapes, lsi, off, logits, refc, dout):
    B, S, M, D = value.shape
    Lq, rd = off.shape[1], refc.shape[-1]
    dout = dout.contiguous()
    gv, goff, glog = torch.empty_like(value), torch.empty_like(off), torch.empty_like(logits)
    _lib.call("mdb_msda_fused_backward_f32", value, shapes, lsi, off, logits, refc, dout, B, S, M, D, 4, Lq, 4, rd, gv, goff, glog)
    return gv, goff, glog


class _MsdaFused(Function):
    """value (B,S,M,32), raw offsets (B,Lq,M*4*4*2), raw logits (B,Lq,M*16), constant reference points (B,Lq,4,rd) -> (B,Lq,M*32):
    softmax / sampling-location pre-processing inside the sampling kernels (forward and backward)."""

    @staticmethod
    def forward(ctx, value, shapes, lsi, off, logits, ref):
        value, off, logits = value.contiguous(), off.contiguous(), logits.contiguous()
        refc = ref.detach().contiguous()
        out = msda_fused_forward_raw(value, shapes, lsi, off, logits, refc)
        ctx.save_for_backward(value, shapes, lsi, off, logits, refc)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        value, shapes, lsi, off, logits, refc = ctx.saved_tensors
        gv, goff, glog = msda_fused_backward_raw(value, shapes, lsi, off, logits, refc, dout)
        return gv, None, None, goff, glog, None


def msda_fused_applicable(value, ref, n_levels, n_points):
    return (value.dtype == torch.float32 and value.shape[-1] == 32 and n_levels == 4 and n_points == 4 and not ref.requires_grad
            and ref.shape[-1] in (2, 6) and not os.environ.get("MDB_MSDA_UNFUSED")
            and not _lib.lib().mdb_get_deterministic())      # reproducible mode: ordered scatter of the two-step path


def msda_fused(value, spatial_shapes, level_start_index, off, logits, ref):
    return _MsdaFused.apply(value, spatial_shapes, level_start_index, off, logits, ref)


# ---- one encoder layer as ONE autograd node ---------------------------------------------------------------------------
ENC_FUSED = not os.environ.get("MDB_NO_ENC_FUSED")
# the six weight-gradient GEMMs of a layer's backward on the side stream, beside the data-gradient chain (LayerNorm / dropout / MSDA
# scatter / dgrad GEMMs) they do not feed
# (measured on one box: 24.21 -> 24.08 ms per step; MDB_NO_ENC_WGRAD_SIDE=1: in line)
ENC_WGRAD_SIDE = not os.environ.get("MDB_NO_ENC_WGRAD_SIDE") and not os.environ.get("MDB_NO_SIDE_STREAM")


class _EncoderLayer(Function):
    """VisualEncoderLayer.forward (depthaware_transformer.py:315-354: deformable self-attention -> dropout / residual / LayerNorm ->
    FFN -> dropout / residual / LayerNorm) as ONE autograd node over the same kernels the separate nodes launch, so that the
    backward can hand every fan-in sum to a GEMM epilogue instead of autograd's stand-alone additions over (B, S, C) tensors:
      * d src1 = dgrad(linear1) + (LayerNorm-2 residual gradient)          -> residual operand of the dgrad epilogue
      * d query = dgrad(sampling_offsets) + dgrad(attention_weights)       -> residual operand
      * d src  = dgrad(value_proj) + (LayerNorm-1 residual gradient) [+ d query: the one addition left]
      * the ReLU mask of linear1 rides in linear2's dgrad epilogue (was a separate pass)
    Per layer 4 of 5 additions and the ReLU pass over 84 MB tensors disappear (B = 8, 1280 x 384).  Forward values are
    bit-identical to the separate nodes (same kernels, same order); gradients differ by the association of those sums."""

    @staticmethod
    def forward(ctx, src, pos, ref, shapes, lsi, n_heads, eps1, eps2, p, training, site,
                Wv, bv, Wo, bo, Wa, ba, Wu, bu, g1, be1, W1, b1, W2, b2, g2, be2):
        B, S, C = src.shape
        M = B * S
        src = src.contiguous()
        q = src + pos
        x2, q2 = src.view(M, C), q.view(M, C)
        sv, so, sa, su, s1, s2 = (tc.lookup_split(w) for w in (Wv, Wo, Wa, Wu, W1, W2))
        value = tc.linear_forward(x2, sv, bv)
        off = tc.linear_forward(q2, so, bo)
        logits = tc.linear_forward(q2, sa, ba)
        refc = ref.detach().contiguous()
        o = msda_fused_forward_raw(value.view(B, S, n_heads, C // n_heads), shapes, lsi, off.view(B, S, -1), logits.view(B, S, -1), refc)
        o2 = o.view(M, C)
        a = tc.linear_forward(o2, su, bu)
        drop = float(p) if training else 0.0
        seed = K.seed_tensor(src.device) if drop > 0 else None
        src1, mean1, rstd1 = K.add_layernorm_forward(x2, a, g1, be1, eps1, drop, site, seed)
        h = tc.linear_forward(src1, s1, b1, relu=True)
        hd = dropout_raw(h, drop, site + 1, seed) if drop > 0 else h
        f = tc.linear_forward(hd, s2, b2)
        out, mean2, rstd2 = K.add_layernorm_forward(src1, f, g2, be2, eps2, drop, site + 2, seed)
        ctx.save_for_backward(x2, q2, value, off, logits, refc, o2, a, src1, mean1, rstd1, h, hd if drop > 0 else None, f,
                              mean2, rstd2, shapes, lsi, g1, g2)
        ctx.splits = (sv, so, sa, su, s1, s2)
        ctx.meta = (B, S, C, n_heads, drop, site, pos.shape)
        ctx.seed = seed
        return out.view(B, S, C)

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        (x2, q2, value, off, logits, refc, o2, a, src1, mean1, rstd1, h, hd, f, mean2, rstd2, shapes, lsi, g1, g2) = ctx.saved_tensors
        sv, so, sa, su, s1, s2 = ctx.splits
        B, S, C, n_heads, drop, site, pos_shape = ctx.meta
        seed = ctx.seed
        M = B * S
        if hd is None:
            hd = h
        fork = _Fork() if (ENC_WGRAD_SIDE and dout.is_cuda) else None

        def wgrad(dy, x):
            """Weight + bias gradient; with the side stream: launched there once everything the main stream has produced so far
            (dy, x among it) is complete.  dy / x stay referenced by this frame until the join below, so the caching allocator cannot
            hand their memory to later main-stream work while the side stream still reads it."""
            if fork is None:
                return tc.linear_wgrad(dy, x, with_bias_grad=True)
            fork.side.wait_stream(fork.main)
            with torch.cuda.stream(fork.side):
                return tc.linear_wgrad(dy, x, with_bias_grad=True)

        # ---- LayerNorm 2, FFN ------------------------------------------------------------------------------------------------
        d_src1_res, d_f, dg2, dbe2 = K.add_layernorm_backward(dout.reshape(M, C), src1, f, g2, mean2, rstd2, drop, site + 2, seed)
        dW2, db2 = wgrad(d_f, hd)
        d_h = tc.linear_dgrad(d_f, s2, relu_mask=h)                        # ReLU mask in the epilogue (commutes with the dropout scaling)
        if drop > 0:
            d_h = dropout_raw(d_h, drop, site + 1, seed)
        dW1, db1 = wgrad(d_h, src1)
        d_src1 = tc.linear_dgrad(d_h, s1, residual=d_src1_res)             # + the residual branch of LayerNorm 2
        # ---- LayerNorm 1, output projection, deformable attention ----------------------------------------------------------
        d_x_res, d_a, dg1, dbe1 = K.add_layernorm_backward(d_src1, x2, a, g1, mean1, rstd1, drop, site, seed)
        dWu, dbu = wgrad(d_a, o2)
        d_o = tc.linear_dgrad(d_a, su)
        gv, goff, glog = msda_fused_backward_raw(value.view(B, S, n_heads, C // n_heads), shapes, lsi, off.view(B, S, -1),
                                                 logits.view(B, S, -1), refc, d_o.view(B, S, C))
        gv2, goff2, glog2 = gv.view(M, C), goff.view(M, -1), glog.view(M, -1)
        dWo, dbo = wgrad(goff2, q2)
        dWa, dba = wgrad(glog2, q2)
        dWv, dbv = wgrad(gv2, x2)
        d_q = tc.linear_dgrad(goff2, so)
        d_q = tc.linear_dgrad(glog2, sa, residual=d_q)                     # d query = both projections' data gradients
        d_pos = d_q.view(B, S, C).sum_to_size(pos_shape) if ctx.needs_input_grad[1] else None
        d_src = tc.linear_dgrad(gv2, sv, residual=d_x_res)                 # + the residual branch of LayerNorm 1
        d_src.add_(d_q)                                                     # + the query path (query = src + pos)
        if fork is not None:
            fork.join(dWv, dbv, dWo, dbo, dWa, dba, dWu, dbu, dW1, db1, dW2, db2)
        return (d_src.view(B, S, C), d_pos, None, None, None, None, None, None, None, None, None,
                dWv, dbv, dWo, dbo, dWa, dba, dWu, dbu, dg1, dbe1, dW1, db1, dW2, db2, dg2, dbe2)


def encoder_layer_fusable(layer, src, reference_points, padding_mask):
    """The fused node covers the configuration the model runs (configs/monodetr.yaml): BF16x3 arithmetic, D = 32 x 4 levels x 4
    points with constant reference points, no padding mask; anything else takes the separate nodes."""
    att = layer.self_attn
    dims_ok = all(w.shape[0] % 4 == 0 and w.shape[1] % 4 == 0 for w in (att.sampling_offsets.weight, att.attention_weights.weight,
                                                                         layer.linear1.weight, layer.linear2.weight))
    return (ENC_FUSED and src.is_cuda and src.dtype == torch.float32 and padding_mask is None and tc.get_precision() == "bf16x3"
            and not getattr(att, "freeze_sampling_locations", False) and dims_ok and src.dim() == 3
            and src.shape[-1] // att.n_heads == 32 and src.shape[-1] % att.n_heads == 0
            and msda_fused_applicable(src.reshape(src.shape[0], src.shape[1], att.n_heads, -1), reference_points, att.n_levels, att.n_points)
            and all(m.bias is not None for m in (att.value_proj, att.sampling_offsets, att.attention_weights, att.output_proj,
                                                 layer.linear1, layer.linear2)))


def encoder_layer(layer, src, pos, reference_points, spatial_shapes, level_start_index):
    att = layer.self_attn
    return _EncoderLayer.apply(src, pos, reference_points, spatial_shapes, level_start_index, att.n_heads, layer.norm1.eps,
                               layer.norm2.eps, layer.dropout1.p, layer.training, layer.site_base,
                               att.value_proj.weight, att.value_proj.bias, att.sampling_offsets.weight, att.sampling_offsets.bias,
                               att.attention_weights.weight, att.attention_weights.bias, att.output_proj.weight, att.output_proj.bias,
                               layer.norm1.weight, layer.norm1.bias, layer.linear1.weight, layer.linear1.bias,
                               layer.linear2.weight, layer.linear2.bias, layer.norm2.weight, layer.norm2.bias)


class _DepthSample(Function):
    """grid_sample(depth[:, None], xy[:, :, None], bilinear, zeros, align_corners=True) -> (B, N); xy is not differentiated."""

    @staticmethod
    def forward(ctx, depth, xy):
        depth = depth.contiguous()
        xy = xy.detach().contiguous()
        B, H, W = depth.shape
        N = xy.shape[1]
        out = torch.empty((B, N), dtype=torch.float32, device=depth.device)
        _lib.call("mdb_depth_sample_forward_f32", depth, xy, out, B, H, W, N)
        ctx.save_for_backward(xy)
        ctx.meta = (B, H, W, N)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        (xy,) = ctx.saved_tensors
        B, H, W, N = ctx.meta
        dd = torch.empty((B, H, W), dtype=torch.float32, device=dout.device)
        _lib.call("mdb_depth_sample_backward_f32", dout.contiguous(), xy, dd, B, H, W, N)
        return dd, None


def depth_sample(depth, xy):
    return _DepthSample.apply(depth, xy)


# ---- fused elementwise chains around the heads / depth predictor tail (csrc/heads.cu) ----------------------------------
import ctypes as _ct


class _BoxRefine(Function):
    """sigmoid(tmp + inverse_sigmoid(ref)) on the first ref_dim components (depthaware_transformer.py:602-613)."""

    @staticmethod
    def forward(ctx, tmp, ref):
        tmp = tmp.contiguous()
        refc = ref.detach().contiguous()
        rd = refc.shape[-1]
        n = tmp.numel() // 6
        y = torch.empty_like(tmp)
        _lib.call("mdb_box_refine_forward_f32", tmp, refc, y, n, rd)
        ctx.save_for_backward(y, refc)
        ctx.meta = (n, rd, ref.shape)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        y, refc = ctx.saved_tensors
        n, rd, rshape = ctx.meta
        dy = dy.contiguous()
        dtmp = torch.empty_like(y)
        dref = torch.empty(rshape, dtype=torch.float32, device=y.device) if ctx.needs_input_grad[1] else None
        _lib.call("mdb_box_refine_backward_f32", dy, y, refc, dtmp, dref, n, rd)
        return dtmp, dref


def box_refine(tmp, ref):
    return _BoxRefine.apply(tmp, ref)


class _HeadDepth(Function):
    """monodetr.py:230-262: ((1/(sigmoid(reg0)+1e-6) - 1) + geometric depth + depth-map lookup) / 3 and reg1 -> (B, N, 2)."""

    @staticmethod
    def forward(ctx, coord, size3d, depth_reg, wdepth, calibs, img_sizes):
        coord, size3d, depth_reg, wdepth = (t.contiguous() for t in (coord, size3d, depth_reg, wdepth))
        calibs = calibs.contiguous().float()
        img_sizes = img_sizes.contiguous().float()
        B, N, _ = coord.shape
        _, H, W = wdepth.shape
        out = torch.empty((B, N, 2), dtype=torch.float32, device=coord.device)
        _lib.call("mdb_head_depth_forward_f32", coord, size3d, depth_reg, wdepth, calibs, img_sizes, out, B, N, H, W)
        ctx.save_for_backward(coord, size3d, depth_reg, calibs, img_sizes)
        ctx.meta = (B, N, H, W)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dout):
        coord, size3d, depth_reg, calibs, img_sizes = ctx.saved_tensors
        B, N, H, W = ctx.meta
        dout = dout.contiguous()
        dcoord, dsize, dreg = torch.empty_like(coord), torch.empty_like(size3d), torch.empty_like(depth_reg)
        dwd = torch.empty((B, H, W), dtype=torch.float32, device=dout.device)
        # reproducible mode: the map gradient is a second (gather) launch
        _lib.call("mdb_head_depth_backward_f32", dout, coord, size3d, depth_reg, calibs, img_sizes, dcoord, dsize, dreg, dwd, B, N, H, W,
                  launches=2 if _lib.deterministic() else 1)
        return dcoord, dsize, dreg, dwd, None, None


def head_depth(coord, size3d, depth_reg, wdepth, calibs, img_sizes):
    return _HeadDepth.apply(coord, size3d, depth_reg, wdepth, calibs, img_sizes)


class _DepthTail(Function):
    """depth_predictor.py:74-104: logits (B,H,W,nb) -> weighted_depth (B,H,W), interpolated depth embedding (B,H,W,C)."""

    @staticmethod
    def forward(ctx, logits, bins, emb, dmax):
        logits = logits.contiguous()
        bins = bins.detach().contiguous()
        embc = emb.contiguous()
        B, H, W, nb = logits.shape
        E, C = embc.shape
        wd = torch.empty((B, H, W), dtype=torch.float32, device=logits.device)
        ip = torch.empty((B, H, W, C), dtype=torch.float32, device=logits.device)
        _lib.call("mdb_depth_tail_forward_f32", logits, bins, embc, wd, ip, B * H * W, nb, E, C, float(dmax))
        ctx.save_for_backward(logits, bins, embc)
        ctx.meta = (B * H * W, nb, E, C, float(dmax))
        return wd, ip

    @staticmethod
    @once_differentiable
    def backward(ctx, dwd, dip):
        logits, bins, embc = ctx.saved_tensors
        npix, nb, E, C, dmax = ctx.meta
        dip = torch.zeros((npix, C), dtype=torch.float32, device=logits.device) if dip is None else dip.contiguous()
        dwd = None if dwd is None else dwd.contiguous()
        dlogits = torch.empty_like(logits)
        demb = torch.empty_like(embc)
        # reproducible mode: the embedding gradient is a second, fixed-order launch
        _lib.call("mdb_depth_tail_backward_f32", logits, bins, embc, dip, dwd, dlogits, demb, npix, nb, E, C, dmax,
                  launches=2 if _lib.deterministic() else 1)
        return dlogits, None, demb, None


def depth_tail(logits, bins, emb, dmax):
    return _DepthTail.apply(logits, bins, emb, dmax)


class _UpsampleBilinear(Function):
    """F.interpolate(x, size, mode="bilinear", align_corners=False) on an NHWC map (B, H, W, C) -> (B, Ho, Wo, C); the backward is a
    gather (no atomics), so it is bit-reproducible."""

    @staticmethod
    def forward(ctx, x, Ho, Wo):
        x = x.contiguous()
        B, H, W, C = x.shape
        y = torch.empty((B, Ho, Wo, C), dtype=torch.float32, device=x.device)
        _lib.call("mdb_upsample_bilinear_nhwc_forward_f32", x, y, B, H, W, Ho, Wo, C)
        ctx.meta = (B, H, W, Ho, Wo, C)
        return y

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        B, H, W, Ho, Wo, C = ctx.meta
        dx = torch.empty((B, H, W, C), dtype=torch.float32, device=dy.device)
        _lib.call("mdb_upsample_bilinear_nhwc_backward_f32", dy.contiguous(), dx, B, H, W, Ho, Wo, C)
        return dx, None, None


def upsample_bilinear_nhwc(x, size):
    """Bilinear resize of an NHWC map to size = (Ho, Wo), torch's align_corners=False rule."""
    return _UpsampleBilinear.apply(x, int(size[0]), int(size[1]))


class _Mean3(Function):
    @staticmethod
    def forward(ctx, a, b, c):
        a, b, c = a.contiguous(), b.contiguous(), c.contiguous()
        out = torch.empty_like(a)
        _lib.call("mdb_mean3_f32", a, b, c, out, a.numel())
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        dy = dy.contiguous()
        g = torch.empty_like(dy)
        _lib.call("mdb_scale_f32", dy, g, dy.numel(), 1.0 / 3.0)
        return g, g, g


def mean3(a, b, c):
    """(a + b + c) / 3 (depth_predictor.py:66)."""
    return _Mean3.apply(a, b, c)


class _SumMeanSquares(Function):
    """sum_k mean(x_k^2) over a list of tensors in ONE launch (and one for the backward): the surrogate loss of SURVEY.md 8(d)."""

    @staticmethod
    def forward(ctx, *xs):
        xs = [x.contiguous() for x in xs]
        n = len(xs)
        loss = torch.empty((), dtype=torch.float32, device=xs[0].device)
        nums = (_ct.c_longlong * n)(*[x.numel() for x in xs])
        _lib.call("mdb_sum_mean_squares_forward_f32", n, xs, nums, loss)
        ctx.save_for_backward(*xs)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, dloss):
        xs = ctx.saved_tensors
        n = len(xs)
        gs = [torch.empty_like(x) for x in xs]
        nums = (_ct.c_longlong * n)(*[x.numel() for x in xs])
        _lib.call("mdb_sum_mean_squares_backward_f32", n, xs, gs, nums, dloss.contiguous().float())
        return tuple(gs)


def sum_mean_squares(tensors):
    return _SumMeanSquares.apply(*tensors)
