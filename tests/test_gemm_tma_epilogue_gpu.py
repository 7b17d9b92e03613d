"""The TMA epilogue of the tensor-core GEMM's forward and data gradient (csrc/conv_gemm.cu): results staged in shared
memory and stored by bulk tensor copies, with the residual or ReLU mask fetched by TMA.  Held to the fp64 bounds of
tests/tc_error_model.py where the tensor maps clip -- partial boxes at the right and bottom edges and in the last image
group, stride-2 dgrad parity classes, forward split-K slices, more tiles than SMs -- and bit for bit against the register
epilogue, which launches TMA cannot describe (operands not 16-byte aligned, a channel count that is not a multiple of 4)
and the weight gradient (accumulated with a row scale) still take."""
import pytest
import torch
import torch.nn.functional as F

import tc_error_model as em

pytestmark = pytest.mark.gpu

MODES = ["bf16x3", "tf32x3", "tf32"]


@pytest.fixture(params=MODES)
def mode(request):
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(request.param)
    yield request.param
    tc.set_precision(prev)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _pack(w):
    O, I, kh, kw = w.shape
    return w.permute(2, 3, 0, 1).reshape(kh * kw, O, I).contiguous()


def _operand(mode, w):
    from monodetr_b200 import tc
    return tc.split_weights([w])[0] if mode == "bf16x3" else _pack(w)


def _misaligned(t):
    """A copy of t whose storage starts 8 bytes after a 16-byte boundary: TMA cannot take it, the register epilogue's
    float2 accesses can."""
    buf = torch.empty(t.numel() + 2, device=t.device, dtype=t.dtype)
    out = buf[2:].view(t.shape)
    out.copy_(t)
    assert out.data_ptr() % 16 != 0
    return out


def _conv_f(k, stride, pad):
    def f(a, b):
        taps, O, I = b.shape
        return F.conv2d(a.permute(0, 3, 1, 2), b.view(k, k, O, I).permute(2, 3, 0, 1), stride=stride, padding=pad).permute(0, 2, 3, 1)
    return f


def _dgrad_f(shape, k, stride, pad):
    def f(a, b):
        taps, O, I = b.shape
        B, H, W, C = shape
        return torch.nn.grad.conv2d_input((B, C, H, W), b.view(k, k, O, I).permute(2, 3, 0, 1), a.permute(0, 3, 1, 2),
                                          stride=stride, padding=pad).permute(0, 2, 3, 1)
    return f


# B, H, W, Cin, Cout, k, stride, pad: images smaller than a tile (tiles span tb > 1 images, B not a multiple of tb), widths
# and heights that leave partial boxes at the right and bottom edges, Cout past a 64 / 128 tile, stride-2 parity classes
# of unequal size, and a 1x1 stride-2 layer whose odd classes no tap reaches (dgrad = residual * mask).
SHAPES = [
    (5, 3, 5, 36, 68, 3, 1, 1),
    (3, 6, 20, 64, 132, 3, 1, 1),
    (2, 13, 11, 68, 64, 3, 2, 1),
    (3, 7, 9, 32, 200, 3, 2, 1),
    (2, 9, 11, 68, 132, 1, 2, 0),
]


@pytest.mark.parametrize("cfg", SHAPES)
def test_conv_partial_boxes(mode, cfg):
    from monodetr_b200 import tc
    B, H, W, Cin, Cout, k, st, pad = cfg
    g = _gen(sum(cfg))
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    wop, wp = _operand(mode, w), _pack(w)
    bias = torch.randn(Cout, device="cuda", generator=g)
    t, s = em.target(_conv_f(k, st, pad), x, wp, mode)
    res = torch.randn(t.shape, device="cuda", generator=g)
    y = tc.conv2d_forward(x, wop, bias, res, k, k, st, pad, relu=True)
    em.assert_gemm(f"fwd {cfg}", y, torch.relu(t + bias.double() + res.double()), s, mode, epi=em.epi_mag(t, bias, res))
    assert torch.equal(y, tc.conv2d_forward(x, wop, bias, _misaligned(res), k, k, st, pad, relu=True))

    dy = torch.randn(t.shape, device="cuda", generator=g)
    t, s = em.target(_dgrad_f(x.shape, k, st, pad), dy, wp, mode)
    r2 = torch.randn(x.shape, device="cuda", generator=g)
    mask = torch.randn(x.shape, device="cuda", generator=g)
    mask[..., ::3] = -0.0
    gate = (mask > 0).double()
    for r, m in ((r2, mask), (None, mask), (r2, None)):
        gr = 1.0 if m is None else gate
        ref = (t + (0 if r is None else r.double())) * gr
        dx = tc.conv2d_dgrad(dy, wop, x.shape, r, m, k, k, st, pad)
        em.assert_gemm(f"dgrad {cfg} res={r is not None} mask={m is not None}", dx, ref, s * gr, mode,
                       epi=None if r is None else em.epi_mag(t, None, r) * gr)
        mis = [None if a is None else _misaligned(a) for a in (r, m)]
        assert torch.equal(dx, tc.conv2d_dgrad(dy, wop, x.shape, mis[0], mis[1], k, k, st, pad))


def test_forward_splitk_partial_channels(mode):
    """3x3 conv over 1024 channels (288 k-blocks: split-K in the compensated modes) with Cout = 132: every slice's box
    clips at 4 channels of its second column tile, and at the right and bottom image edges."""
    from monodetr_b200 import tc
    B, H, W, Cin, Cout = 3, 7, 13, 1024, 132
    g = _gen(7)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (Cin * 9) ** 0.5
    bias = torch.randn(Cout, device="cuda", generator=g)
    t, s = em.target(_conv_f(3, 2, 1), x, _pack(w), mode)
    y = tc.conv2d_forward(x, _operand(mode, w), bias, None, 3, 3, 2, 1)
    em.assert_gemm("fwd split-K", y, t + bias.double(), s, mode, epi=em.epi_mag(t, bias))


@pytest.mark.parametrize("cfg", [(2, 13, 11, 68, 64, 3, 2, 1), (1, 1, 4400, 256, 128, 1, 1, 0)])
def test_wgrad_accumulate_rowscale(mode, cfg):
    """dw (+)= rowscale * dy^T x (register epilogue): onto a zeroed buffer, then accumulated onto itself, in the default
    (split-K) and the reproducible (one split) mode."""
    import monodetr_b200
    from monodetr_b200 import _lib
    B, H, W, Cin, Cout, k, st, pad = cfg
    g = _gen(sum(cfg) + 1)
    Ho, Wo = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
    dy = torch.randn(B, Ho, Wo, Cout, device="cuda", generator=g)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5

    def wgrad_f(a, b):
        return _pack(torch.nn.grad.conv2d_weight(b.permute(0, 3, 1, 2), (Cout, Cin, k, k), a.permute(0, 3, 1, 2), stride=st, padding=pad))

    t, s = em.target(wgrad_f, dy, x, mode)
    sc = scale.double().view(1, -1, 1)
    for det in (False, True):
        prev = monodetr_b200.set_deterministic(det)
        try:
            dw = torch.full((k * k, Cout, Cin), float("nan"), device="cuda")
            for acc in (0, 1):
                _lib.call("mdb_conv2d_wgrad_f32", dy, x, scale, dw, B, H, W, Cin, Cout, k, k, st, pad, acc)
            torch.cuda.synchronize()
        finally:
            monodetr_b200.set_deterministic(prev)
        em.assert_gemm(f"wgrad x2 {cfg} reproducible={det}", dw, 2 * t * sc, 2 * s * sc, mode, epi=2 * t.abs() * sc)


def test_many_tiles(mode):
    """81 601 rows x 256 (1 276 tiles on 132 SMs, the last box 1 row tall): forward with residual + ReLU, dgrad with the
    mask alone (fetched by TMA) -- the staging tile is reused across ~10 tiles per CTA."""
    from monodetr_b200 import tc
    M, N, K = 81601, 256, 64
    g = _gen(3)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    r = torch.randn(M, N, device="cuda", generator=g)
    t, s = em.target(lambda a, b: a @ b.t(), x, w, mode)
    y = tc.linear_forward(x, w, None, r, relu=True)
    em.assert_gemm("linear+r+relu", y, torch.relu(t + r.double()), s, mode, epi=em.epi_mag(t, None, r))
    dy = torch.randn(M, N, device="cuda", generator=g)
    mask = torch.randn(M, K, device="cuda", generator=g)
    t, s = em.target(lambda a, b: a @ b, dy, w, mode)
    gate = (mask > 0).double()
    dx = tc.linear_dgrad(dy, w, None, mask)
    em.assert_gemm("dgrad+mask", dx, t * gate, s * gate, mode)
    assert torch.equal(dx, tc.linear_dgrad(dy, w, None, _misaligned(mask)))


def test_register_fallback_odd_channels(mode):
    """Cout = 65 (no 16-byte output pitch): the forward keeps the register epilogue's scalar stores."""
    from monodetr_b200 import tc
    M, N, K = 1000, 65, 36
    g = _gen(65)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(M, N, device="cuda", generator=g)
    t, s = em.target(lambda a, c: a @ c.t(), x, w, mode)
    y = tc.linear_forward(x, w, b, r, relu=True)
    em.assert_gemm("linear N=65", y, torch.relu(t + b.double() + r.double()), s, mode, epi=em.epi_mag(t, b, r))
