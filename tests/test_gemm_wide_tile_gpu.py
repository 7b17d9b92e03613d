"""The 128 x 256 tile of the BF16x3 forward / data-gradient GEMM (csrc/conv_gemm.cu: `m64n256k16` wgmmas, 128
accumulators per consumer thread, an epilogue staged through two 32-channel boxes per warpgroup in turn).

Every case runs at a shape whose launch selects the wide tile (`pick_bn`, restated below and asserted, so that a shape
never silently tests the 128-wide tile: N a multiple of 256 and at least 64 k-blocks of reduction) and is held to the fp64
bounds of tests/tc_error_model.py: output widths 256 to 2048, row tails, 3x3 stride 1 and 2, a stride-2 data gradient whose
odd parity classes no tap reaches, bias + residual + ReLU, a mask beside a residual, and more tiles than SMs.  (Split-K
slices are 32 k-blocks long, so the neck convolution keeps the 128-wide tile.)  The wide tile must also give the 128-wide
tile's bits: each output element sees the same wgmmas in the same k order, which is what lets the width depend on the
batch while an image's output does not."""
import pytest
import torch
import torch.nn.functional as F

import tc_error_model as em

pytestmark = pytest.mark.gpu

MODE = "bf16x3"


@pytest.fixture(autouse=True)
def bf16x3():
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(MODE)
    yield
    tc.set_precision(prev)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _pick_tile3(W, H, B, n_pix=128):
    """(tw, th, tb) of an M tile: pick_tile3 of conv_gemm.cu."""
    best, res, b = -1, (n_pix, 1, 1), 1
    while b <= n_pix:
        w = n_pix // b
        while w >= 1:
            h = n_pix // b // w
            if not (b > 1 and b >= 2 * B):
                cov = -(-W // w) * w * -(-H // h) * h * -(-B // b) * b
                if best < 0 or cov < best:
                    best, res = cov, (w, h, b)
            w >>= 1
        b <<= 1
    return res


def _m_tiles(W, H, B):
    tw, th, tb = _pick_tile3(W, H, B)
    return -(-W // tw) * -(-H // th) * -(-B // tb)


def _wide(N, m_tiles, kblocks):
    """pick_bn of conv_gemm.cu: True when the launch runs 128 x 256 tiles."""
    if N % 256 or kblocks < 64:
        return False
    sms, t = _sms(), m_tiles * (N // 256)
    return 2 * -(-t // sms) <= -(-2 * t // sms)


def _pack(w):
    O, I, kh, kw = w.shape
    return w.permute(2, 3, 0, 1).reshape(kh * kw, O, I).contiguous()


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


# M, K, N: row tails (M % 128 != 0) at every output width the model has, each with enough tiles to select the wide tile
LINEARS = [(8577, 2048, 256), (4353, 2048, 512), (2177, 2080, 1024), (1537, 2048, 2048)]


@pytest.mark.parametrize("cfg", LINEARS)
def test_linear_widths(cfg):
    """Forward with bias + residual + ReLU, data gradient (K -> N, output width N) with a residual and a mask beside it."""
    from monodetr_b200 import tc
    M, K, N = cfg
    assert _wide(N, -(-M // 128), -(-K // 32))
    g = _gen(M)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(M, N, device="cuda", generator=g)
    t, s = em.target(lambda a, c: a @ c.t(), x, w, MODE)
    y = tc.linear_forward(x, tc.split_weights([w])[0], b, r, relu=True)
    em.assert_gemm(f"fwd {cfg}", y, torch.relu(t + b.double() + r.double()), s, MODE, epi=em.epi_mag(t, b, r))

    wd = torch.randn(K, N, device="cuda", generator=g) / K ** 0.5    # layer N -> K: its data gradient is N wide
    dy = torch.randn(M, K, device="cuda", generator=g)
    mask = torch.randn(M, N, device="cuda", generator=g)
    mask[:, ::3] = -0.0
    gate = (mask > 0).double()
    t, s = em.target(lambda a, c: a @ c, dy, wd, MODE)
    wds = tc.split_weights([wd])[0]
    for rr, m in ((r, mask), (None, mask), (r, None), (None, None)):
        gr = 1.0 if m is None else gate
        ref = (t + (0 if rr is None else rr.double())) * gr
        dx = tc.linear_dgrad(dy, wds, rr, m)
        em.assert_gemm(f"dgrad {cfg} res={rr is not None} mask={m is not None}", dx, ref, s * gr, MODE,
                       epi=None if rr is None else em.epi_mag(t, None, rr) * gr)


# B, H, W, Cin, Cout, k, stride, pad: the layer-3 3x3 shape (24 x 80 out, 120 tiles, 72 k-blocks) at stride 1 and 2, and
# a 1x1 stride-2 projection over 2048 channels whose odd dgrad parity classes no tap reaches (those run 128-wide: no k-blocks)
CONVS = [
    (8, 24, 80, 256, 256, 3, 1, 1),
    (8, 48, 160, 256, 256, 3, 2, 1),
    (8, 48, 160, 256, 2048, 1, 2, 0),
]


@pytest.mark.parametrize("cfg", CONVS)
def test_conv(cfg):
    """Forward (bias + residual + ReLU) where Cout selects the wide tile, data gradient (residual and mask, each alone
    and both) where Cin does."""
    from monodetr_b200 import tc
    B, H, W, Cin, Cout, k, st, pad = cfg
    Ho, Wo = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
    g = _gen(sum(cfg))
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    ws, wp = tc.split_weights([w])[0], _pack(w)
    fwd_wide = _wide(Cout, _m_tiles(Wo, Ho, B), k * k * -(-Cin // 32))
    taps = [sum((py + pad - ky) % st == 0 for ky in range(k)) * sum((px + pad - kx) % st == 0 for kx in range(k))
            for py in range(st) for px in range(st)]
    dgrad_wide = any(_wide(Cin, _m_tiles(-(-(W - px) // st), -(-(H - py) // st), B), taps[py * st + px] * -(-Cout // 32))
                     for py in range(st) for px in range(st))
    assert fwd_wide or dgrad_wide
    if fwd_wide:
        bias = torch.randn(Cout, device="cuda", generator=g)
        t, s = em.target(_conv_f(k, st, pad), x, wp, MODE)
        res = torch.randn(t.shape, device="cuda", generator=g)
        y = tc.conv2d_forward(x, ws, bias, res, k, k, st, pad, relu=True)
        em.assert_gemm(f"fwd {cfg}", y, torch.relu(t + bias.double() + res.double()), s, MODE, epi=em.epi_mag(t, bias, res))
    if dgrad_wide:
        dy = torch.randn(B, Ho, Wo, Cout, device="cuda", generator=g)
        t, s = em.target(_dgrad_f(x.shape, k, st, pad), dy, wp, MODE)
        r2 = torch.randn(x.shape, device="cuda", generator=g)
        mask = torch.randn(x.shape, device="cuda", generator=g)
        mask[..., ::3] = -0.0
        gate = (mask > 0).double()
        for r, m in ((r2, mask), (None, mask), (r2, None)):
            gr = 1.0 if m is None else gate
            ref = (t + (0 if r is None else r.double())) * gr
            dx = tc.conv2d_dgrad(dy, ws, x.shape, r, m, k, k, st, pad)
            em.assert_gemm(f"dgrad {cfg} res={r is not None} mask={m is not None}", dx, ref, s * gr, MODE,
                           epi=None if r is None else em.epi_mag(t, None, r) * gr)


def test_many_tiles():
    """3x3 256 -> 256 over 16 images at 24 x 80 (240 wide tiles on 132 SMs: each CTA's ring, staging boxes and epilogue
    barriers cycle through two tiles): forward with bias + residual + ReLU, data gradient with the mask alone (fetched by
    TMA) and with a mask beside a residual."""
    from monodetr_b200 import tc
    B, H, W, C = 16, 24, 80, 256
    assert _wide(C, _m_tiles(W, H, B), 72) and _m_tiles(W, H, B) > _sms()
    g = _gen(3)
    x = torch.randn(B, H, W, C, device="cuda", generator=g)
    w = torch.randn(C, C, 3, 3, device="cuda", generator=g) / (C * 9) ** 0.5
    ws, wp = tc.split_weights([w])[0], _pack(w)
    bias = torch.randn(C, device="cuda", generator=g)
    r = torch.randn(B, H, W, C, device="cuda", generator=g)
    t, s = em.target(_conv_f(3, 1, 1), x, wp, MODE)
    y = tc.conv2d_forward(x, ws, bias, r, 3, 3, 1, 1, relu=True)
    em.assert_gemm("fwd+b+r+relu", y, torch.relu(t + bias.double() + r.double()), s, MODE, epi=em.epi_mag(t, bias, r))
    dy = torch.randn(B, H, W, C, device="cuda", generator=g)
    mask = torch.randn(B, H, W, C, device="cuda", generator=g)
    t, s = em.target(_dgrad_f(x.shape, 3, 1, 1), dy, wp, MODE)
    gate = (mask > 0).double()
    em.assert_gemm("dgrad+mask", tc.conv2d_dgrad(dy, ws, x.shape, None, mask, 3, 3, 1, 1), t * gate, s * gate, MODE)
    em.assert_gemm("dgrad+res+mask", tc.conv2d_dgrad(dy, ws, x.shape, r, mask, 3, 3, 1, 1), (t + r.double()) * gate,
                   s * gate, MODE, epi=em.epi_mag(t, None, r) * gate)


def test_wide_equals_narrow_bits():
    """A 256-wide launch gives the bits of two 128-wide launches over its column halves (forward with bias + residual +
    ReLU, data gradient with residual + mask), and an image's output does not depend on the batch it runs in (batch 8:
    wide tiles; batch 1: 128-wide)."""
    from monodetr_b200 import tc
    B, H, W, Cin, Cout = 8, 24, 80, 256, 256
    assert _wide(Cout, _m_tiles(W, H, B), 72) and not _wide(Cout, _m_tiles(W, H, 1), 72)
    g = _gen(5)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (Cin * 9) ** 0.5
    bias = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    y = tc.conv2d_forward(x, tc.split_weights([w])[0], bias, res, 3, 3, 1, 1, relu=True)
    halves = [tc.conv2d_forward(x, tc.split_weights([w[i:i + 128].contiguous()])[0], bias[i:i + 128].contiguous(),
                                res[..., i:i + 128].contiguous(), 3, 3, 1, 1, relu=True) for i in (0, 128)]
    assert torch.equal(y, torch.cat(halves, -1))
    y1 = tc.conv2d_forward(x[:1].contiguous(), tc.split_weights([w])[0], bias, res[:1].contiguous(), 3, 3, 1, 1, relu=True)
    assert torch.equal(y[:1], y1)

    # data gradient of a layer 256 -> 256: output width 256, 72 k-blocks
    wd = torch.randn(256, Cout, 3, 3, device="cuda", generator=g) / (Cout * 9) ** 0.5
    dy = torch.randn(B, H, W, 256, device="cuda", generator=g)
    mask = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    dx = tc.conv2d_dgrad(dy, tc.split_weights([wd])[0], (B, H, W, Cout), res, mask, 3, 3, 1, 1)
    parts = [tc.conv2d_dgrad(dy, tc.split_weights([wd[:, i:i + 128].contiguous()])[0], (B, H, W, 128),
                             res[..., i:i + 128].contiguous(), mask[..., i:i + 128].contiguous(), 3, 3, 1, 1) for i in (0, 128)]
    assert torch.equal(dx, torch.cat(parts, -1))
    dx1 = tc.conv2d_dgrad(dy[:1].contiguous(), tc.split_weights([wd])[0], (1, H, W, Cout), res[:1].contiguous(),
                          mask[:1].contiguous(), 3, 3, 1, 1)
    assert torch.equal(dx[:1], dx1)
