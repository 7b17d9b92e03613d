"""GPU: the grouped 3x3 convolutions (ResNeXt's conv2) on the channel-banded wgmma kernels, per element against float64
torch.nn.functional.conv2d(..., groups=g) under the bounds of tests/tc_error_model.py, in every precision mode: forward,
data gradient and weight gradient; channels per group 4..64 at C = 128 and at C >= 1024; stride 1 and 2, dilation 2;
partial spatial tiles; both epilogue kinds; reproducibility, batch independence and the weight pack / unpack round trip."""
import pytest
import torch
import torch.nn.functional as F

import tc_error_model as em

pytestmark = pytest.mark.gpu

# (C, groups, B, H, W, stride, dilation): channels per group 4 / 8 / 16 / 32 / 64 at C = 128 and 4 / 32 / 64 at C >= 1024,
# spatial sizes that leave partial 128-pixel tiles
CASES = [
    (128, 32, 3, 13, 21, 1, 1),
    (128, 16, 1, 9, 40, 2, 1),
    (128, 8, 8, 6, 10, 1, 2),
    (128, 4, 3, 11, 7, 2, 1),
    (128, 2, 1, 12, 40, 1, 1),
    (1024, 32, 3, 7, 9, 1, 1),
    (1024, 256, 1, 12, 13, 2, 1),
    (2048, 32, 8, 3, 5, 1, 2),
]


@pytest.fixture(params=["bf16x3", "tf32x3", "tf32"])
def mode(request):
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(request.param)
    yield request.param
    tc.set_precision(prev)


def _data(C, groups, B, H, W, stride, dil, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g)
    # TF32-representable weights: the fp32 pack rounds to TF32 in mode 'tf32', so the target needs no extra rounding term
    w = em.rn_tf32(torch.randn(C, C // groups, 3, 3, generator=g) / (9 * C // groups) ** 0.5)
    Ho, Wo = (H + 2 * dil - 2 * dil - 1) // stride + 1, (W + 2 * dil - 2 * dil - 1) // stride + 1
    return g, x, w, Ho, Wo


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _case_id(c):
    return "C{}g{}b{}_{}x{}_s{}d{}".format(*c)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
@pytest.mark.parametrize("epilogue", ["plain", "bias_res_relu", "res_relu_register"])
def test_forward(mode, case, epilogue):
    from monodetr_b200 import tc
    C, groups, B, H, W, stride, dil = case
    g, x, w, Ho, Wo = _data(*case, seed=sum(case))
    bias = torch.randn(C, generator=g) if epilogue == "bias_res_relu" else None
    res = torch.randn(B, Ho, Wo, C, generator=g) if epilogue != "plain" else None
    relu = epilogue != "plain"

    def f(a, b):
        return _nhwc(F.conv2d(_nchw(a), b, stride=stride, padding=dil, dilation=dil, groups=groups))
    t, s = em.target(f, x, w, mode)
    epi = em.epi_mag(t, bias, res) if epilogue != "plain" else None
    if bias is not None:
        t = t + bias.double()
    if res is not None:
        t = t + res.double()
    if relu:
        t = t.clamp_min(0)

    xd = x.cuda()
    if epilogue == "res_relu_register":
        # a residual 8 bytes past a 16-byte boundary: TMA cannot describe it, the register epilogue runs (its paired
        # accesses need 8-byte alignment)
        buf = torch.empty(res.numel() + 2, device="cuda")
        rd = buf[2:].view(res.shape)
        rd.copy_(res)
    else:
        rd = None if res is None else res.cuda()
    y = tc.conv2d_forward(xd, w.cuda(), None if bias is None else bias.cuda(), rd, 3, 3, stride, dil, relu=relu, dilation=dil,
                          groups=groups)
    em.assert_gemm(f"grouped fprop {_case_id(case)} {epilogue}", y.cpu(), t, s, mode, epi)
    if epilogue == "res_relu_register":   # the TMA epilogue gives the same bits
        y2 = tc.conv2d_forward(xd, w.cuda(), None, res.cuda(), 3, 3, stride, dil, relu=True, dilation=dil, groups=groups)
        assert torch.equal(y, y2)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
@pytest.mark.parametrize("epilogue", ["plain", "res_mask", "res_mask_register"])
def test_dgrad(mode, case, epilogue):
    from monodetr_b200 import tc
    C, groups, B, H, W, stride, dil = case
    g, x, w, Ho, Wo = _data(*case, seed=sum(case) + 1)
    dy = torch.randn(B, Ho, Wo, C, generator=g)
    res = torch.randn(B, H, W, C, generator=g) if epilogue != "plain" else None
    mask = torch.randn(B, H, W, C, generator=g).clamp_min(0) if epilogue != "plain" else None

    def f(a, b):
        return _nhwc(torch.nn.grad.conv2d_input((B, C, H, W), b, _nchw(a), stride=stride, padding=dil, dilation=dil,
                                                groups=groups))
    t, s = em.target(f, dy, w, mode)
    epi = em.epi_mag(t, None, res) if res is not None else None
    if res is not None:
        t = (t + res.double()) * (mask > 0)
    if epilogue == "res_mask_register":
        buf = torch.empty(res.numel() + 2, device="cuda")
        rd = buf[2:].view(res.shape)
        rd.copy_(res)
    else:
        rd = None if res is None else res.cuda()
    md = None if mask is None else mask.cuda()
    dx = tc.conv2d_dgrad(dy.cuda(), w.cuda(), (B, H, W, C), rd, md, 3, 3, stride, dil, dilation=dil, groups=groups)
    em.assert_gemm(f"grouped dgrad {_case_id(case)} {epilogue}", dx.cpu(), t, s, mode, epi)
    if epilogue == "res_mask_register":
        dx2 = tc.conv2d_dgrad(dy.cuda(), w.cuda(), (B, H, W, C), res.cuda(), md, 3, 3, stride, dil, dilation=dil, groups=groups)
        assert torch.equal(dx, dx2)


@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_wgrad(mode, case):
    """The band-local gradient through unpack (its in-group entries) against the float64 target; rowscale and
    reproducibility."""
    from monodetr_b200 import _lib, tc
    C, groups, B, H, W, stride, dil = case
    g, x, w, Ho, Wo = _data(*case, seed=sum(case) + 2)
    dy = torch.randn(B, Ho, Wo, C, generator=g)

    def f(a, b):
        return torch.nn.grad.conv2d_weight(_nchw(b), (C, C // groups, 3, 3), _nchw(a), stride=stride, padding=dil, dilation=dil,
                                           groups=groups)
    t, s = em.target(f, dy, x, mode)
    dwb = tc.conv2d_wgrad(dy.cuda(), x.cuda(), None, 3, 3, stride, dil, dilation=dil, groups=groups)
    dw = tc.unpack_grouped_wgrads_multi([dwb], [groups])[0]
    em.assert_gemm(f"grouped wgrad {_case_id(case)}", dw.cpu(), t, s, mode)
    # rowscale (the FrozenBN fold): in reproducible mode one multiplication of each launch's finished sum
    sc = torch.rand(C, generator=g) + 0.5
    _lib.lib().mdb_set_deterministic(1)
    try:
        a = tc.conv2d_wgrad(dy.cuda(), x.cuda(), None, 3, 3, stride, dil, dilation=dil, groups=groups)
        b = tc.conv2d_wgrad(dy.cuda(), x.cuda(), sc.cuda(), 3, 3, stride, dil, dilation=dil, groups=groups)
        a2 = tc.conv2d_wgrad(dy.cuda(), x.cuda(), None, 3, 3, stride, dil, dilation=dil, groups=groups)
    finally:
        _lib.lib().mdb_set_deterministic(0)
    assert torch.equal(a, a2), "reproducible mode is not bit-identical run to run"
    if dil == 1:   # (a dilated gradient adds its lattice classes' scaled sums)
        assert torch.equal(b, a * sc.cuda().view(1, C, 1))


@pytest.mark.parametrize("case", [CASES[0], CASES[2], CASES[6]], ids=_case_id)
def test_batch_independent_and_reproducible(mode, case):
    from monodetr_b200 import tc
    C, groups, B, H, W, stride, dil = case
    g, x, w, Ho, Wo = _data(C, groups, 8, H, W, stride, dil, seed=7)
    dy = torch.randn(8, Ho, Wo, C, generator=g)
    xd, wd, dyd = x.cuda(), w.cuda(), dy.cuda()
    y8 = tc.conv2d_forward(xd, wd, None, None, 3, 3, stride, dil, dilation=dil, groups=groups)
    dx8 = tc.conv2d_dgrad(dyd, wd, (8, H, W, C), None, None, 3, 3, stride, dil, dilation=dil, groups=groups)
    assert torch.equal(y8, tc.conv2d_forward(xd, wd, None, None, 3, 3, stride, dil, dilation=dil, groups=groups))
    assert torch.equal(dx8, tc.conv2d_dgrad(dyd, wd, (8, H, W, C), None, None, 3, 3, stride, dil, dilation=dil, groups=groups))
    for lo, hi in ((0, 1), (2, 5), (5, 8)):
        assert torch.equal(y8[lo:hi], tc.conv2d_forward(xd[lo:hi].contiguous(), wd, None, None, 3, 3, stride, dil, dilation=dil,
                                                        groups=groups))
        assert torch.equal(dx8[lo:hi], tc.conv2d_dgrad(dyd[lo:hi].contiguous(), wd, (hi - lo, H, W, C), None, None, 3, 3, stride,
                                                       dil, dilation=dil, groups=groups))


@pytest.mark.parametrize("C,groups", [(128, 32), (256, 64), (1024, 32), (2048, 32)])
def test_pack_unpack_round_trip(mode, C, groups):
    """The band-local layouts against a block-diagonal expansion of the OIHW weight (scale folded), and unpack of a band-local
    tensor back to the in-group entries."""
    from monodetr_b200 import tc
    g = torch.Generator().manual_seed(C + groups)
    gc = C // groups
    w = torch.randn(C, gc, 3, 3, generator=g)
    sc = torch.rand(C, generator=g) + 0.5
    ws = w * sc.view(C, 1, 1, 1)
    dense = torch.zeros(C, C, 3, 3)
    for q in range(groups):
        dense[q * gc:(q + 1) * gc, q * gc:(q + 1) * gc] = ws[q * gc:(q + 1) * gc]
    # band-local [tap][row][128]: wf rows = output channels, wd rows = input channels
    bands = torch.arange(C).view(C, 1) // 128 * 128 + torch.arange(128).view(1, 128)
    want_f = torch.stack([dense.permute(2, 3, 0, 1).reshape(9, C, C)[t].gather(1, bands) for t in range(9)])
    want_d = torch.stack([dense.permute(2, 3, 1, 0).reshape(9, C, C)[t].gather(1, bands) for t in range(9)])
    gw = tc.pack_grouped_multi([w.cuda()], [sc.cuda()], [groups])[0]
    if mode == "bf16x3":
        assert gw.split and gw.wf.shape == (9, C, 4, 64)
        for got, want in ((gw.wf, want_f), (gw.wd, want_d)):
            got = got.cpu().float().view(9, C, 4, 2, 32)
            hi, lo = em.split(want, "bf16x3")
            assert torch.equal(got[:, :, :, 0].reshape(9, C, 128), hi)
            assert torch.equal(got[:, :, :, 1].reshape(9, C, 128), lo)
    else:
        assert not gw.split and gw.wf.shape == (9, C, 128)
        r = em.rn_tf32 if mode == "tf32" else (lambda v: v)
        assert torch.equal(gw.wf.cpu(), r(want_f))
        assert torch.equal(gw.wd.cpu(), r(want_d))
    # unpack: the in-group entries of a band-local gradient, as OIHW
    dwb = torch.randn(9, C, 128, generator=g)
    got = tc.unpack_grouped_wgrads_multi([dwb.cuda()], [groups])[0].cpu()
    full = torch.zeros(9, C, C)
    full.scatter_(2, bands.expand(9, C, 128), dwb)
    want = torch.stack([full[:, o, (o // gc) * gc:(o // gc + 1) * gc] for o in range(C)]).permute(0, 2, 1).reshape(C, gc, 3, 3)
    assert torch.equal(got, want)


def test_multi_tensor_pack_spans_launches():
    """More than 64 grouped weights in one call (two launches), mixed widths and groups: each the same as packed alone."""
    from monodetr_b200 import tc
    g = torch.Generator().manual_seed(3)
    specs = [(128 << (i % 3), (32, 8, 64)[i % 3]) for i in range(70)]
    ws = [torch.randn(C, C // q, 3, 3, generator=g).cuda() for C, q in specs]
    many = tc.pack_grouped_multi(ws, None, [q for _, q in specs])
    for (C, q), w, gw in zip(specs, ws, many):
        one = tc.pack_grouped_multi([w], None, [q])[0]
        assert torch.equal(gw.wf, one.wf) and torch.equal(gw.wd, one.wd)


@pytest.mark.parametrize("C,groups,stride,dil", [(96, 32, 1, 1), (384, 2, 1, 1), (256, 3, 1, 1), (256, 32, 2, 2)])
def test_unsupported_geometry_raises(C, groups, stride, dil):
    from monodetr_b200 import tc
    x = torch.zeros(1, 8, 8, C, device="cuda")
    w = torch.zeros(C, C // groups, 3, 3, device="cuda")
    with pytest.raises((RuntimeError, AssertionError)):
        tc.conv2d_forward(x, w, None, None, 3, 3, stride, dil, dilation=dil, groups=groups)
