"""The tensor-core GEMM family (csrc/conv_gemm.cu) held per element to its documented arithmetic (tests/tc_error_model.py):
the float64 sum of the products of the split operands, plus fp32 accumulation and the epilogue's rounding, at the tile
edges where such kernels go wrong -- k-block tails, the 64/128 tile-width switch, odd widths with the scalar epilogue,
the persistent walk, dgrad parity classes without pixels or taps, wgrad split-K, the forward split-K path -- and the
promise of include/monodetr_b200.h that an image's bits do not depend on the batch it is in.

The measured worst ratios and the constants derived from them are in tests/tc_error_model.py."""
import pytest
import torch
import torch.nn.functional as F

import tc_error_model as em

pytestmark = pytest.mark.gpu

MODES = ["bf16x3", "tf32x3", "tf32"]
F64 = torch.float64


@pytest.fixture(params=MODES)
def mode(request):
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(request.param)
    yield request.param
    tc.set_precision(prev)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _mm(a, b):                      # y = a b^T
    return a @ b.t()


def _zero_rows(x, every=7):
    """Zero a few rows so that some outputs have S == 0 and must come out as the exact epilogue."""
    x = x.clone()
    x[::every] = 0
    return x


def _epilogue32(n, bias, res, relu):
    """The fp32 epilogue of an exact zero accumulator, as the kernel computes it."""
    z = torch.zeros(n, device="cuda")
    if bias is not None:
        z = z + bias
    if res is not None:
        z = z + res
    return torch.relu(z) if relu else z


# ---- linear forward -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("K", [4, 36, 100, 260])
@pytest.mark.parametrize("N", [1, 3, 5, 63, 64, 65, 127, 128, 129, 200])
def test_linear_forward_edges(mode, N, K):
    from monodetr_b200 import tc
    for M in (1, 127, 129):
        g = _gen(M * 1000 + N * 10 + K)
        x = _zero_rows(torch.randn(M, K, device="cuda", generator=g))
        w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        b = torch.randn(N, device="cuda", generator=g)
        r = torch.randn(M, N, device="cuda", generator=g)
        t, s = em.target(_mm, x, w, mode)
        y = tc.linear_forward(x, w)
        em.assert_gemm(f"linear M={M} N={N} K={K}", y, t, s, mode, exact_zero=torch.zeros((), device="cuda"))
        y = tc.linear_forward(x, w, b, r, relu=True)
        pre = t + b.double() + r.double()
        em.assert_gemm(f"linear+b+r+relu M={M} N={N} K={K}", y, torch.relu(pre), s, mode, epi=em.epi_mag(t, b, r),
                       exact_zero=_epilogue32((M, N), b, r, True))


@pytest.mark.parametrize("K", [96, 160])
def test_linear_forward_persistent_walk(mode, K):
    """1276 tiles on 132 SMs, k-blocks per tile (3 or 5) not a multiple of the ring depth: stage / phase bookkeeping
    across tiles."""
    from monodetr_b200 import tc
    M, N = 81601, 256
    g = _gen(K)
    x = _zero_rows(torch.randn(M, K, device="cuda", generator=g), 1001)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    t, s = em.target(_mm, x, w, mode)
    y = tc.linear_forward(x, w, b)
    em.assert_gemm(f"linear M={M} K={K}", y, t + b.double(), s, mode, epi=em.epi_mag(t, b), exact_zero=_epilogue32((M, N), b, None, False))


# ---- linear dgrad / wgrad -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cout", [4, 36])
@pytest.mark.parametrize("Cin", [64, 68, 128, 132])
def test_linear_dgrad_edges(mode, Cin, Cout):
    """Reduction over Cout (one partial k-block), output width at the bf path's bn = 64 / 128 switch; residual + a
    relu_mask holding exact +0.0 and -0.0 (both gate)."""
    from monodetr_b200 import tc
    M = 333
    g = _gen(Cin * 100 + Cout)
    dy = _zero_rows(torch.randn(M, Cout, device="cuda", generator=g), 5)
    w = torch.randn(Cout, Cin, device="cuda", generator=g) / Cout ** 0.5
    res = torch.randn(M, Cin, device="cuda", generator=g)
    mask = torch.randn(M, Cin, device="cuda", generator=g)
    mask[:, ::5] = 0.0
    mask[:, 1::5] = -0.0
    t, s = em.target(lambda a, b: a @ b, dy, w, mode)
    dx = tc.linear_dgrad(dy, w)
    em.assert_gemm(f"dgrad Cin={Cin} Cout={Cout}", dx, t, s, mode, exact_zero=torch.zeros((), device="cuda"))
    dx = tc.linear_dgrad(dy, w, residual=res, relu_mask=mask)
    gate = (mask > 0).double()
    em.assert_gemm(f"dgrad+res+mask Cin={Cin} Cout={Cout}", dx, (t + res.double()) * gate, s * gate, mode,
                   epi=em.epi_mag(t, None, res) * gate, exact_zero=res * (mask > 0))
    assert bool((dx[mask <= 0] == 0).all())


def test_linear_dgrad_padded_dy(mode):
    """dy wider than the weight (O = 81 padded to 84 with zero columns, as functional._Linear.backward does): the SplitW
    keeps O = 81 and its k-block padding; fp32 weights get zero rows."""
    from monodetr_b200 import tc
    M, O, Op, K = 550, 81, 84, 256
    g = _gen(81)
    w = torch.randn(O, K, device="cuda", generator=g) / O ** 0.5
    dy = F.pad(torch.randn(M, O, device="cuda", generator=g), (0, Op - O))
    wop = tc.split_weights([w])[0] if mode == "bf16x3" else F.pad(w, (0, 0, 0, Op - O))
    t, s = em.target(lambda a, b: a @ b, dy[:, :O], w, mode)
    dx = tc.linear_dgrad(dy, wop)
    em.assert_gemm("dgrad O=81 Op=84", dx, t, s, mode)


def _wgrad_splits(M, N, K, sms):
    """Restatement of mdb_conv2d_wgrad_bias_f32's split count for a linear layer: (raw split count, reduction tiles)."""
    total_red = (M + 31) // 32
    tiles = ((N + 127) // 128) * ((K + 127) // 128)
    big = min((2 * sms + tiles - 1) // tiles, total_red // 24)
    small = min(sms // tiles, total_red // 8)
    return max(big, small, 1), total_red


@pytest.mark.parametrize("M,N,K", [(4400, 256, 256), (4400, 128, 68), (1000, 36, 32), (81600, 256, 256), (31, 4, 4)])
def test_linear_wgrad_splits(mode, M, N, K):
    """Split-K weight gradient, in the default and the reproducible (one split) mode, both held to the same bound.  The
    two M = 4400 shapes have a raw split count (17 splits of 9 steps over 138) whose last split would be empty; the
    launcher then runs 16 splits."""
    import monodetr_b200
    from monodetr_b200 import tc
    g = _gen(M + N + K)
    dy = torch.randn(M, N, device="cuda", generator=g)
    x = torch.randn(M, K, device="cuda", generator=g)
    splits, total_red = _wgrad_splits(M, N, K, torch.cuda.get_device_properties(0).multi_processor_count)
    rps = -(-total_red // splits)
    print(f"M={M}: {splits} raw splits of {rps} steps over {total_red}; last raw split empty: {rps * (splits - 1) >= total_red}")
    t, s = em.target(lambda a, b: a.t() @ b, dy, x, mode)
    dw = tc.linear_wgrad(dy, x)
    em.assert_gemm(f"wgrad M={M} N={N} K={K}", dw, t, s, mode)
    prev = monodetr_b200.set_deterministic(True)
    try:
        dw1 = tc.linear_wgrad(dy, x)
    finally:
        monodetr_b200.set_deterministic(prev)
    em.assert_gemm(f"wgrad reproducible M={M} N={N} K={K}", dw1, t, s, mode)


# ---- convolutions ------------------------------------------------------------------------------------------------------
def _pack(w):
    O, I, kh, kw = w.shape
    return w.permute(2, 3, 0, 1).reshape(kh * kw, O, I).contiguous()


def _conv_f(k, stride, pad):
    def f(a, b):                    # a: NHWC, b: packed (taps, O, I) -> NHWC
        taps, O, I = b.shape
        w = b.view(k, k, O, I).permute(2, 3, 0, 1)
        return F.conv2d(a.permute(0, 3, 1, 2), w, stride=stride, padding=pad).permute(0, 2, 3, 1)
    return f


def _dgrad_f(shape, k, stride, pad):
    def f(a, b):                    # a: dy NHWC, b: packed weights -> dx NHWC
        taps, O, I = b.shape
        w = b.view(k, k, O, I).permute(2, 3, 0, 1)
        B, H, W, C = shape
        return torch.nn.grad.conv2d_input((B, C, H, W), w, a.permute(0, 3, 1, 2), stride=stride, padding=pad).permute(0, 2, 3, 1)
    return f


def _wgrad_f(k, stride, pad):
    def f(a, b):                    # a: dy NHWC, b: x NHWC -> packed dw
        O, I = a.shape[-1], b.shape[-1]
        dw = torch.nn.grad.conv2d_weight(b.permute(0, 3, 1, 2), (O, I, k, k), a.permute(0, 3, 1, 2), stride=stride, padding=pad)
        return _pack(dw)
    return f


def _weights(mode, w, scale):
    """The operand the model passes: bf16x3 splits straight from the OIHW parameter with the FrozenBN scale folded in fp32;
    the other modes take the fp32 packed fold."""
    from monodetr_b200 import tc
    ws = w * scale.view(-1, 1, 1, 1)
    return (tc.split_weights([w], [scale])[0] if mode == "bf16x3" else _pack(ws)), _pack(ws)


CONV_EDGES = [
    # B, H, W, Cin, Cout, k, stride, pad
    (2, 1, 1, 36, 64, 3, 1, 1),
    (2, 1, 1, 36, 68, 3, 2, 1),
    (2, 2, 2, 100, 65, 3, 2, 1),
    (3, 3, 3, 4, 129, 3, 1, 1),
    (2, 3, 2, 68, 36, 3, 2, 1),
    (2, 7, 9, 260, 128, 3, 2, 1),
    (2, 7, 1, 32, 64, 3, 2, 1),
    (3, 6, 20, 64, 64, 3, 1, 1),            # B not a multiple of the image-spanning tile's tb
    (5, 6, 20, 100, 132, 3, 1, 1),
    (5, 6, 20, 256, 256, 3, 2, 1),
    (2, 13, 21, 32, 64, 3, 2, 1),            # odd H, W: wgrad reduction tiles start outside the image
    (2, 9, 11, 68, 132, 1, 2, 0),            # 1x1 stride 2: dgrad classes no tap reaches
]


@pytest.mark.parametrize("cfg", CONV_EDGES)
def test_conv_edges(mode, cfg):
    from monodetr_b200 import tc
    B, H, W, Cin, Cout, k, st, pad = cfg
    g = _gen(sum(cfg) * 31 + Cin)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    x[-1] = 0                                                        # last image: S == 0 everywhere
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
    bias = torch.randn(Cout, device="cuda", generator=g)
    wop, wp = _weights(mode, w, scale)
    name = f"conv {cfg}"
    # forward, with bias + residual + ReLU (odd Cout: scalar epilogue)
    t, s = em.target(_conv_f(k, st, pad), x, wp, mode)
    res = torch.randn(t.shape, device="cuda", generator=g)
    y = tc.conv2d_forward(x, wop, bias, None, k, k, st, pad)
    em.assert_gemm(name + " fwd+b", y, t + bias.double(), s, mode, epi=em.epi_mag(t, bias),
                   exact_zero=_epilogue32(y.shape, bias, None, False))
    y = tc.conv2d_forward(x, wop, bias, res, k, k, st, pad, relu=True)
    em.assert_gemm(name + " fwd+b+r+relu", y, torch.relu(t + bias.double() + res.double()), s, mode, epi=em.epi_mag(t, bias, res),
                   exact_zero=_epilogue32(y.shape, bias, res, True))
    if Cout % 4:
        return                                                       # dgrad / wgrad need 16-byte pitches of dy
    # dgrad over every parity class, with residual + mask
    dy = torch.randn(t.shape, device="cuda", generator=g)
    dy[-1] = 0
    t, s = em.target(_dgrad_f(x.shape, k, st, pad), dy, wp, mode)
    dx = tc.conv2d_dgrad(dy, wop, x.shape, None, None, k, k, st, pad)
    em.assert_gemm(name + " dgrad", dx, t, s, mode, exact_zero=torch.zeros((), device="cuda"))
    r2 = torch.randn(x.shape, device="cuda", generator=g)
    mask = torch.randn(x.shape, device="cuda", generator=g)
    gate = (mask > 0).double()
    dx = tc.conv2d_dgrad(dy, wop, x.shape, r2, mask, k, k, st, pad)
    em.assert_gemm(name + " dgrad+res+mask", dx, (t + r2.double()) * gate, s * gate, mode, epi=em.epi_mag(t, None, r2) * gate,
                   exact_zero=r2 * (mask > 0))
    # wgrad with the FrozenBN row scale (rowscale multiplies the accumulator once)
    x = torch.randn(x.shape, device="cuda", generator=g)
    t, s = em.target(_wgrad_f(k, st, pad), dy, x, mode)
    sc = scale.double().view(1, -1, 1)
    dw = tc.conv2d_wgrad(dy, x, scale, k, k, st, pad)
    em.assert_gemm(name + " wgrad*rowscale", dw, t * sc, s * sc, mode, epi=t.abs() * sc)


# ---- forward split-K next to the unsplit path -----------------------------------------------------------------------------
@pytest.mark.parametrize("Cin", [2048, 928])
@pytest.mark.parametrize("bias_kind", ["none", "aligned", "offset"])
def test_forward_splitk_and_unsplit_same_bound(mode, Cin, bias_kind):
    """The neck conv (3x3 stride 2 on 12x40, 576 k-blocks: 18 slices) and Cin = 928 (261 k-blocks: the last of 9 slices
    holds 5).  A bias at a 4-byte offset takes the unsplit path; both paths meet the same bound."""
    from monodetr_b200 import _lib, tc
    B, H, W, Cout, k, st, pad = 2, 12, 40, 256, 3, 2, 1
    g = _gen(Cin + len(bias_kind))
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
    store = torch.randn(Cout + 4, device="cuda", generator=g)
    bias = None if bias_kind == "none" else (store[:Cout] if bias_kind == "aligned" else store[1:Cout + 1])
    wop, wp = _weights(mode, w, scale)
    need = _lib.lib().mdb_conv2d_forward_workspace_bytes(B, H, W, Cin, Cout, k, k, st, pad, 0, 0, int(mode == "bf16x3"))
    slices = need // (4 * B * 6 * 20 * Cout)
    assert slices == (0 if mode == "tf32" else -(-(k * k * -(-Cin // 32)) // 32))
    t, s = em.target(_conv_f(k, st, pad), x, wp, mode)
    y = tc.conv2d_forward(x, wop, bias, None, k, k, st, pad)
    ref = t if bias is None else t + bias.double()
    em.assert_gemm(f"neck Cin={Cin} bias={bias_kind} ({'split' if slices and bias_kind != 'offset' else 'unsplit'})", y, ref, s, mode,
                   epi=em.epi_mag(t, bias))


# ---- batch invariance ------------------------------------------------------------------------------------------------------
BATCH_CLASSES = {
    # name: (H, W, Cin, Cout, k, stride, pad, relu, bias)
    "backbone 1x1 s1": (24, 80, 64, 256, 1, 1, 0, True, True),
    "backbone 3x3 s1": (24, 80, 64, 64, 3, 1, 1, True, True),
    "backbone 1x1 s2": (24, 80, 256, 512, 1, 2, 0, False, True),
    "backbone 3x3 s2": (24, 80, 128, 128, 3, 2, 1, True, True),
    "input_proj 1x1": (12, 40, 2048, 256, 1, 1, 0, False, True),
    "input_proj 3x3 s2": (12, 40, 2048, 256, 3, 2, 1, False, True),
    "depth predictor 3x3": (24, 80, 256, 256, 3, 1, 1, False, True),
    "depth predictor 1x1": (24, 80, 256, 256, 1, 1, 0, False, True),
}
LINEAR_CLASSES = {
    # name: (tokens per image, K, N)
    "encoder ffn": (1280, 256, 1024),
    "encoder ffn out": (1280, 1024, 256),
    "decoder qkv": (50, 256, 768),
}
BATCHES = [2, 8, 32, 33, 40]


@pytest.mark.parametrize("cls", list(BATCH_CLASSES))
def test_conv_batch_invariance(mode, cls):
    """Image 0 alone and inside batches of 2..40 gives the same forward and dgrad bits, and the forward scratch size is
    linear in the batch."""
    from monodetr_b200 import _lib, tc
    H, W, Cin, Cout, k, st, pad, relu, has_b = BATCH_CLASSES[cls]
    g = _gen(Cin * 7 + Cout + k)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    bias = torch.randn(Cout, device="cuda", generator=g) if has_b else None
    wop, _ = _weights(mode, w, torch.ones(Cout, device="cuda"))
    Ho, Wo = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
    x0 = torch.randn(1, H, W, Cin, device="cuda", generator=g)
    dy0 = torch.randn(1, Ho, Wo, Cout, device="cuda", generator=g)
    y1 = tc.conv2d_forward(x0, wop, bias, None, k, k, st, pad, relu=relu)
    dx1 = tc.conv2d_dgrad(dy0, wop, x0.shape, None, None, k, k, st, pad)
    per_image = _lib.lib().mdb_conv2d_forward_workspace_bytes(1, H, W, Cin, Cout, k, k, st, pad, int(relu), 0, int(mode == "bf16x3"))
    bad = []
    for B in BATCHES:
        x = torch.cat((x0, torch.randn(B - 1, H, W, Cin, device="cuda", generator=g)))
        dy = torch.cat((dy0, torch.randn(B - 1, Ho, Wo, Cout, device="cuda", generator=g)))
        yB = tc.conv2d_forward(x, wop, bias, None, k, k, st, pad, relu=relu)
        dxB = tc.conv2d_dgrad(dy, wop, x.shape, None, None, k, k, st, pad)
        ws = _lib.lib().mdb_conv2d_forward_workspace_bytes(B, H, W, Cin, Cout, k, k, st, pad, int(relu), 0, int(mode == "bf16x3"))
        if not torch.equal(yB[:1], y1):
            bad.append(f"forward B={B}: max |diff| {float((yB[:1] - y1).abs().max()):.3e}")
        if not torch.equal(dxB[:1], dx1):
            bad.append(f"dgrad B={B}")
        if ws != B * per_image:
            bad.append(f"workspace B={B}: {ws} != {B} x {per_image}")
    assert not bad, f"{cls} [{mode}]: " + "; ".join(bad)


@pytest.mark.parametrize("cls", list(LINEAR_CLASSES))
def test_linear_batch_invariance(mode, cls):
    from monodetr_b200 import tc
    L, K, N = LINEAR_CLASSES[cls]
    g = _gen(L + K + N)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    wop = tc.split_weights([w])[0] if mode == "bf16x3" else w
    x0 = torch.randn(L, K, device="cuda", generator=g)
    dy0 = torch.randn(L, N, device="cuda", generator=g)
    y1 = tc.linear_forward(x0, wop, b)
    dx1 = tc.linear_dgrad(dy0, wop)
    for B in BATCHES:
        x = torch.cat((x0, torch.randn((B - 1) * L, K, device="cuda", generator=g)))
        dy = torch.cat((dy0, torch.randn((B - 1) * L, N, device="cuda", generator=g)))
        assert torch.equal(tc.linear_forward(x, wop, b)[:L], y1), f"{cls} [{mode}] forward B={B}"
        assert torch.equal(tc.linear_dgrad(dy, wop)[:L], dx1), f"{cls} [{mode}] dgrad B={B}"
