"""The software-pipelined consumer loop of the tensor-core GEMM (csrc/conv_gemm.cu): k-block i's wgmmas run while k-block
i+1 is loaded into the other of two fragment buffers (and, for the weight gradient and the TF32 modes, the other of two B
operand tile sets), and a ring stage is released one k-block after it is issued.  Held to the fp64 bounds of
tests/tc_error_model.py at the pipeline's edges: 1 to 7 k-blocks per tile (around every instance's ring depth, 3 to 6
stages), ring positions that wrap inside and across tiles of a persistent walk, tiles with no k-block (a stride-2 dgrad
parity class no tap reaches), weight-gradient splits whose last split is short, and the same results bit for bit on a
repeated call."""
import pytest
import torch

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


@pytest.mark.parametrize("kb", [1, 2, 3, 4, 5, 6, 7])
@pytest.mark.parametrize("N", [64, 256])
def test_linear_kblocks(mode, kb, N):
    """K = 32 * kb (the last k-block ragged for kb > 1) on 700 rows: fewer tiles than SMs, one tile per CTA.  Forward with
    bias + residual + ReLU and dgrad with a mask, both tile widths (BN = 64 and 128 instances)."""
    from monodetr_b200 import tc
    M, K = 700, 32 * kb - (4 if kb > 1 else 0)
    g = _gen(100 * kb + N)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(M, N, device="cuda", generator=g)
    t, s = em.target(lambda a, c: a @ c.t(), x, w, mode)
    y = tc.linear_forward(x, w, b, r, relu=True)
    em.assert_gemm(f"linear K={K} N={N}", y, torch.relu(t + b.double() + r.double()), s, mode, epi=em.epi_mag(t, b, r))
    assert torch.equal(y, tc.linear_forward(x, w, b, r, relu=True))

    # dgrad: N / 32 k-blocks, K output channels
    dy = torch.randn(M, N, device="cuda", generator=g)
    mask = torch.randn(M, K, device="cuda", generator=g)
    gate = (mask > 0).double()
    t, s = em.target(lambda a, c: a @ c, dy, w, mode)
    dx = tc.linear_dgrad(dy, w, None, mask)
    em.assert_gemm(f"dgrad K={K} N={N}", dx, t * gate, s * gate, mode)


@pytest.mark.parametrize("K", [96, 160, 288])
def test_persistent_walk_ring_wrap(mode, K):
    """81 600 rows x 256 (1 276 tiles, ~10 per CTA) with 3, 5 or 9 k-blocks per tile: the ring position carried from tile
    to tile wraps in the middle of tiles, at every phase of every ring depth."""
    from monodetr_b200 import tc
    M, N = 81600, 256
    g = _gen(K)
    x = torch.randn(M, K, device="cuda", generator=g)
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    t, s = em.target(lambda a, c: a @ c.t(), x, w, mode)
    y = tc.linear_forward(x, w)
    em.assert_gemm(f"linear M={M} K={K}", y, t, s, mode, epi=em.epi_mag(t))
    assert torch.equal(y, tc.linear_forward(x, w))


@pytest.mark.parametrize("cfg", [(3, 10, 14, 68, 132, 3, 1, 1), (2, 9, 11, 68, 132, 1, 2, 0), (2, 13, 11, 36, 64, 3, 2, 1)])
def test_conv_taps_and_empty_classes(mode, cfg):
    """3x3 convs (9 taps x up to 3 channel blocks per tile) and dgrads; the 1x1 stride-2 dgrad has parity classes with no
    tap, whose tiles have no k-block: their result is the epilogue of an exact zero (residual * mask)."""
    from monodetr_b200 import tc
    import torch.nn.functional as F
    B, H, W, Cin, Cout, k, st, pad = cfg
    g = _gen(sum(cfg))
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, k, k, device="cuda", generator=g) / (Cin * k * k) ** 0.5
    wop, wp = _operand(mode, w), _pack(w)

    def conv_f(a, c):
        taps, O, I = c.shape
        return F.conv2d(a.permute(0, 3, 1, 2), c.view(k, k, O, I).permute(2, 3, 0, 1), stride=st, padding=pad).permute(0, 2, 3, 1)

    def dgrad_f(a, c):
        taps, O, I = c.shape
        return torch.nn.grad.conv2d_input((B, Cin, H, W), c.view(k, k, O, I).permute(2, 3, 0, 1), a.permute(0, 3, 1, 2),
                                          stride=st, padding=pad).permute(0, 2, 3, 1)

    t, s = em.target(conv_f, x, wp, mode)
    y = tc.conv2d_forward(x, wop, None, None, k, k, st, pad)
    em.assert_gemm(f"fwd {cfg}", y, t, s, mode, epi=em.epi_mag(t))
    dy = torch.randn(t.shape, device="cuda", generator=g)
    r = torch.randn(x.shape, device="cuda", generator=g)
    mask = torch.randn(x.shape, device="cuda", generator=g)
    gate = (mask > 0).double()
    t, s = em.target(dgrad_f, dy, wp, mode)
    dx = tc.conv2d_dgrad(dy, wop, x.shape, r, mask, k, k, st, pad)
    em.assert_gemm(f"dgrad {cfg}", dx, (t + r.double()) * gate, s * gate, mode, epi=em.epi_mag(t, None, r) * gate,
                   exact_zero=(r * (mask > 0)).to(dx.dtype))
    assert torch.equal(dx, tc.conv2d_dgrad(dy, wop, x.shape, r, mask, k, k, st, pad))


@pytest.mark.parametrize("M", [4400, 4417, 20400])
def test_wgrad_short_last_split(mode, M):
    """Pointwise weight gradient 256 x 256 over M rows: 138, 139 or 638 reduction steps of 32 rows, split so that the last
    split is shorter than the others (and, at M = 4417, ends in a partial reduction tile); in the reproducible mode one
    split, twice bit for bit."""
    import monodetr_b200
    from monodetr_b200 import _lib
    N = 256
    g = _gen(M)
    dy = torch.randn(M, N, device="cuda", generator=g)
    x = torch.randn(M, N, device="cuda", generator=g)
    t, s = em.target(lambda a, b: (a.t() @ b).unsqueeze(0), dy, x, mode)
    for det in (False, True):
        prev = monodetr_b200.set_deterministic(det)
        try:
            outs = []
            for _ in range(2 if det else 1):
                dw = torch.full((1, N, N), float("nan"), device="cuda")
                _lib.call("mdb_conv2d_wgrad_f32", dy, x, None, dw, 1, 1, M, N, N, 1, 1, 1, 0, 0)
                torch.cuda.synchronize()
                outs.append(dw)
        finally:
            monodetr_b200.set_deterministic(prev)
        em.assert_gemm(f"wgrad M={M} reproducible={det}", outs[0], t, s, mode, epi=t.abs())
        if det:
            assert torch.equal(outs[0], outs[1])
