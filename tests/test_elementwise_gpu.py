"""GPU unit parity of the small kernels around the tensor-core GEMMs, each against a plain PyTorch fp32 restatement of
the reference expression it replaces:
  * frozen ResNet stem: conv1 7x7/2 + FrozenBatchNorm2d affine + ReLU (backbone.py:54-64,100-102) and torchvision's
    maxpool(3, 2, 1);
  * MSDeformAttn pre-processing: softmax over the 16 (level, point) logits and the sampling-location arithmetic for 2-d
    and 6-d reference points (ops/modules/ms_deform_attn.py:145-155), forward and backward incl. the box gradient;
  * hash dropout: determinism, keep statistics, site / seed decorrelation, forward/backward mask identity, and the
    per-forward seed snapshot (kernels.begin_forward);
  * column sums (bias gradients) at ragged sizes.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


@pytest.mark.parametrize("B,H,W", [(2, 384, 1280), (1, 96, 320), (3, 50, 70), (1, 37, 41)])
def test_stem_conv_bn_relu_and_maxpool(B, H, W):
    from monodetr_b200 import _lib, tc
    torch.backends.cudnn.allow_tf32 = False
    prev = tc.get_precision()
    tc.set_precision("tf32x3")                # ('tf32' mode additionally rounds the stem output to TF32 for its consumer)
    try:
        g = torch.Generator(device="cuda").manual_seed(H + W)
        x = torch.randn(B, 3, H, W, device="cuda", generator=g)
        w = torch.randn(64, 3, 7, 7, device="cuda", generator=g) / 147 ** 0.5
        scale = torch.rand(64, device="cuda", generator=g) + 0.5
        shift = torch.randn(64, device="cuda", generator=g)
        H1, W1 = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        y = torch.empty(B, H1, W1, 64, device="cuda")
        _lib.call("mdb_stem_conv7x7_bn_relu_f32", x, w, scale, shift, y, B, H, W)
        ref = torch.relu(F.conv2d(x, w, None, stride=2, padding=3) * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1))
        assert _rel(y.permute(0, 3, 1, 2), ref) < 1e-5          # plain fp32 CUDA-core kernel
        H2, W2 = (H1 + 2 - 3) // 2 + 1, (W1 + 2 - 3) // 2 + 1
        p = torch.empty(B, H2, W2, 64, device="cuda")
        _lib.call("mdb_maxpool3x3s2_nhwc_f32", y, p, B, H1, W1, 64)
        assert torch.equal(p.permute(0, 3, 1, 2), F.max_pool2d(y.permute(0, 3, 1, 2), 3, 2, 1))   # exact: a selection
    finally:
        tc.set_precision(prev)


def _ref_prep(off, logits, ref, shapes, M, L, P):
    """ops/modules/ms_deform_attn.py:145-155 restated."""
    B, Lq = off.shape[:2]
    off = off.view(B, Lq, M, L, P, 2)
    attn = torch.softmax(logits.view(B, Lq, M, L * P), -1).view(B, Lq, M, L, P)
    if ref.shape[-1] == 2:
        norm = torch.stack((shapes[..., 1], shapes[..., 0]), -1).to(off.dtype)
        loc = ref[:, :, None, :, None, :] + off / norm[None, None, None, :, None, :]
    else:
        loc = ref[:, :, None, :, None, :2] + off / P * (ref[:, :, None, :, None, 2::2] + ref[:, :, None, :, None, 3::2]) * 0.5
    return loc, attn


@pytest.mark.parametrize("B,Lq,rd", [(2, 53, 2), (1, 10200, 2), (2, 550, 6), (3, 1, 6), (1, 77, 2)])
def test_msda_prep_forward_backward(B, Lq, rd):
    from monodetr_b200 import functional as Fn
    M, L, P = 8, 4, 4
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + Lq + rd)
    shapes = torch.as_tensor([(48, 160), (24, 80), (12, 40), (6, 20)], dtype=torch.long, device="cuda")
    off = (torch.randn(B, Lq, M * L * P * 2, device="cuda", generator=g) * 2).requires_grad_()
    logits = torch.randn(B, Lq, M * L * P, device="cuda", generator=g).requires_grad_()
    ref = torch.rand(B, Lq, L, rd, device="cuda", generator=g).requires_grad_()
    dloc = torch.randn(B, Lq, M, L, P, 2, device="cuda", generator=g)
    dattn = torch.randn(B, Lq, M, L, P, device="cuda", generator=g)
    loc, attn = Fn.msda_prep(off, logits, ref, shapes, M, L, P)
    go, gl, gr = torch.autograd.grad((loc, attn), (off, logits, ref), (dloc, dattn))
    o2, l2, r2 = (t.detach().clone().requires_grad_() for t in (off, logits, ref))
    rloc, rattn = _ref_prep(o2, l2, r2, shapes, M, L, P)
    ro, rl, rr = torch.autograd.grad((rloc, rattn), (o2, l2, r2), (dloc, dattn))
    assert _rel(loc, rloc) < 1e-6 and _rel(attn, rattn) < 1e-5
    assert _rel(go, ro) < 1e-5 and _rel(gl, rl) < 1e-4
    assert _rel(gr, rr) < 1e-4                                  # incl. the 6-d box gradient (cx, cy, l, r, t, b)


def test_dropout_determinism_statistics_and_seed_snapshot():
    from monodetr_b200 import functional as Fn, kernels as K
    dev = torch.device("cuda", torch.cuda.current_device())
    K.reseed(dev, 1234)
    x = torch.ones(1 << 20, device="cuda", requires_grad=True)
    a = Fn.dropout(x, 0.1, True, 7)
    b = Fn.dropout(x, 0.1, True, 7)
    c = Fn.dropout(x, 0.1, True, 8)
    assert torch.equal(a, b)                                     # same seed, same site -> same mask
    assert not torch.equal(a, c)                                 # another site -> another mask
    keep = (a > 0).float().mean().item()
    assert abs(keep - 0.9) < 2e-3                                # 1M Bernoulli(0.9) draws: sigma = 3e-4
    assert torch.allclose(a[a > 0], torch.full_like(a[a > 0], 1 / 0.9))
    assert abs(float(((a > 0) & (c > 0)).float().mean()) - 0.81) < 3e-3     # sites are independent
    # forward/backward mask identity survives a NEW forward (and a seed advance) in between: the mask belongs to the
    # snapshot taken when its forward ran, not to the live seed
    K.begin_forward(dev)
    y1 = Fn.dropout(x, 0.1, True, 7)
    K.begin_forward(dev)
    y2 = Fn.dropout(x, 0.1, True, 7)
    assert not torch.equal(y1, y2)                               # masks change from step to step
    (g1,) = torch.autograd.grad(y1.sum(), x)
    assert torch.equal(g1, y1.detach())                          # d/dx sum(mask/(1-p) * x) = mask/(1-p) = y1 (x = 1)
    K.reseed(dev, 1234)
    assert torch.equal(Fn.dropout(x, 0.1, True, 7), a)           # reseed reproduces the run
    assert Fn.dropout(x, 0.1, False, 7) is x and Fn.dropout(x, 0.0, True, 7) is x


@pytest.mark.parametrize("M,N", [(1, 4), (77, 3), (4400, 81), (81600, 256), (1000, 1025)])
def test_colsum_ragged(M, N):
    from monodetr_b200 import tc
    g = torch.Generator(device="cuda").manual_seed(M + N)
    x = torch.randn(M, N, device="cuda", generator=g)
    ref = x.double().sum(0).float()
    assert float((tc.colsum(x) - ref).abs().max()) < 1e-5 * max(1.0, float(x.abs().sum(0).max()))
