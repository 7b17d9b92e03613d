"""GPU numerics of the fused attention core and the LayerNorm / GroupNorm kernels against plain PyTorch fp32
references of the same ops.  Tolerance 1e-4 relative to max|ref| (pure fp32 kernels; __expf in softmax)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-20))


def _ref_attn(q, k, v, kpm):
    B, Lq, E = q.shape
    H = E // 32
    qh = q.view(B, Lq, H, 32).transpose(1, 2)
    kh = k.view(B, -1, H, 32).transpose(1, 2)
    vh = v.view(B, -1, H, 32).transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) / 32 ** 0.5
    if kpm is not None:
        s = s.masked_fill(kpm[:, None, None, :], float("-inf"))
    return (torch.softmax(s, -1) @ vh).transpose(1, 2).reshape(B, Lq, E)


@pytest.mark.parametrize("B,Lq,Lk,mask", [(2, 50, 1920, False), (2, 550, 1920, True), (3, 50, 50, False), (1, 1920, 1920, False),
                                           (2, 37, 101, True)])
def test_attention_forward_backward(B, Lq, Lk, mask):
    from monodetr_b200 import kernels as K
    torch.backends.cuda.matmul.allow_tf32 = False
    g = torch.Generator(device="cuda").manual_seed(Lq + Lk)
    q = torch.randn(B, Lq, 256, device="cuda", generator=g)
    k = torch.randn(B, Lk, 256, device="cuda", generator=g)
    v = torch.randn(B, Lk, 256, device="cuda", generator=g)
    kpm = (torch.rand(B, Lk, device="cuda", generator=g) < 0.2) if mask else None
    dout = torch.randn(B, Lq, 256, device="cuda", generator=g)
    out, lse, kp = K.attention_forward(q, k, v, kpm)
    qr, kr, vr = (t.clone().requires_grad_(True) for t in (q, k, v))
    ref = _ref_attn(qr, kr, vr, kpm)
    ref.backward(dout)
    assert _rel(out, ref.detach()) < 1e-4
    dq, dk, dv = K.attention_backward(q, k, v, kp, out, lse, dout)
    # gradient contractions are single-pass TF32 (round-to-nearest operands); the scores they use are 3xTF32
    assert _rel(dq, qr.grad) < 2e-3
    assert _rel(dk, kr.grad) < 2e-3
    assert _rel(dv, vr.grad) < 2e-3


def test_attention_packed_strided_inputs():
    from monodetr_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(3)
    qkv = torch.randn(2, 100, 768, device="cuda", generator=g)
    q, k, v = qkv[..., :256], qkv[..., 256:512], qkv[..., 512:]
    out, _, _ = K.attention_forward(q, k, v)
    assert _rel(out, _ref_attn(q.contiguous(), k.contiguous(), v.contiguous(), None)) < 1e-4


def test_attention_dropout_statistics_and_determinism():
    from monodetr_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(4)
    q = torch.zeros(1, 64, 256, device="cuda")            # uniform attention
    k = torch.randn(1, 2000, 256, device="cuda", generator=g)
    v = torch.ones(1, 2000, 256, device="cuda")
    o1, lse, _ = K.attention_forward(q, k, v, drop_p=0.1, site=5)
    o2, _, _ = K.attention_forward(q, k, v, drop_p=0.1, site=5)
    assert torch.equal(o1, o2)                            # same seed -> same mask
    assert abs(float(o1.mean()) - 1.0) < 0.02             # E[mask/(1-p)] = 1
    assert float(o1.std()) > 1e-3                         # masks differ per (i, h)
    o3, _, _ = K.attention_forward(q, k, v, drop_p=0.1, site=6)
    assert not torch.equal(o1, o3)                        # another site -> another mask
    # gradient consistency under dropout: O is linear in V, so <dO, O(V)> == <dV, V> when backward regenerates the
    # SAME mask.  The tolerance is relative to sum|dO.O| (NOT to the cancelling sum): the contraction noise is
    # ~1e-6 of it; a fwd/bwd mask mismatch shows up as ~1e-4 of it (std 0.0105 per output x ||dO|| = 1.3 here).
    dout = torch.randn(o1.shape, device="cuda", generator=g)
    dq, dk, dv = K.attention_backward(q, k, v, None, o1, lse, dout, drop_p=0.1, site=5)
    lhs = float((dout.double() * o1.double()).sum()); rhs = float((dv.double() * v.double()).sum())
    scale = float((dout.double() * o1.double()).abs().sum())
    assert abs(lhs - rhs) < 1.5e-5 * scale, (lhs, rhs, scale)
    # backward with another site's mask gives a different dV (the masks really are regenerated per site)
    _, _, dv_bad = K.attention_backward(q, k, v, None, o1, lse, dout, drop_p=0.1, site=6)
    assert float((dv_bad - dv).abs().max()) > 1e-3


@pytest.mark.parametrize("M,C,with_res", [(1000, 256, True), (81600, 256, True), (333, 256, False), (77, 512, True), (64, 128, True),
                                          (1, 128, True), (7, 512, False)])
def test_add_layernorm(M, C, with_res):
    from monodetr_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(M)
    x = torch.randn(M, C, device="cuda", generator=g) * 2 + 0.5
    res = torch.randn(M, C, device="cuda", generator=g) if with_res else None
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g)
    dy = torch.randn(M, C, device="cuda", generator=g)
    y, mean, rstd = K.add_layernorm_forward(x, res, gamma, beta)
    xr = x.clone().requires_grad_(True)
    rr = res.clone().requires_grad_(True) if with_res else None
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ref = F.layer_norm(xr + rr if with_res else xr, (C,), gr, br, 1e-5)
    ref.backward(dy)
    assert _rel(y, ref.detach()) < 1e-5
    dx, dres, dg, db = K.add_layernorm_backward(dy, x, res, gamma, mean, rstd)
    assert _rel(dx, xr.grad) < 1e-4
    assert _rel(dg, gr.grad) < 1e-4 and _rel(db, br.grad) < 1e-4


def test_add_layernorm_dropout():
    from monodetr_b200 import kernels as K
    x = torch.zeros(4096, 256, device="cuda")
    res = torch.ones(4096, 256, device="cuda")
    gamma = torch.ones(256, device="cuda"); beta = torch.zeros(256, device="cuda")
    y, mean, rstd = K.add_layernorm_forward(x, res, gamma, beta, drop_p=0.1, site=9)
    # z = mask/(1-p): mean of z per row ~ 1, and exactly the two values {0, 1/0.9}
    assert abs(float(mean.mean()) - 1.0) < 0.01
    dy = torch.randn_like(x)
    dx, dres, _, _ = K.add_layernorm_backward(dy, x, res, gamma, mean, rstd, drop_p=0.1, site=9)
    keep = (y > y.min(dim=1, keepdim=True).values + 1e-6)          # kept entries have the larger normalised value
    assert torch.allclose(dres, dx * keep / 0.9, atol=1e-6)
    assert 0.88 < float(keep.float().mean()) < 0.92


@pytest.mark.parametrize("B,HW,C,relu", [(2, 1920, 256, False), (2, 1920, 256, True), (3, 7680, 256, False), (2, 120, 256, True), (1, 77, 64, False),
                                         (9, 257, 512, True), (2, 1, 1024, False)])
def test_groupnorm(B, HW, C, relu):
    from monodetr_b200 import kernels as K
    G = 32 if C >= 256 else 8
    g = torch.Generator(device="cuda").manual_seed(HW + C)
    x = torch.randn(B, HW, C, device="cuda", generator=g) * 3 + 1
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g)
    dy = torch.randn(B, HW, C, device="cuda", generator=g)
    y, mean, rstd = K.groupnorm_forward(x, gamma, beta, G, 1e-5, relu)
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    ref = F.group_norm(xr.transpose(1, 2), G, gr, br, 1e-5).transpose(1, 2)
    if relu:
        ref = torch.relu(ref)
    ref.backward(dy)
    assert _rel(y, ref.detach()) < 1e-5
    dx, dg, db = K.groupnorm_backward(dy, x, y, gamma, mean, rstd, G, relu)
    assert _rel(dx, xr.grad) < 1e-4
    assert _rel(dg, gr.grad) < 1e-4 and _rel(db, br.grad) < 1e-4
