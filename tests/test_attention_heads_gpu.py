"""The fused attention core (csrc/attention.cu) at head widths 16 and 64 (nheads 16 and 4 at d_model 256) against a float64
softmax(Q K^T / sqrt(d)) V with autograd, per element with the bounds of tests/tc_error_model.py, as
tests/test_attention_error_model_gpu.py holds width 32: tails in Lq and Lk, the four mask kinds, a batch with every key
masked, peaked logits whose row maximum arrives in a later key tile, the model's packed q / kv views, H = 1, 4 and 16,
dropout keep rate and same-seed bits, batch-independent and run-to-run identical outputs, and the widths the kernels refuse."""
import pytest
import torch

import tc_error_model as em

pytestmark = pytest.mark.gpu

F64 = torch.float64
WIDTHS = [16, 64]


def _heads(t, H, hd):
    B, L, _ = t.shape
    return t.reshape(B, L, H, hd).transpose(1, 2)


def _ref(q, k, v, kpm, dout, H):
    """float64 reference with autograd; a row whose keys are all masked gets p = 0 (the kernel's documented result)."""
    B, Lq, E = q.shape
    hd = E // H
    qr, kr, vr = (t.detach().to(F64).requires_grad_(True) for t in (q, k, v))
    s = _heads(qr, H, hd) @ _heads(kr, H, hd).transpose(-1, -2) / hd ** 0.5
    if kpm is not None:
        s = s.masked_fill(kpm[:, None, None, :], float("-inf"))
    m = s.detach().amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    vh = _heads(vr, H, hd)
    o = p @ vh
    dof = _heads(dout.to(F64), H, hd)
    o.backward(dof)
    P = p.detach()
    scale = hd ** -0.5
    fwd_mag = P @ vh.detach().abs()
    delta = (dof * o.detach()).sum(-1, keepdim=True)
    dp_mag = dof.abs() @ vh.detach().abs().transpose(-1, -2)
    ds_mag = P * (dp_mag + delta.abs())
    dq_mag = scale * ds_mag @ _heads(kr.detach(), H, hd).abs()
    dk_mag = scale * ds_mag.transpose(-1, -2) @ _heads(qr.detach(), H, hd).abs()
    dv_mag = P.transpose(-1, -2) @ dof.abs()
    back = lambda t: t.transpose(1, 2).reshape(B, t.shape[2], E)
    return (back(o.detach()), qr.grad, kr.grad, vr.grad,
            back(fwd_mag), back(dq_mag), back(dk_mag), back(dv_mag))


def _check(name, q, k, v, kpm, dout, H):
    from monodetr_b200 import kernels as K
    out, lse, kp = K.attention_forward(q, k, v, kpm, heads=H)
    dq, dk, dv = K.attention_backward(q, k, v, kp, out, lse, dout, heads=H)
    o, gq, gk, gv, mo, mq, mk, mv = _ref(q, k, v, kpm, dout, H)
    em.assert_rel(name + " out", out, o, mo, em.C_ATT_FWD)
    em.assert_rel(name + " dq", dq, gq, mq, em.C_ATT_BWD)
    em.assert_rel(name + " dk", dk, gk, mk, em.C_ATT_BWD)
    em.assert_rel(name + " dv", dv, gv, mv, em.C_ATT_BWD)
    return out, lse, dq, dk, dv


def _mask(kind, B, Lk, g):
    if kind == "none":
        return None
    if kind == "random":
        return torch.rand(B, Lk, device="cuda", generator=g) < 0.2
    m = torch.zeros(B, Lk, dtype=torch.bool, device="cuda")
    if kind == "first tile":
        m[:, :min(64, Lk - 1)] = True
    elif kind == "last key only":
        m[:, :-1] = True
    return m


SHAPES = [(1, 1), (1, 1920), (63, 65), (65, 63), (129, 64), (129, 1920), (1920, 65)]


@pytest.mark.parametrize("hd", WIDTHS)
@pytest.mark.parametrize("Lq,Lk", SHAPES)
@pytest.mark.parametrize("H", [1, 4, 16])
@pytest.mark.parametrize("mask", ["none", "random", "first tile", "last key only"])
def test_attention_error_model(hd, Lq, Lk, H, mask):
    if H * hd > 256:
        pytest.skip("the model's widths: E <= 256")
    if Lq * Lk > 129 * 1920 // 2 and mask not in ("none", "random"):
        pytest.skip("one large case per mask kind is enough")
    B = 2
    g = torch.Generator(device="cuda").manual_seed(Lq * 7 + Lk + H + hd)
    E = hd * H
    q = torch.randn(B, Lq, E, device="cuda", generator=g)
    k = torch.randn(B, Lk, E, device="cuda", generator=g)
    v = torch.randn(B, Lk, E, device="cuda", generator=g)
    dout = torch.randn(B, Lq, E, device="cuda", generator=g)
    _check(f"attn hd={hd} Lq={Lq} Lk={Lk} H={H} mask={mask}", q, k, v, _mask(mask, B, Lk, g), dout, H)


@pytest.mark.parametrize("hd", WIDTHS)
def test_attention_model_shapes(hd):
    """The model's three call shapes at width 256: the depth cross-attention (550 x 1920, train), the grouped
    self-attention (88 x (50 x 50)) and the depth encoder's self-attention shape (1920 x 1920, here at cfg heads)."""
    H = 256 // hd
    for B, Lq, Lk in ((2, 550, 1920), (88, 50, 50), (1, 1920, 1920)):
        g = torch.Generator(device="cuda").manual_seed(B + Lq + Lk + hd)
        q, dout = (torch.randn(B, Lq, 256, device="cuda", generator=g) for _ in range(2))
        k, v = (torch.randn(B, Lk, 256, device="cuda", generator=g) for _ in range(2))
        _check(f"attn hd={hd} {B}x{Lq}x{Lk}", q, k, v, None, dout, H)


@pytest.mark.parametrize("hd", WIDTHS)
@pytest.mark.parametrize("peak", [25.0, 4.0])
def test_attention_peaked_logits_rescale(hd, peak):
    """Each row's maximum logit sits in a later key tile than the first: the online-softmax rescale."""
    Lq, Lk = 129, 1920
    H = 256 // hd
    g = torch.Generator(device="cuda").manual_seed(Lq + Lk + int(peak) + hd)
    B = 2
    q = torch.randn(B, Lq, 256, device="cuda", generator=g)
    k = torch.randn(B, Lk, 256, device="cuda", generator=g) * 0.5
    v = torch.randn(B, Lk, 256, device="cuda", generator=g)
    dout = torch.randn(B, Lq, 256, device="cuda", generator=g)
    for i in range(Lq):
        j = 64 + (i * 7) % (Lk - 64)
        qi = q[:, i].view(B, H, hd)
        k[:, j] = (qi * (peak * hd ** 0.5 / (qi * qi).sum(-1, keepdim=True))).view(B, 256)
    s = (_heads(q, H, hd) @ _heads(k, H, hd).transpose(-1, -2)) / hd ** 0.5
    assert float(s.abs().max()) > 0.8 * peak            # (at width 16 unrelated q . k products can exceed the peak)
    assert bool((s.argmax(-1) >= 64).float().mean() > 0.9)
    _check(f"attn hd={hd} peaked {peak}", q, k, v, None, dout, H)


@pytest.mark.parametrize("hd", WIDTHS)
def test_attention_packed_views_forward_backward(hd):
    """The model's calls: q from a 768-wide buffer, k and v from a 512-wide kv buffer (token strides 768 / 512), bit-equal
    to contiguous copies."""
    from monodetr_b200 import kernels as K
    H = 256 // hd
    g = torch.Generator(device="cuda").manual_seed(768 + hd)
    qkv = torch.randn(2, 100, 768, device="cuda", generator=g)
    kv = torch.randn(2, 129, 512, device="cuda", generator=g)
    q, k, v = qkv[..., :256], kv[..., :256], kv[..., 256:]
    kpm = torch.rand(2, 129, device="cuda", generator=g) < 0.2
    dout = torch.randn(2, 100, 256, device="cuda", generator=g)
    _check(f"attn hd={hd} packed views", q, k, v, kpm, dout, H)
    out, lse, kp = K.attention_forward(q, k, v, kpm, heads=H)
    got = K.attention_backward(q, k, v, kp, out, lse, dout, heads=H)
    qc, kc, vc = q.contiguous(), k.contiguous(), v.contiguous()
    out_c, lse_c, kp_c = K.attention_forward(qc, kc, vc, kpm, heads=H)
    assert torch.equal(out, out_c) and torch.equal(lse, lse_c)
    for a, b in zip(got, K.attention_backward(qc, kc, vc, kp_c, out_c, lse_c, dout, heads=H)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("hd", WIDTHS)
def test_attention_fully_masked_batch_and_bits(hd):
    """Every key of batch 1 masked: output rows 0, lse -inf, no gradient; the other batches finite, bit-equal when run
    alone, and two runs give the same bits."""
    from monodetr_b200 import kernels as K
    H = 256 // hd
    g = torch.Generator(device="cuda").manual_seed(5 + hd)
    B, Lq, Lk = 3, 65, 129
    q, dout = (torch.randn(B, Lq, 256, device="cuda", generator=g) for _ in range(2))
    k, v = (torch.randn(B, Lk, 256, device="cuda", generator=g) for _ in range(2))
    kpm = torch.rand(B, Lk, device="cuda", generator=g) < 0.2
    kpm[1] = True
    out, lse, dq, dk, dv = _check(f"attn hd={hd} fully masked batch", q, k, v, kpm, dout, H)
    assert bool((out[1] == 0).all()) and bool((lse[1] == float("-inf")).all())
    assert bool((dq[1] == 0).all()) and bool((dk[1] == 0).all()) and bool((dv[1] == 0).all())
    for t in (out, dq, dk, dv):
        assert bool(torch.isfinite(t).all())
    assert bool(torch.isfinite(lse[[0, 2]]).all())
    keep = [0, 2]
    sq, sk, sv, sd = (t[keep].contiguous() for t in (q, k, v, dout))
    so, sl, skp = K.attention_forward(sq, sk, sv, kpm[keep], heads=H)
    assert torch.equal(so, out[keep]) and torch.equal(sl, lse[keep])
    for a, b in zip(K.attention_backward(sq, sk, sv, skp, so, sl, sd, heads=H), (dq, dk, dv)):
        assert torch.equal(a, b[keep])
    o2, l2, kp2 = K.attention_forward(q, k, v, kpm, heads=H)
    assert torch.equal(o2, out) and torch.equal(l2, lse)
    for a, b in zip(K.attention_backward(q, k, v, kp2, o2, l2, dout, heads=H), (dq, dk, dv)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("hd", WIDTHS)
def test_attention_dropout_statistics_and_determinism(hd):
    """Keep rate 1 - p (E[mask / (1 - p)] = 1 under uniform attention), same seed and site -> same bits, another site ->
    another mask; the backward regenerates the forward's mask (<dO, O(V)> == <dV, V>)."""
    from monodetr_b200 import kernels as K
    H = 256 // hd
    g = torch.Generator(device="cuda").manual_seed(4 + hd)
    q = torch.zeros(1, 64, 256, device="cuda")
    k = torch.randn(1, 2000, 256, device="cuda", generator=g)
    v = torch.ones(1, 2000, 256, device="cuda")
    o1, lse, _ = K.attention_forward(q, k, v, drop_p=0.1, site=5, heads=H)
    o2, _, _ = K.attention_forward(q, k, v, drop_p=0.1, site=5, heads=H)
    assert torch.equal(o1, o2)
    assert abs(float(o1.mean()) - 1.0) < 0.02
    assert float(o1.std()) > 1e-3
    o3, _, _ = K.attention_forward(q, k, v, drop_p=0.1, site=6, heads=H)
    assert not torch.equal(o1, o3)
    dout = torch.randn(o1.shape, device="cuda", generator=g)
    dq, dk, dv = K.attention_backward(q, k, v, None, o1, lse, dout, drop_p=0.1, site=5, heads=H)
    lhs = float((dout.double() * o1.double()).sum()); rhs = float((dv.double() * v.double()).sum())
    scale = float((dout.double() * o1.double()).abs().sum())
    assert abs(lhs - rhs) < 1.5e-5 * scale, (lhs, rhs, scale)
    # the mask of a head does not depend on its width: one head of width 32 and one of width hd share the key (b*H + h = 0)
    o32, _, _ = K.attention_forward(q[..., :32].contiguous(), k[..., :32].contiguous(), v[..., :32].contiguous(), drop_p=0.1,
                                    site=5, heads=1)
    ohd, _, _ = K.attention_forward(q[..., :hd].contiguous(), k[..., :hd].contiguous(), v[..., :hd].contiguous(), drop_p=0.1,
                                    site=5, heads=1)
    assert float((o32[..., 0] - ohd[..., 0]).abs().max()) < 1e-5       # another mask would differ by ~1e-2


@pytest.mark.parametrize("hd", [8, 48, 128])
def test_unsupported_head_widths_raise(hd):
    from monodetr_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(hd)
    q, k, v = (torch.randn(1, 65, 2 * hd, device="cuda", generator=g) for _ in range(3))
    with pytest.raises(RuntimeError, match="mdb_attention_forward_f32"):
        K.attention_forward(q, k, v, heads=2)
    with pytest.raises(RuntimeError, match="mdb_attention_backward_f32"):
        K.attention_backward(q, k, v, None, torch.zeros_like(q), torch.zeros(1, 2, 65, device="cuda"), q, heads=2)
    with pytest.raises(ValueError, match="do not divide"):
        K.attention_forward(q, k, v, heads=3 if hd != 48 else 5)
