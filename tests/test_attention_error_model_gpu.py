"""The fused attention core (csrc/attention.cu) against a float64 softmax(Q K^T / sqrt(32)) V with autograd, per element
(tests/tc_error_model.py): the forward (3xTF32) relative to sum_j p_ij |v_jd|, the backward (single-pass TF32 gradient
contractions) relative to the float64 magnitudes of the same contractions.  Cases: tails in Lq and Lk, a fully masked
first key tile, a lone live key in a partial tile, a batch with every key masked, peaked logits whose row maximum
arrives in a later key tile (the online-softmax rescale), and the model's packed q / kv views in forward and backward."""
import pytest
import torch

import tc_error_model as em

pytestmark = pytest.mark.gpu

F64 = torch.float64


def _heads(t, H):
    B, L, _ = t.shape
    return t.reshape(B, L, H, 32).transpose(1, 2)


def _ref(q, k, v, kpm, dout):
    """float64 reference with autograd; a row whose keys are all masked gets p = 0 (the kernel's documented result)."""
    B, Lq, E = q.shape
    H = E // 32
    qr, kr, vr = (t.detach().to(F64).requires_grad_(True) for t in (q, k, v))
    s = _heads(qr, H) @ _heads(kr, H).transpose(-1, -2) / 32 ** 0.5
    if kpm is not None:
        s = s.masked_fill(kpm[:, None, None, :], float("-inf"))
    m = s.detach().amax(-1, keepdim=True)
    m = torch.where(torch.isinf(m), torch.zeros_like(m), m)
    e = torch.exp(s - m)
    l = e.sum(-1, keepdim=True)
    p = e / torch.where(l > 0, l, torch.ones_like(l))
    vh = _heads(vr, H)
    o = p @ vh
    dof = _heads(dout.to(F64), H)
    o.backward(dof)
    P = p.detach()
    # magnitudes of the contractions the kernels compute
    scale = 32 ** -0.5
    fwd_mag = P @ vh.detach().abs()
    delta = (dof * o.detach()).sum(-1, keepdim=True)
    dp_mag = dof.abs() @ vh.detach().abs().transpose(-1, -2)
    ds_mag = P * (dp_mag + delta.abs())
    dq_mag = scale * ds_mag @ _heads(kr.detach(), H).abs()
    dk_mag = scale * ds_mag.transpose(-1, -2) @ _heads(qr.detach(), H).abs()
    dv_mag = P.transpose(-1, -2) @ dof.abs()
    back = lambda t: t.transpose(1, 2).reshape(B, t.shape[2], E)
    return (back(o.detach()), qr.grad, kr.grad, vr.grad,
            back(fwd_mag), back(dq_mag), back(dk_mag), back(dv_mag))


def _check(name, q, k, v, kpm, dout):
    from monodetr_b200 import kernels as K
    out, lse, kp = K.attention_forward(q, k, v, kpm)
    dq, dk, dv = K.attention_backward(q, k, v, kp, out, lse, dout)
    o, gq, gk, gv, mo, mq, mk, mv = _ref(q, k, v, kpm, dout)
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


SHAPES = [(1, 1), (1, 1920), (63, 65), (65, 63), (64, 129), (129, 64), (129, 1920), (1920, 65), (65, 129), (1920, 1920)]


@pytest.mark.parametrize("Lq,Lk", SHAPES)
@pytest.mark.parametrize("H", [1, 8])
@pytest.mark.parametrize("mask", ["none", "random", "first tile", "last key only"])
def test_attention_error_model(Lq, Lk, H, mask):
    if (Lq, Lk) == (1920, 1920) and (H == 1 or mask not in ("none", "random")):
        pytest.skip("one large case per mask kind is enough")
    B = 2
    g = torch.Generator(device="cuda").manual_seed(Lq * 7 + Lk + H)
    E = 32 * H
    q = torch.randn(B, Lq, E, device="cuda", generator=g)
    k = torch.randn(B, Lk, E, device="cuda", generator=g)
    v = torch.randn(B, Lk, E, device="cuda", generator=g)
    dout = torch.randn(B, Lq, E, device="cuda", generator=g)
    _check(f"attn Lq={Lq} Lk={Lk} H={H} mask={mask}", q, k, v, _mask(mask, B, Lk, g), dout)


def test_attention_grouped_self_attention():
    """The decoder's grouped self-attention: Lq = Lk = 50 at batch 88."""
    g = torch.Generator(device="cuda").manual_seed(88)
    q, k, v, dout = (torch.randn(88, 50, 256, device="cuda", generator=g) for _ in range(4))
    _check("attn 88x50x50", q, k, v, None, dout)


@pytest.mark.parametrize("Lq,Lk", [(129, 1920), (65, 129)])
@pytest.mark.parametrize("peak", [25.0, 4.0])
def test_attention_peaked_logits_rescale(Lq, Lk, peak):
    """Each row's maximum logit (25: max |s| ~ 25; 4: a dominant key whose probability is not 1) sits in a later key tile
    than the first: the running maximum jumps and the accumulated tile is rescaled by exp(m_old - m_new) < 1."""
    g = torch.Generator(device="cuda").manual_seed(Lq + Lk + int(peak))
    B, H = 2, 8
    q = torch.randn(B, Lq, 256, device="cuda", generator=g)
    k = torch.randn(B, Lk, 256, device="cuda", generator=g) * 0.5
    v = torch.randn(B, Lk, 256, device="cuda", generator=g)
    dout = torch.randn(B, Lq, 256, device="cuda", generator=g)
    for i in range(Lq):
        j = 64 + (i * 7) % (Lk - 64)
        qi = q[:, i].view(B, H, 32)
        k[:, j] = (qi * (peak * 32 ** 0.5 / (qi * qi).sum(-1, keepdim=True))).view(B, 256)
    s = (_heads(q, H) @ _heads(k, H).transpose(-1, -2)) / 32 ** 0.5
    assert 0.8 * peak < float(s.abs().max()) < 1.6 * peak
    assert bool((s.argmax(-1) >= 64).float().mean() > 0.9)
    _check(f"attn peaked {peak} Lq={Lq} Lk={Lk}", q, k, v, None, dout)


def test_attention_packed_views_forward_backward():
    """The model's calls: q from a 768-wide qkv buffer, k and v from a 512-wide kv buffer (token strides 768 / 512)."""
    g = torch.Generator(device="cuda").manual_seed(768)
    qkv = torch.randn(2, 100, 768, device="cuda", generator=g)
    kv = torch.randn(2, 129, 512, device="cuda", generator=g)
    q, k, v = qkv[..., :256], kv[..., :256], kv[..., 256:]
    kpm = torch.rand(2, 129, device="cuda", generator=g) < 0.2
    dout = torch.randn(2, 100, 256, device="cuda", generator=g)
    _check("attn packed views", q, k, v, kpm, dout)
    from monodetr_b200 import kernels as K
    out, lse, kp = K.attention_forward(q, k, v, kpm)
    got = K.attention_backward(q, k, v, kp, out, lse, dout)
    qc, kc, vc = q.contiguous(), k.contiguous(), v.contiguous()
    out_c, lse_c, kp_c = K.attention_forward(qc, kc, vc, kpm)
    assert torch.equal(out, out_c) and torch.equal(lse, lse_c)
    for a, b in zip(got, K.attention_backward(qc, kc, vc, kp_c, out_c, lse_c, dout)):
        assert torch.equal(a, b)


def test_attention_fully_masked_batch():
    """Every key of batch 1 masked: its output rows are 0 and lse = -inf, its gradients are 0, and the other batches are
    unaffected and finite (torch's MHA gives NaN for such rows)."""
    from monodetr_b200 import kernels as K
    g = torch.Generator(device="cuda").manual_seed(5)
    B, Lq, Lk = 3, 65, 129
    q, dout = (torch.randn(B, Lq, 256, device="cuda", generator=g) for _ in range(2))
    k, v = (torch.randn(B, Lk, 256, device="cuda", generator=g) for _ in range(2))
    kpm = torch.rand(B, Lk, device="cuda", generator=g) < 0.2
    kpm[1] = True
    out, lse, dq, dk, dv = _check("attn fully masked batch", q, k, v, kpm, dout)
    assert bool((out[1] == 0).all()) and bool((lse[1] == float("-inf")).all())
    assert bool((dq[1] == 0).all()) and bool((dk[1] == 0).all()) and bool((dv[1] == 0).all())
    for t in (out, dq, dk, dv):
        assert bool(torch.isfinite(t).all())
    assert bool(torch.isfinite(lse[[0, 2]]).all())
    keep = [0, 2]
    solo = K.attention_forward(q[keep].contiguous(), k[keep].contiguous(), v[keep].contiguous(), kpm[keep])
    assert torch.equal(solo[0], out[keep])
