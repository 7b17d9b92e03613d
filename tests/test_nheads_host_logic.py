"""CPU: the whole product model with the reference's other head counts (cfg `nheads` 4 and 16: head widths 64 and 16) through
the stand-in device library (tests/fake_device_lib.py), whose attention entry points are extended here to honour head_dim,
against the oracle (tests/oracle_nheads.py): outputs and every parameter gradient, in both GEMM precisions.  The decoder's
two attention cores must use cfg heads, the depth predictor's encoder 8, and the deformable attention (value width 64 / 16)
takes the separate-node encoder path and the two-step decoder path, in both modes."""
import ctypes
import math

import pytest
import torch

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import _buf, _grad, f32, u8
import oracle_nheads as on      # tests/oracle_nheads.py

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


def strided(ptr, B, L, H, hd, ld):
    """(B, L, H, hd) view of a token-strided buffer: token stride ld floats, batch stride L * ld."""
    n = (B * L - 1) * ld + H * hd
    return _buf(ptr, n, ctypes.c_float, torch.float32).as_strided((B, L, H, hd), (L * ld, ld, hd, 1))


class HeadsFakeLib(fake_device_lib.FakeLib):
    """FakeLib whose attention entry points take any head width the C ABI accepts (16, 32, 64) and log (H, head_dim)."""

    def __init__(self, precision):
        super().__init__(precision)
        self.attn_log = []

    def mdb_attention_forward_f32(self, q, k, v, kpm, out, lse, B, H, Lq, Lk, hd, ldq, ldk, ldv, ldo, drop_p, seed, site, stream):
        assert drop_p == 0.0 and hd in (16, 32, 64)
        self.attn_log.append((H, hd))
        o, l = self._attn(strided(q, B, Lq, H, hd, ldq), strided(k, B, Lk, H, hd, ldk), strided(v, B, Lk, H, hd, ldv),
                          u8(kpm, B, Lk))
        strided(out, B, Lq, H, hd, ldo).copy_(o)
        f32(lse, B, H, Lq).copy_(l)
        return 0

    def mdb_attention_backward_f32(self, q, k, v, kpm, out, lse, dout, ws, dq, dk, dv, B, H, Lq, Lk, hd, ldq, ldk, ldv, ldo, lddq,
                                   lddk, lddv, drop_p, seed, site, stream):
        assert drop_p == 0.0 and hd in (16, 32, 64)
        with torch.enable_grad():
            ins = [strided(p, B, L_, H, hd, ld).clone().requires_grad_() for p, L_, ld in ((q, Lq, ldq), (k, Lk, ldk),
                                                                                          (v, Lk, ldv))]
            o, _ = self._attn(*ins, u8(kpm, B, Lk))
            gq, gk, gv = _grad([o], ins, [strided(dout, B, Lq, H, hd, ldo)])
        strided(dq, B, Lq, H, hd, lddq).copy_(gq)
        strided(dk, B, Lk, H, hd, lddk).copy_(gk)
        strided(dv, B, Lk, H, hd, lddv).copy_(gv)
        return 0


def _build(monkeypatch, precision, nheads):
    fake_device_lib.install(monkeypatch, {"tf32x3": 1, "bf16x3": 2}[precision])
    from monodetr_b200 import _lib, build_monodetr, tc
    fake = HeadsFakeLib({"tf32x3": 1, "bf16x3": 2}[precision])
    monkeypatch.setattr(_lib, "_lib", fake)
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    assert tc.get_precision() == precision
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, nheads=nheads, dropout=0.0, device="cpu"))
    sd = on.deterministic_state_dict(on.heads_cfg(nheads))
    m.load_state_dict(om.with_aliases(sd))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return fake, m, sd


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def _check_outputs(out, ref):
    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, k
        assert _rel(out[k].detach(), ref[k].detach()) < 1e-4, (k, _rel(out[k].detach(), ref[k].detach()))
    for a, b in zip(out["aux_outputs"], ref["aux_outputs"]):
        for k in a:
            assert _rel(a[k].detach(), b[k].detach()) < 1e-4, ("aux", k)


@pytest.mark.parametrize("nheads", [4, 16])
@pytest.mark.parametrize("precision,deterministic", [("bf16x3", False), ("tf32x3", False), ("tf32x3", True)])
def test_train_mode_forward_and_every_gradient_match_the_oracle(monkeypatch, nheads, precision, deterministic):
    """Outputs within 1e-4 and every gradient with the bars of tests/test_model_host_logic.py."""
    from monodetr_b200.bench_model import surrogate_loss
    fake, m, sd = _build(monkeypatch, precision, nheads)
    fake.deterministic = int(deterministic)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    out = m(images, calibs, None, sizes)
    surrogate_loss(out).backward()

    cfg = on.heads_cfg(nheads)
    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = on.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
    om.surrogate_loss(ref).backward()
    _check_outputs(out, ref)

    by_name = om.with_aliases(sdg)
    errs = []
    for name, p in m.named_parameters():
        want = by_name[name].grad
        if not p.requires_grad:
            assert p.grad is None, name
            continue
        if p.grad is None:
            assert want is None or not want.any(), name            # sa_v_proj, label_enc
            continue
        assert want is not None, name
        errs.append((_rel(p.grad, want), name, float(want.abs().max())))
    errs.sort()
    print("gradient errors (max-norm relative, per tensor): median %.2e; worst:" % errs[len(errs) // 2][0], errs[-8:])
    med_bar, worst_bar = (1e-3, 1e-1) if precision == "bf16x3" else (3e-4, 3e-2)
    assert errs[len(errs) // 2][0] < med_bar, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < worst_bar or scale < 1e-6, (name, err, scale)

    # 3 decoder layers x (depth cross-attention + group self-attention) at cfg heads, one depth-encoder call at 8 (forward)
    hd = 256 // nheads
    assert sorted(fake.attn_log) == sorted([(8, 32)] + [(nheads, hd)] * 6), fake.attn_log
    calls = fake.calls
    assert calls.get("mdb_msda_fused_forward_f32", 0) == 0 and calls.get("mdb_msda_fused_backward_ref_f32", 0) == 0


@pytest.mark.parametrize("nheads", [4, 16])
def test_eval_mode_forward_matches_the_oracle(monkeypatch, nheads):
    fake, m, sd = _build(monkeypatch, "tf32x3", nheads)
    m.eval()
    images, calibs, sizes = om.synthetic_inputs(2, 1, H=96, W=320)
    with torch.no_grad():
        out = m(images, calibs, None, sizes)
        ref = on.forward(sd, images, calibs, sizes, training=False, cfg=on.heads_cfg(nheads))
    _check_outputs(out, ref)
    assert sorted(fake.attn_log) == sorted([(8, 32)] + [(nheads, 256 // nheads)] * 6), fake.attn_log


def test_eight_heads_oracle_is_the_base_oracle():
    """At nheads 8 the head-count oracle is om itself: same weights, same outputs bit for bit."""
    cfg = on.heads_cfg(8)
    sd = on.deterministic_state_dict(cfg)
    base = om.deterministic_state_dict()
    assert sd.keys() == base.keys() and all(torch.equal(sd[k], base[k]) for k in sd)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    with torch.no_grad():
        a = on.forward(sd, images, calibs, sizes, training=False, cfg=cfg)
        b = om.forward(base, images, calibs, sizes, training=False)
    for k in OUT_KEYS:
        assert torch.equal(a[k], b[k]), k
    assert math.isclose(float(om.surrogate_loss(a)), float(om.surrogate_loss(b)))
