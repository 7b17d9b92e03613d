"""CPU: the HOST logic of the use_dab model -- the anchor / sine-embedding / query-position autograd functions, the shared-box
deformable attention (fused with box partials, or the two-step path in reproducible mode), the decoder's per-layer position
schedule -- driven end to end through the stand-in device library (tests/fake_device_lib.py), extended here by host
restatements of the use_dab entry points of include/monodetr_b200.h, and compared with the use_dab oracle (tests/oracle_dab.py,
pinned to the unmodified reference by tests/test_oracle_dab.py): train-mode outputs and the gradient of every parameter,
refpoint_embed and tgt_embed included, and the eval forward."""
import pytest
import torch

from oracle import monodetr_torch as om
from oracle.msda_torch import msda_core_torch
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import _grad, _prep, f32, i64
import oracle_dab as od          # tests/oracle_dab.py


def _qp_raw(raw, B, rows, C, shared):
    return f32(raw, rows, C) if shared else f32(raw, B, rows, C)


class DabFakeLib(fake_device_lib.FakeLib):
    """FakeLib plus the use_dab entry points, each restated with torch from the header's statement of what it computes
    (backward entry points through torch.autograd of the restatement)."""

    def mdb_dab_sine_embed_forward_f32(self, box, out, n, stream):
        f32(out, n, 768).copy_(od.gen_sineembed_for_position(f32(box, n, 6)[None])[0])
        return 0

    def mdb_dab_sine_embed_backward_f32(self, box, dout, dbox, n, stream):
        with torch.enable_grad():
            b = f32(box, n, 6).clone().requires_grad_()
            (g,) = _grad([od.gen_sineembed_for_position(b[None])[0]], [b], [f32(dout, n, 768)])
        f32(dbox, n, 6).copy_(g)
        return 0

    def mdb_dab_query_pos_forward_f32(self, scale, raw, out, B, rows, C, shared, stream):
        r = _qp_raw(raw, B, rows, C, shared).expand(B, rows, C)
        s = f32(scale, B, rows, C)
        f32(out, B, rows, C).copy_(r if s is None else s * r)
        return 0

    def mdb_dab_query_pos_backward_f32(self, dqp, scale, raw, dscale, draw, B, rows, C, shared, stream):
        g, s, r = f32(dqp, B, rows, C), f32(scale, B, rows, C), _qp_raw(raw, B, rows, C, shared)
        if dscale:
            f32(dscale, B, rows, C).copy_(g * r.expand(B, rows, C))
        if draw:
            d = g if s is None else g * s
            _qp_raw(draw, B, rows, C, shared).copy_(d.sum(0) if shared else d)
        return 0

    @staticmethod
    def _box_grad(sx, sy, wx, wy, P):
        return torch.stack((sx, sy, wx, wx, wy, wy), -1) * torch.tensor([1, 1, 0.5 / P, 0.5 / P, 0.5 / P, 0.5 / P])

    def mdb_msda_ref_grad_f32(self, dloc, off, B, Lq, M, L, P, shared, dref, stream):
        g, o = f32(dloc, B, Lq, M * L * P, 2), f32(off, B, Lq, M * L * P, 2)
        dims = (0, 2) if shared else (2,)
        d = self._box_grad(g[..., 0].sum(dims), g[..., 1].sum(dims), (g[..., 0] * o[..., 0]).sum(dims),
                           (g[..., 1] * o[..., 1]).sum(dims), P)
        f32(dref, *((Lq, 6) if shared else (B, Lq, 6))).copy_(d)
        return 0

    def mdb_msda_fused_backward_ref_f32(self, value, shapes, lsi, off, logits, ref, gout, B, S, M, D, L, Lq, P, rd, gv, goff, glog,
                                        part, stream):
        assert rd == 6
        self.mdb_msda_fused_backward_f32(value, shapes, lsi, off, logits, ref, gout, B, S, M, D, L, Lq, P, rd, gv, goff, glog, stream)
        sh = i64(shapes, L, 2)
        o = f32(off, B, Lq, M, L, P, 2)
        with torch.enable_grad():
            lo, at = _prep(o, f32(logits, B, Lq, M * L * P), f32(ref, B, Lq, L, rd), sh, M, L, P, rd)
            lo = lo.detach().requires_grad_()
            (gl,) = _grad([msda_core_torch(f32(value, B, S, M, D), sh, lo, at)], [lo], [f32(gout, B, Lq, M * D)])
        f32(part, B, Lq, M, L, 4).copy_(torch.stack((gl[..., 0].sum(-1), gl[..., 1].sum(-1), (gl[..., 0] * o[..., 0]).sum(-1),
                                                     (gl[..., 1] * o[..., 1]).sum(-1)), -1))
        return 0

    def mdb_msda_ref_partials_reduce_f32(self, part, B, Lq, M, L, P, shared, dref, stream):
        p = f32(part, B, Lq, M * L, 4)
        s = p.sum((0, 2)) if shared else p.sum(2)
        f32(dref, *((Lq, 6) if shared else (B, Lq, 6))).copy_(self._box_grad(s[..., 0], s[..., 1], s[..., 2], s[..., 3], P))
        return 0

    def mdb_dab_anchor_forward_f32(self, w, r, r2, rb, B, n, stream):
        s = f32(w, n).sigmoid()
        f32(r, n).copy_(s)
        f32(r2, n).copy_(s)
        f32(rb, B, n).copy_(s.expand(B, n))
        return 0

    def mdb_dab_anchor_backward_f32(self, r, d_sine, d_msda, d_head, B, n, dw, stream):
        acc = torch.zeros(n)
        for t in (f32(d_sine, n), f32(d_msda, n)):
            if t is not None:
                acc += t
        if d_head:
            acc += f32(d_head, B, n).sum(0)
        s = f32(r, n)
        f32(dw, n).copy_(acc * s * (1 - s))
        return 0


def _build(monkeypatch, precision):
    fake_device_lib.install(monkeypatch, {"tf32x3": 1, "bf16x3": 2}[precision])
    from monodetr_b200 import _lib, build_monodetr, tc
    fake = DabFakeLib({"tf32x3": 1, "bf16x3": 2}[precision])
    monkeypatch.setattr(_lib, "_lib", fake)
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    assert tc.get_precision() == precision
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, use_dab=True, dropout=0.0, device="cpu"))
    sd = od.deterministic_state_dict()
    m.load_state_dict(om.with_aliases(sd))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return fake, m, sd


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.mark.parametrize("precision,batch,deterministic", [("bf16x3", 1, False), ("tf32x3", 1, False), ("bf16x3", 2, True)])
def test_train_mode_forward_and_every_gradient_match_the_oracle(monkeypatch, precision, batch, deterministic):
    """Outputs within 1e-4 and every gradient with the bars of tests/test_model_host_logic.py; the anchors' gradient goes through
    the fused backward's box partials by default and through the two-step path's box reduction in reproducible mode."""
    from monodetr_b200.bench_model import surrogate_loss
    fake, m, sd = _build(monkeypatch, precision)
    fake.deterministic = int(deterministic)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(batch, 0, H=96, W=320)
    out = m(images, calibs, None, sizes)
    surrogate_loss(out).backward()

    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = od.forward(sdg, images, calibs, sizes, training=True)
    om.surrogate_loss(ref).backward()

    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, k
        assert _rel(out[k].detach(), ref[k].detach()) < 1e-4, (k, _rel(out[k].detach(), ref[k].detach()))
    for a, b in zip(out["aux_outputs"], ref["aux_outputs"]):
        for k in a:
            assert _rel(a[k].detach(), b[k].detach()) < 1e-4, ("aux", k)

    by_name = om.with_aliases(sdg)
    errs = []
    for name, p in m.named_parameters():
        want = by_name[name].grad
        if not p.requires_grad:
            assert p.grad is None, name
            continue
        if p.grad is None:
            assert want is None or not want.any(), name            # sa_v_proj, label_enc, query_scale_bbox
            continue
        assert want is not None, name
        errs.append((_rel(p.grad, want), name, float(want.abs().max())))
    errs.sort()
    print("gradient errors (max-norm relative, per tensor): median %.2e; worst:" % errs[len(errs) // 2][0], errs[-8:])
    assert len(errs) == 320                                         # every parameter the reference's DAB model gives a gradient
    names = {n for _, n, _ in errs}
    assert {"refpoint_embed.weight", "tgt_embed.weight", "depthaware_transformer.decoder.query_scale.layers.0.weight",
            "depthaware_transformer.decoder.ref_point_head.layers.0.weight"} <= names
    assert all(p.grad is None for p in m.depthaware_transformer.decoder.query_scale_bbox.parameters())
    med_bar, worst_bar = (1e-3, 1e-1) if precision == "bf16x3" else (3e-4, 3e-2)
    assert errs[len(errs) // 2][0] < med_bar, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < worst_bar or scale < 1e-6, (name, err, scale)
    # the anchors: a sum over all 550 queries' three contributions, held tighter than the worst-tensor bar
    assert _rel(m.refpoint_embed.weight.grad, sdg["refpoint_embed.weight"].grad) < (3e-2 if precision == "bf16x3" else 1e-2)

    calls = fake.calls
    for fn in ("mdb_dab_sine_embed_forward_f32", "mdb_dab_sine_embed_backward_f32", "mdb_dab_query_pos_forward_f32",
               "mdb_dab_query_pos_backward_f32", "mdb_dab_anchor_forward_f32", "mdb_dab_anchor_backward_f32"):
        assert calls.get(fn, 0) > 0, fn
    assert calls["mdb_dab_sine_embed_forward_f32"] == 3 and calls["mdb_dab_sine_embed_backward_f32"] == 1   # layer 0 only
    if deterministic:
        assert calls.get("mdb_msda_fused_backward_ref_f32", 0) == 0 and calls["mdb_msda_ref_grad_f32"] == 1
    else:
        assert calls["mdb_msda_fused_backward_ref_f32"] == 1 and calls["mdb_msda_ref_partials_reduce_f32"] == 1
        assert calls.get("mdb_msda_ref_grad_f32", 0) == 0


def test_eval_mode_forward_matches_the_oracle(monkeypatch):
    """Eval: the first 50 anchors, layer 0's deformable attention through the plain fused forward (no box gradient wanted)."""
    fake, m, sd = _build(monkeypatch, "tf32x3")
    m.eval()
    images, calibs, sizes = om.synthetic_inputs(2, 1, H=96, W=320)
    with torch.no_grad():
        out = m(images, calibs, None, sizes)
        ref = od.forward(sd, images, calibs, sizes, training=False)
    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, k
        assert _rel(out[k], ref[k]) < 1e-4, (k, _rel(out[k], ref[k]))
    assert fake.calls.get("mdb_msda_prep_forward_f32", 0) == 0 and fake.calls["mdb_msda_fused_forward_f32"] == 6
