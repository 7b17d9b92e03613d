"""CPU: the HOST logic of the learned position embedding (`position_embedding: 'learned'`) -- its autograd function, the four
levels' tables (the three backbone levels and the extra 1/64 level), the gradient from both consumers (the encoder's query path and
the depth predictor's encoder layer, which meet at level 1) -- driven end to end through the stand-in device library
(tests/fake_device_lib.py), extended here by host restatements of the two entry points of include/monodetr_b200.h, and compared
with the oracle (tests/oracle_learned_pos.py, pinned to the unmodified reference by tests/test_oracle_learned_pos.py): train-mode
outputs and the gradient of every parameter, both tables included, and the eval forward."""
import pytest
import torch

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import _grad, f32
import oracle_learned_pos as ol  # tests/oracle_learned_pos.py


class LearnedFakeLib(fake_device_lib.FakeLib):
    """FakeLib plus the learned-embedding entry points, restated with torch from the header's statement of what they compute
    (the backward through torch.autograd of the restatement)."""

    def mdb_pos_learned_forward_f32(self, col, row, H, W, out, stream):
        f32(out, H * W, 256).copy_(ol.table_nhwc(f32(col, 50, 128), f32(row, 50, 128), H, W))
        return 0

    def mdb_pos_learned_backward_f32(self, dpos, H, W, dcol, drow, stream):
        with torch.enable_grad():
            c = f32(dcol, 50, 128)
            col, row = torch.zeros(50, 128, requires_grad=True), torch.zeros(50, 128, requires_grad=True)
            gc, gr = _grad([ol.table_nhwc(col, row, H, W)], [col, row], [f32(dpos, H * W, 256)])
        c.copy_(gc)
        f32(drow, 50, 128).copy_(gr)
        return 0


def _build(monkeypatch, precision):
    fake_device_lib.install(monkeypatch, {"tf32x3": 1, "bf16x3": 2}[precision])
    from monodetr_b200 import _lib, build_monodetr, tc
    fake = LearnedFakeLib({"tf32x3": 1, "bf16x3": 2}[precision])
    monkeypatch.setattr(_lib, "_lib", fake)
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    assert tc.get_precision() == precision
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, position_embedding="learned", dropout=0.0, device="cpu"))
    sd = ol.with_tables(om.deterministic_state_dict())
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
    """Outputs within 1e-4 and every gradient with the bars of tests/test_dab_host_logic.py; both tables get their gradient from
    one backward launch per level."""
    from monodetr_b200.bench_model import surrogate_loss
    fake, m, sd = _build(monkeypatch, precision)
    fake.deterministic = int(deterministic)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(batch, 0, H=96, W=320)
    out = m(images, calibs, None, sizes)
    surrogate_loss(out).backward()

    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = ol.forward(sdg, images, calibs, sizes, training=True)
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
            assert want is None or not want.any(), name            # sa_v_proj, label_enc, query_scale, ref_point_head
            continue
        assert want is not None, name
        errs.append((_rel(p.grad, want), name, float(want.abs().max())))
    errs.sort()
    print("gradient errors (max-norm relative, per tensor): median %.2e; worst:" % errs[len(errs) // 2][0], errs[-8:])
    assert len(errs) == 315                                         # the default model's 313 and the two tables
    assert {ol.ROW, ol.COL} <= {n for _, n, _ in errs}
    med_bar, worst_bar = (1e-3, 1e-1) if precision == "bf16x3" else (3e-4, 3e-2)
    assert errs[len(errs) // 2][0] < med_bar, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < worst_bar or scale < 1e-6, (name, err, scale)
    for name in (ol.ROW, ol.COL):
        assert _rel(dict(m.named_parameters())[name].grad, sdg[name].grad) < (3e-2 if precision == "bf16x3" else 1e-2), name

    calls = fake.calls
    assert calls["mdb_pos_learned_forward_f32"] == 4 and calls["mdb_pos_learned_backward_f32"] == 4     # one per level each


def test_eval_mode_forward_matches_the_oracle(monkeypatch):
    """Eval under no_grad: one forward launch per level and no backward."""
    fake, m, sd = _build(monkeypatch, "tf32x3")
    m.eval()
    images, calibs, sizes = om.synthetic_inputs(2, 1, H=96, W=320)
    with torch.no_grad():
        out = m(images, calibs, None, sizes)
        ref = ol.forward(sd, images, calibs, sizes, training=False)
    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, k
        assert _rel(out[k], ref[k]) < 1e-4, (k, _rel(out[k], ref[k]))
    assert fake.calls["mdb_pos_learned_forward_f32"] == 4 and fake.calls.get("mdb_pos_learned_backward_f32", 0) == 0


def test_module_forward_and_backward_through_the_entry_points(monkeypatch):
    """The module alone at the fixture's shapes: the table is the oracle's exactly (the stand-in restates the same fp32
    operations), and one backward launch returns both tables' gradients, the oracle's within fp32 summation order."""
    fake_device_lib.install(monkeypatch, 2)
    from monodetr_b200 import _lib
    from monodetr_b200.position_encoding import PositionEmbeddingLearned
    fake = LearnedFakeLib(2)
    monkeypatch.setattr(_lib, "_lib", fake)
    torch.manual_seed(3)
    pe = PositionEmbeddingLearned(128)
    for H, W in ol.SHAPES:
        pe.zero_grad(set_to_none=True)
        t = pe(torch.zeros(2, H, W, 8))
        want = ol.table_nhwc(pe.col_embed.weight.detach(), pe.row_embed.weight.detach(), H, W)
        assert t.shape == (H * W, 256) and torch.equal(t.detach(), want)
        g = torch.randn(H * W, 256, generator=torch.Generator().manual_seed(H * 1000 + W))
        t.backward(g)
        col = pe.col_embed.weight.detach().clone().requires_grad_()
        row = pe.row_embed.weight.detach().clone().requires_grad_()
        ol.table_nhwc(col, row, H, W).backward(g)
        assert torch.allclose(pe.col_embed.weight.grad, col.grad, rtol=0, atol=1e-5 * float(col.grad.abs().max()))
        assert torch.allclose(pe.row_embed.weight.grad, row.grad, rtol=0, atol=1e-5 * float(row.grad.abs().max()))
    assert fake.calls["mdb_pos_learned_forward_f32"] == len(ol.SHAPES)
    assert fake.calls["mdb_pos_learned_backward_f32"] == len(ol.SHAPES)
