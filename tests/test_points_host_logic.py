"""CPU: the whole product model with the reference's other sampling-point counts (cfg `enc_n_points` / `dec_n_points` 2 / 2,
8 / 8 and 3 / 6) through the stand-in device library (tests/fake_device_lib.py), against the oracle (tests/oracle_points.py):
outputs and every parameter gradient, in both GEMM precisions and in reproducible mode.  The stand-in is extended here to refuse
what the real deformable-attention entry points refuse (csrc/msda.cu): the fused kernels take D = 32, 4 levels and 2, 4 or 8
points; the pre-processing takes up to 32 (level, point) pairs.  In the default mode the counts 2 and 8 must run fused, without a
pre-processing call; every other count, and reproducible mode, takes the two-step path."""
import pytest
import torch

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
import oracle_points as op      # tests/oracle_points.py

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")
MDB_EUNSUPPORTED = -2
VARIANTS = {"p2": (2, 2), "p8": (8, 8), "p3_6": (3, 6)}


class PointsFakeLib(fake_device_lib.FakeLib):
    """FakeLib whose deformable-attention entry points return MDB_EUNSUPPORTED wherever the device library's do, and log the
    point count of every call."""

    def __init__(self, precision):
        super().__init__(precision)
        self.msda_log = []

    def mdb_msda_prep_forward_f32(self, off, logits, ref, shapes, B, Lq, M, L, P, rd, loc, attn, stream):
        self.msda_log.append(("prep", P))
        if L * P > 32 or rd not in (2, 6):
            return MDB_EUNSUPPORTED
        return super().mdb_msda_prep_forward_f32(off, logits, ref, shapes, B, Lq, M, L, P, rd, loc, attn, stream)

    def mdb_msda_prep_backward_f32(self, dloc, dattn, attn, ref, shapes, B, Lq, M, L, P, rd, doff, dlogits, stream):
        if L * P > 32 or rd not in (2, 6):
            return MDB_EUNSUPPORTED
        return super().mdb_msda_prep_backward_f32(dloc, dattn, attn, ref, shapes, B, Lq, M, L, P, rd, doff, dlogits, stream)

    def mdb_msda_fused_forward_f32(self, value, shapes, lsi, off, logits, ref, B, S, M, D, L, Lq, P, rd, out, stream):
        self.msda_log.append(("fused", P))
        if D != 32 or L != 4 or P not in (2, 4, 8) or rd not in (2, 6):
            return MDB_EUNSUPPORTED
        return super().mdb_msda_fused_forward_f32(value, shapes, lsi, off, logits, ref, B, S, M, D, L, Lq, P, rd, out, stream)

    def mdb_msda_fused_backward_f32(self, value, shapes, lsi, off, logits, ref, gout, B, S, M, D, L, Lq, P, rd, gv, goff, glog,
                                    stream):
        if D != 32 or L != 4 or P not in (2, 4, 8) or rd not in (2, 6) or self.deterministic:
            return MDB_EUNSUPPORTED
        return super().mdb_msda_fused_backward_f32(value, shapes, lsi, off, logits, ref, gout, B, S, M, D, L, Lq, P, rd, gv, goff,
                                                   glog, stream)

    def mdb_msda_fused_backward_ref_f32(self, value, shapes, lsi, off, logits, ref, gout, B, S, M, D, L, Lq, P, rd, gv, goff, glog,
                                        part, stream):
        # the stand-in has no box-partial kernel: any call the real library would accept is a path this model must not take
        if D != 32 or L != 4 or P not in (2, 4, 8) or rd != 6 or self.deterministic:
            return MDB_EUNSUPPORTED
        raise AssertionError("mdb_msda_fused_backward_ref_f32 is not on the path of a model without use_dab")


def _build(monkeypatch, precision, points):
    fake_device_lib.install(monkeypatch, {"tf32x3": 1, "bf16x3": 2}[precision])
    from monodetr_b200 import _lib, build_monodetr, tc
    fake = PointsFakeLib({"tf32x3": 1, "bf16x3": 2}[precision])
    monkeypatch.setattr(_lib, "_lib", fake)
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    assert tc.get_precision() == precision
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, enc_n_points=points[0], dec_n_points=points[1], dropout=0.0, device="cpu"))
    sd = op.deterministic_state_dict(op.points_cfg(*points))
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


@pytest.mark.parametrize("tag", list(VARIANTS))
@pytest.mark.parametrize("precision,deterministic", [("bf16x3", False), ("tf32x3", False), ("tf32x3", True)])
def test_train_mode_forward_and_every_gradient_match_the_oracle(monkeypatch, tag, precision, deterministic):
    """Outputs within 1e-4 and every gradient with the bars of tests/test_model_host_logic.py; the path each layer takes."""
    from monodetr_b200.bench_model import surrogate_loss
    points = VARIANTS[tag]
    fake, m, sd = _build(monkeypatch, precision, points)
    fake.deterministic = int(deterministic)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    out = m(images, calibs, None, sizes)
    surrogate_loss(out).backward()

    cfg = op.points_cfg(*points)
    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = op.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
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

    # every deformable-attention call ran at its layer's count, on the path that count selects
    assert {P for _, P in fake.msda_log} == set(points)
    assert not any(kind == "fused" and P not in (2, 4, 8) for kind, P in fake.msda_log), fake.msda_log
    calls = fake.calls
    if deterministic:
        assert calls.get("mdb_msda_fused_backward_f32", 0) == 0
        assert calls.get("mdb_msda_prep_backward_f32", 0) > 0
    fused_counts = all(P in (2, 4, 8) for P in points)
    if fused_counts and not deterministic:
        # the one two-step call is decoder layer 0, whose reference points (a learned projection) need a gradient -- as at 4 / 4
        assert calls.get("mdb_msda_prep_forward_f32", 0) == 1 and calls.get("mdb_msda_prep_backward_f32", 0) == 1, calls
        assert fake.msda_log.count(("prep", points[1])) == 1
        assert calls.get("mdb_msda_fused_backward_f32", 0) == 3 + 2         # 3 encoder layers, decoder layers 1 and 2
    if not fused_counts:
        assert calls.get("mdb_msda_fused_forward_f32", 0) == 0 and calls.get("mdb_msda_prep_forward_f32", 0) > 0


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_eval_mode_forward_matches_the_oracle(monkeypatch, tag):
    points = VARIANTS[tag]
    fake, m, sd = _build(monkeypatch, "tf32x3", points)
    m.eval()
    images, calibs, sizes = om.synthetic_inputs(2, 1, H=96, W=320)
    with torch.no_grad():
        out = m(images, calibs, None, sizes)
        ref = op.forward(sd, images, calibs, sizes, training=False, cfg=op.points_cfg(*points))
    _check_outputs(out, ref)
    # no gradient anywhere: every layer at a fused count runs fused
    fused = [P in (2, 4, 8) for P in points]
    assert fake.calls.get("mdb_msda_prep_forward_f32", 0) == 3 * (not fused[0]) + 3 * (not fused[1]), fake.calls
    assert fake.calls.get("mdb_msda_fused_forward_f32", 0) == 3 * fused[0] + 3 * fused[1]


def test_four_point_oracle_is_the_base_oracle():
    """At 4 / 4 the point-count oracle is om itself: same weights, same outputs bit for bit."""
    cfg = op.points_cfg(4, 4)
    sd = op.deterministic_state_dict(cfg)
    base = om.deterministic_state_dict()
    assert sd.keys() == base.keys() and all(torch.equal(sd[k], base[k]) for k in sd)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    with torch.no_grad():
        a = op.forward(sd, images, calibs, sizes, training=False, cfg=cfg)
        b = om.forward(base, images, calibs, sizes, training=False)
    for k in OUT_KEYS:
        assert torch.equal(a[k], b[k]), k
