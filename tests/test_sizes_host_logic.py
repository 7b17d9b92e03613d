"""CPU: the whole product model at the reference's other transformer sizes (tests/oracle_sizes.VARIANTS: 6 / 6 layers with
dim_feedforward 1024, 300 queries with dim_feedforward 2048, 1 / 1 layers without aux outputs, use_dab with 100 queries and 4
decoder layers) through the stand-in device library (tests/fake_device_lib.py), against the oracle (tests/oracle_sizes.py):
train-mode outputs and every parameter gradient, and the eval-mode outputs."""
import pytest
import torch

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
import oracle_sizes as osz      # tests/oracle_sizes.py
from test_dab_host_logic import DabFakeLib      # the stand-in extended by the anchor-box kernels

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


def _build(monkeypatch, tag):
    fake_device_lib.install(monkeypatch, 1)
    from monodetr_b200 import _lib, build_monodetr
    monkeypatch.setattr(_lib, "_lib", DabFakeLib(1))
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, dropout=0.0, device="cpu", **osz.VARIANTS[tag]))
    sd = osz.deterministic_state_dict(osz.sizes_cfg(tag))
    m.load_state_dict(om.with_aliases(sd))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return _lib._lib, m, sd


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


def _check_outputs(out, ref, cfg):
    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, k
        assert _rel(out[k].detach(), ref[k].detach()) < 1e-4, (k, _rel(out[k].detach(), ref[k].detach()))
    assert ("aux_outputs" in out) == cfg["aux_loss"] == ("aux_outputs" in ref)
    if cfg["aux_loss"]:
        assert len(out["aux_outputs"]) == len(ref["aux_outputs"]) == cfg["dec_layers"] - 1
        for a, b in zip(out["aux_outputs"], ref["aux_outputs"]):
            for k in a:
                assert _rel(a[k].detach(), b[k].detach()) < 1e-4, ("aux", k)


@pytest.mark.parametrize("tag", list(osz.VARIANTS))
def test_train_mode_forward_and_every_gradient_match_the_oracle(monkeypatch, tag):
    """Outputs within 1e-4 and every gradient with the bars tests/test_points_host_logic.py holds the point counts to."""
    from monodetr_b200.bench_model import surrogate_loss
    fake, m, sd = _build(monkeypatch, tag)
    cfg = osz.sizes_cfg(tag)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    out = m(images, calibs, None, sizes)
    assert out["pred_logits"].shape[1] == cfg["num_queries"] * 11
    surrogate_loss(out).backward()

    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = osz.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
    om.surrogate_loss(ref).backward()
    _check_outputs(out, ref, cfg)

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
    assert errs[len(errs) // 2][0] < 3e-4, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < 3e-2 or scale < 1e-6, (name, err, scale)
    # every decoder layer ran: one set of heads per layer
    assert sum(1 for n, p in m.named_parameters() if n.startswith("class_embed.") and p.grad is not None) == 2 * cfg["dec_layers"]


@pytest.mark.parametrize("tag", list(osz.VARIANTS))
def test_eval_mode_forward_matches_the_oracle(monkeypatch, tag):
    fake, m, sd = _build(monkeypatch, tag)
    cfg = osz.sizes_cfg(tag)
    m.eval()
    images, calibs, sizes = om.synthetic_inputs(2, 1, H=96, W=320)
    with torch.no_grad():
        out = m(images, calibs, None, sizes)
        ref = osz.forward(sd, images, calibs, sizes, training=False, cfg=cfg)
    assert out["pred_logits"].shape[1] == cfg["num_queries"]
    _check_outputs(out, ref, cfg)
