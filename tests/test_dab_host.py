"""CPU: the use_dab model's host contract -- state_dict names / shapes / trainability against the unmodified reference
(tests/golden/dab.npz) for resnet50 and resnet101, strict loading of a reference-keyed checkpoint, the query rows eval uses,
what the GEMM prepacking covers, and that the default branch keeps its 582 keys."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import monodetr_torch as om
import oracle_backbones as ob     # tests/oracle_backbones.py
import oracle_dab as od          # tests/oracle_dab.py


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "dab.npz"))


def _build(**kw):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    return build_monodetr(dict(DEFAULT_MODEL_CFG, **kw))[0]


@pytest.mark.parametrize("tag,backbone,n", [("dab", "resnet50", 585), ("r101", "resnet101", 840)])
def test_state_dict_matches_the_reference(tag, backbone, n, golden):
    m = _build(use_dab=True, backbone=backbone)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    assert {k: tuple(s) for k, s, _ in spec} == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n_ for n_, p in m.named_parameters() if p.requires_grad}
    assert len(spec) == n
    base = ob.state_dict_spec(ob.variant_cfg(backbone, False))
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in od.state_dict_spec(od.CFG, base).items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == {k: tuple(s) for k, s, _ in spec}


def test_initialisation_follows_the_reference_rules():
    m = _build(use_dab=True)
    dec = m.depthaware_transformer.decoder
    assert not hasattr(m, "query_embed") and not hasattr(m.depthaware_transformer, "reference_points")
    # nn.Embedding's N(0, 1); the decoder MLPs' weights re-drawn by the transformer's xavier_uniform_, biases as nn.Linear left them
    for w in (m.tgt_embed.weight.detach(), m.refpoint_embed.weight.detach()):
        assert abs(float(w.std()) - 1.0) < 0.1 and abs(float(w.mean())) < 0.1
    for mlp in (dec.query_scale, dec.query_scale_bbox, dec.ref_point_head):
        for lin in mlp.layers:
            fan_in, fan_out = lin.weight.shape[1], lin.weight.shape[0]
            assert float(lin.weight.abs().max()) <= (6.0 / (fan_in + fan_out)) ** 0.5 + 1e-6
    assert dec.ref_point_head.layers[0].weight.shape == (256, 768)


def test_reference_keyed_checkpoint_loads_strictly():
    m = _build(use_dab=True)
    sd = om.with_aliases(od.deterministic_state_dict())
    sd["backbone.0.body.bn1.num_batches_tracked"] = torch.tensor(0)           # dropped like the reference (backbone.py:41-50)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.refpoint_embed.weight, sd["refpoint_embed.weight"])


def test_eval_uses_the_first_num_queries_anchors():
    m = _build(use_dab=True)
    tgt, anchors = m.train()._query_embeds()
    assert tgt is m.tgt_embed.weight and anchors is m.refpoint_embed.weight and anchors.shape == (550, 6)
    tgt, anchors = m.eval()._query_embeds()
    assert tgt.shape == (50, 256) and anchors.shape == (50, 6)
    assert tgt.data_ptr() == m.tgt_embed.weight.data_ptr() and anchors.data_ptr() == m.refpoint_embed.weight.data_ptr()


def test_dab_mlps_are_prepacked_and_query_scale_bbox_is_not():
    m = _build(use_dab=True)
    dec = m.depthaware_transformer.decoder
    packed = {id(w) for w in m._gemm_weights()}
    for lin in (*dec.query_scale.layers, *dec.ref_point_head.layers):
        assert id(lin.weight) in packed
    assert not any(id(lin.weight) in packed for lin in dec.query_scale_bbox.layers)
    d = _build()
    packed = {id(w) for w in d._gemm_weights()}
    dd = d.depthaware_transformer.decoder
    assert not any(id(lin.weight) in packed for lin in (*dd.query_scale.layers, *dd.ref_point_head.layers))


def test_flat_gradient_bucket_covers_the_dab_parameters():
    from monodetr_b200.ddp import FlatGradBucket
    m = _build(use_dab=True)
    names = set(FlatGradBucket(m).names)
    assert {"tgt_embed.weight", "refpoint_embed.weight"} <= names
    for p in ("query_scale", "ref_point_head"):
        assert {f"depthaware_transformer.decoder.{p}.layers.{i}.{k}" for i in (0, 1) for k in ("weight", "bias")} <= names
    assert not any("query_scale_bbox" in n or "sa_v_proj" in n or "label_enc" in n for n in names)
    d = _build()
    assert not any("query_scale" in n or "ref_point_head" in n for n in FlatGradBucket(d).names)


def test_default_branch_keeps_582_keys():
    m = _build()
    assert len(m.state_dict()) == 582 and hasattr(m, "query_embed")
    assert m.depthaware_transformer.decoder.ref_point_head.layers[-1].weight.shape == (2, 256)


@pytest.mark.parametrize("flag", ["two_stage", "two_stage_dino"])
def test_failing_reference_branches_still_raise(flag):
    with pytest.raises(NotImplementedError, match="the reference itself fails"):
        _build(**{flag: True})
