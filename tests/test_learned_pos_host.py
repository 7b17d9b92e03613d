"""CPU: the host contract of the learned position embedding (`position_embedding: 'learned'` / 'v3') -- state_dict names / shapes /
trainability against the unmodified reference (tests/golden/learned_pos.npz) for resnet50 and resnet50 + DC5, the reference's
initialisation, strict loading of a reference-keyed checkpoint, the gradient bucket and the fused optimizer holding both tables,
and that the default sine branch keeps its 582 keys and 313 gradient tensors."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py
import oracle_backbones as ob    # tests/oracle_backbones.py
import oracle_learned_pos as ol  # tests/oracle_learned_pos.py


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "learned_pos.npz"))


def _build(**kw):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    return build_monodetr(dict(DEFAULT_MODEL_CFG, device="cpu", **kw))[0]


@pytest.mark.parametrize("tag,dilation", [("learned", False), ("dc5", True)])
def test_state_dict_matches_the_reference(tag, dilation, golden):
    m = _build(position_embedding="learned", dilation=dilation)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    assert {k: tuple(s) for k, s, _ in spec} == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n_ for n_, p in m.named_parameters() if p.requires_grad}
    assert len(spec) == 584
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in
                                   ol.state_dict_spec(ob.state_dict_spec(ob.variant_cfg("resnet50", dilation))).items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == {k: tuple(s) for k, s, _ in spec}


@pytest.mark.parametrize("name", ["learned", "v3"])
def test_both_names_build_the_learned_module(name):
    from monodetr_b200.position_encoding import PositionEmbeddingLearned
    m = _build(position_embedding=name)
    pe = m.backbone[1]
    assert isinstance(pe, PositionEmbeddingLearned)
    # nn.Embedding's N(0, 1), as the reference leaves it
    for w in (pe.row_embed.weight.detach(), pe.col_embed.weight.detach()):
        assert w.shape == (50, 128) and abs(float(w.std()) - 1.0) < 0.1 and abs(float(w.mean())) < 0.1


def test_other_names_and_widths_raise():
    with pytest.raises(NotImplementedError):
        _build(position_embedding="cosine")
    from monodetr_b200.position_encoding import build_position_encoding
    with pytest.raises(NotImplementedError, match="hidden_dim 256"):
        build_position_encoding({"hidden_dim": 128, "position_embedding": "learned"})


def test_tables_train_with_a_frozen_backbone():
    """The reference's freeze rule walks the ResNet body only (backbone.py:71-73): both tables train with train_backbone False."""
    m = _build(position_embedding="learned", train_backbone=False)
    trainable = {n for n, p in m.named_parameters() if p.requires_grad}
    assert {ol.ROW, ol.COL} <= trainable
    assert not any(n.startswith("backbone.0.") for n in trainable)


def test_reference_keyed_checkpoint_loads_strictly():
    m = _build(position_embedding="learned")
    sd = om.with_aliases(ol.with_tables(om.deterministic_state_dict()))
    sd["backbone.0.body.bn1.num_batches_tracked"] = torch.tensor(0)           # dropped like the reference (backbone.py:41-50)
    m.load_state_dict(sd, strict=True)
    assert torch.equal(m.backbone[1].row_embed.weight, sd[ol.ROW]) and torch.equal(m.backbone[1].col_embed.weight, sd[ol.COL])


def test_bucket_and_optimizer_hold_both_tables(monkeypatch):
    fake_device_lib.install(monkeypatch, 2)
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.optim import FusedAdamW
    m = _build(position_embedding="learned")
    bucket = FlatGradBucket(m)
    assert len(bucket.names) == 315 and {ol.ROW, ol.COL} <= set(bucket.names)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt = FusedAdamW(m, bucket, lr=2e-4, weight_decay=1e-4)
    lo, hi = opt.flat_p.data_ptr(), opt.flat_p.data_ptr() + opt.flat_p.numel() * 4
    for name in (ol.ROW, ol.COL):
        p = dict(m.named_parameters())[name]
        assert lo <= p.data_ptr() < hi and p.data_ptr() % 16 == 0          # a view of the flat buffer, aligned for float4 loads
        assert torch.equal(p.detach(), before[name])
        assert bucket.offsets[bucket.names.index(name)] < bucket.n_decay   # weight decay applies: no 'bias' in the name
    assert sum(len(g["params"]) for g in opt.param_groups) == 315


def test_default_branch_keeps_582_keys_and_313_gradient_tensors():
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.position_encoding import PositionEmbeddingSine
    m = _build()
    assert len(m.state_dict()) == 582 and isinstance(m.backbone[1], PositionEmbeddingSine)
    assert not any("_embed" in n for n, _ in m.backbone.named_parameters())
    assert len(FlatGradBucket(m).names) == 313
