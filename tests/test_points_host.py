"""CPU: the reference's other sampling-point counts (cfg `enc_n_points` / `dec_n_points`) -- the product model's state_dict
contract against the unmodified reference (tests/golden/points.npz, written by tools/gen_golden_points.py), the oracle
(tests/oracle_points.py) against the reference's outputs and gradients, and the counts the product refuses."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import monodetr_torch as om
import oracle_points as op      # tests/oracle_points.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import grad_index  # noqa: E402
from gen_golden_points import VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "points.npz"))


def _build(enc, dec, **kw):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    return build_monodetr(dict(DEFAULT_MODEL_CFG, enc_n_points=enc, dec_n_points=dec, **kw))[0]


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_state_dict_matches_the_reference(tag, golden):
    enc, dec = VARIANTS[tag]
    m = _build(enc, dec)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert len(spec) == 582
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    assert {k: tuple(s) for k, s, _ in spec} == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n for n, p in m.named_parameters() if p.requires_grad}
    shapes = {k: tuple(s) for k, s, _ in spec}
    assert shapes["depthaware_transformer.encoder.layers.0.self_attn.sampling_offsets.weight"] == (8 * 4 * enc * 2, 256)
    assert shapes["depthaware_transformer.encoder.layers.0.self_attn.attention_weights.weight"] == (8 * 4 * enc, 256)
    assert shapes["depthaware_transformer.decoder.layers.0.cross_attn.sampling_offsets.weight"] == (8 * 4 * dec * 2, 256)
    assert shapes["depthaware_transformer.decoder.layers.0.cross_attn.attention_weights.weight"] == (8 * 4 * dec, 256)
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in op.state_dict_spec(op.points_cfg(enc, dec)).items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == shapes


@pytest.mark.parametrize("enc,dec", [(2, 2), (8, 8), (3, 6), (1, 7), (5, 1)])
def test_reference_shaped_checkpoint_loads_strictly(enc, dec):
    m = _build(enc, dec)
    m.load_state_dict(om.with_aliases(op.deterministic_state_dict(op.points_cfg(enc, dec))), strict=True)
    assert all(layer.self_attn.n_points == enc for layer in m.depthaware_transformer.encoder.layers)
    assert all(layer.cross_attn.n_points == dec for layer in m.depthaware_transformer.decoder.layers)


@pytest.mark.parametrize("kw", [dict(use_dab=True), dict(position_embedding="learned"), dict(nheads=4), dict(nheads=16)])
def test_counts_combine_with_the_other_model_options(kw):
    m = _build(8, 3, **kw)
    assert m.depthaware_transformer.encoder.layers[0].self_attn.n_points == 8
    assert m.depthaware_transformer.decoder.layers[0].cross_attn.n_points == 3


@pytest.mark.parametrize("enc,dec", [(0, 4), (9, 4), (4, 0), (4, 9), (-1, 4)])
def test_unsupported_point_counts_raise(enc, dec):
    with pytest.raises(NotImplementedError, match="1 to 8 sampling points per level"):
        _build(enc, dec)


def _check_outputs(golden, prefix, out, rtol, atol):
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_{k}", out[k].detach().numpy()), rtol=rtol, atol=atol,
                                   err_msg=prefix + " " + k)
    assert len(out["aux_outputs"]) == 2
    for i, a in enumerate(out["aux_outputs"]):
        for k in a:
            np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_aux{i}_{k}", a[k].detach().numpy()), rtol=rtol,
                                       atol=atol, err_msg=f"{prefix} aux{i} {k}")


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_oracle_matches_the_reference(tag, golden):
    """Eval outputs at 192 x 640 and train outputs + every parameter gradient at 96 x 320, with the bars
    tests/test_nheads_host.py holds the head-count oracle to."""
    cfg = op.points_cfg(*VARIANTS[tag])
    sd = op.deterministic_state_dict(cfg)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        _check_outputs(golden, f"{tag}.fwd_eval", op.forward(sd, images, calibs, sizes, training=False, cfg=cfg), 2e-4, 2e-5)

    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    sdg = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    out = op.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
    _check_outputs(golden, f"{tag}.fwd_train", out, 2e-4, 2e-5)
    om.surrogate_loss(out).backward()
    names = json.loads(golden[f"{tag}.grad_names"].tobytes())
    offs = np.concatenate([[0], np.cumsum(golden[f"{tag}.grad_len"])])
    rels = []
    for j, name in enumerate(names):
        if name not in sdg:
            continue                                          # decoder alias of a shared head
        gm = sdg[name].grad
        assert gm is not None, name
        scale = float(golden[f"{tag}.grad_max"][j])
        if scale < 1e-6:
            continue                                          # analytically zero (key biases of a softmax)
        gm = gm.reshape(-1)
        # gradients through the bilinear sampling locations can differ by O(1e-2) between two fp32 evaluation orders
        rel = float(np.abs(gm[grad_index(gm.numel(), name)].numpy() - golden[f"{tag}.grad_val"][offs[j]:offs[j + 1]]).max()) / scale
        assert rel <= 5e-2, (name, rel)
        assert abs(float(gm.abs().max()) - scale) <= 5e-2 * scale, name
        rels.append(rel)
    assert len(rels) > 250
    assert sorted(rels)[len(rels) // 2] < 1e-3
