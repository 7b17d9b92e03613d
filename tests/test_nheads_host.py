"""CPU: the reference's other head counts (cfg `nheads` 4 and 16) -- the product model's state_dict contract against the
unmodified reference (tests/golden/nheads.npz, written by tools/gen_golden_nheads.py), the oracle (tests/oracle_nheads.py)
against the reference's outputs and gradients, and the head counts the product refuses."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import monodetr_torch as om
import oracle_nheads as on      # tests/oracle_nheads.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import grad_index  # noqa: E402
from gen_golden_nheads import VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "nheads.npz"))


def _build(nheads):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    return build_monodetr(dict(DEFAULT_MODEL_CFG, nheads=nheads))[0]


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_state_dict_matches_the_reference(tag, golden):
    nheads = VARIANTS[tag]
    m = _build(nheads)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert len(spec) == 582
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    assert {k: tuple(s) for k, s, _ in spec} == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n for n, p in m.named_parameters() if p.requires_grad}
    shapes = {k: tuple(s) for k, s, _ in spec}
    assert shapes["depthaware_transformer.encoder.layers.0.self_attn.sampling_offsets.weight"] == (nheads * 32, 256)
    assert shapes["depthaware_transformer.decoder.layers.0.cross_attn.attention_weights.weight"] == (nheads * 16, 256)
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in on.state_dict_spec(on.heads_cfg(nheads)).items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == shapes


@pytest.mark.parametrize("nheads", [4, 16])
def test_reference_shaped_checkpoint_loads_strictly(nheads):
    m = _build(nheads)
    m.load_state_dict(om.with_aliases(on.deterministic_state_dict(on.heads_cfg(nheads))), strict=True)
    dec = m.depthaware_transformer.decoder.layers[0]
    assert dec.nhead == nheads and dec.cross_attn.n_heads == nheads
    assert dec.cross_attn_depth.num_heads == nheads and dec.self_attn.num_heads == nheads
    assert m.depthaware_transformer.encoder.layers[0].self_attn.n_heads == nheads
    assert m.depth_predictor.depth_encoder.layers[0].self_attn.num_heads == 8      # pinned like the reference


@pytest.mark.parametrize("nheads", [1, 2, 3, 5, 6, 7, 12, 32, 64])
def test_unsupported_head_counts_raise(nheads):
    with pytest.raises(NotImplementedError, match="nheads must be one of 4, 8, 16"):
        _build(nheads)


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
    tests/test_backbone_variants_host.py holds the backbone oracle to."""
    cfg = on.heads_cfg(VARIANTS[tag])
    sd = on.deterministic_state_dict(cfg)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        _check_outputs(golden, f"{tag}.fwd_eval", on.forward(sd, images, calibs, sizes, training=False, cfg=cfg), 2e-4, 2e-5)

    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    sdg = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    out = on.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
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
