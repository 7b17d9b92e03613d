"""CPU: the use_dab oracle (tests/oracle_dab.py) against the unmodified reference (tests/golden/dab.npz, written by
tools/gen_golden_dab.py): eval outputs at 192 x 640, train outputs and every parameter gradient at 96 x 320 for batch 1 and 2,
with the bars of tests/test_oracle_model.py."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import monodetr_torch as om
import oracle_dab as od          # tests/oracle_dab.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import grad_index  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "dab.npz"))


def check_outputs(golden, prefix, out, rtol, atol):
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_{k}", out[k].detach().cpu().numpy()), rtol=rtol,
                                   atol=atol, err_msg=prefix + " " + k)
    assert len(out["aux_outputs"]) == 2
    for i, a in enumerate(out["aux_outputs"]):
        for k in a:
            np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_aux{i}_{k}", a[k].detach().cpu().numpy()), rtol=rtol,
                                       atol=atol, err_msg=f"{prefix} aux{i} {k}")


def test_oracle_spec_is_the_references(golden):
    spec = json.loads(golden["dab.spec"].tobytes())
    assert len(spec) == 585
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in od.state_dict_spec().items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == {k: tuple(s) for k, s, _ in spec}


def test_oracle_eval_matches_the_reference(golden):
    sd = od.deterministic_state_dict()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        check_outputs(golden, "fwd_eval", od.forward(sd, images, calibs, sizes, training=False), 2e-4, 2e-5)


@pytest.mark.parametrize("B", [1, 2])
def test_oracle_train_and_gradients_match_the_reference(B, golden):
    sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in od.deterministic_state_dict().items()}
    images, calibs, sizes = om.synthetic_inputs(B, 0, H=96, W=320)
    out = od.forward(sd, images, calibs, sizes, training=True)
    tag = f"b{B}"
    check_outputs(golden, f"{tag}.fwd_train", out, 2e-4, 2e-5)
    om.surrogate_loss(out).backward()
    names = json.loads(golden[f"{tag}.grad_names"].tobytes())
    assert "refpoint_embed.weight" in names and "tgt_embed.weight" in names
    assert not any("query_scale_bbox" in n for n in names)               # never called by the reference
    offs = np.concatenate([[0], np.cumsum(golden[f"{tag}.grad_len"])])
    rels = []
    for j, name in enumerate(names):
        if name not in sd:
            continue                                          # decoder alias of a shared head
        gm = sd[name].grad
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
    for name in ("refpoint_embed.weight", "depthaware_transformer.decoder.ref_point_head.layers.0.bias",
                 "depthaware_transformer.decoder.query_scale.layers.0.bias"):
        full = golden[f"{tag}.grad_full.{name}"]
        l2 = float(np.linalg.norm(sd[name].grad.numpy() - full) / np.linalg.norm(full))
        assert l2 < 2e-2, (name, l2)
