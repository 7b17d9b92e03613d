"""CPU: the learned-position-embedding oracle (tests/oracle_learned_pos.py) against the unmodified reference
(tests/golden/learned_pos.npz, written by tools/gen_golden_learned_pos.py): the module alone at every fixture shape, its table
bit for bit (SHA-256 of both axes) and its gradients at sampled positions; the model's eval outputs at 192 x 640; train outputs
and every parameter gradient at 96 x 320 for batch 1 and 2, with the bars of tests/test_oracle_dab.py, and at batch 2 the whole
gradients of both tables."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import monodetr_torch as om
import oracle_learned_pos as ol  # tests/oracle_learned_pos.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import grad_index  # noqa: E402
from test_oracle_dab import check_outputs  # noqa: E402


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "learned_pos.npz"))


def test_oracle_spec_is_the_references(golden):
    for tag in ("learned", "dc5"):
        spec = json.loads(golden[f"{tag}.spec"].tobytes())
        assert len(spec) == 584
        assert {(k, tuple(s), t) for k, s, t in spec if "_embed" in k and k.startswith("backbone.")} == \
            {(ol.ROW, ol.TABLE_SHAPE, True), (ol.COL, ol.TABLE_SHAPE, True)}
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in ol.state_dict_spec(om.state_dict_spec()).items()})
    spec = json.loads(golden["learned.spec"].tobytes())
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == {k: tuple(s) for k, s, _ in spec}


@pytest.mark.parametrize("h,w", ol.SHAPES)
def test_module_forward_is_exact_and_gradients_match(h, w, golden):
    col, row = ol.module_tables()
    x_emb, y_emb = ol.axis_embeds(col, row, h, w)
    tag = f"mod.{h}x{w}"
    assert np.array_equal(ol.digest(x_emb), golden[tag + ".x_sha"]) and np.array_equal(ol.digest(y_emb), golden[tag + ".y_sha"])
    pos = ol.position_embedding_learned(col, row, 1, h, w)
    assert torch.equal(pos[0, :128, 0, :].T, x_emb) and torch.equal(pos[0, 128:, :, 0].T, y_emb)
    c, r = col.clone().requires_grad_(), row.clone().requires_grad_()
    ol.position_embedding_learned(c, r, 1, h, w).backward(ol.upstream_grad(h, w))
    for got, key in ((c.grad, "dcol"), (r.grad, "drow")):
        scale = float(golden[f"{tag}.{key}.max"])
        assert abs(float(got.abs().max()) - scale) <= 1e-5 * scale, key
        idx = golden[f"{tag}.{key}.idx"]
        assert idx.size > 0
        np.testing.assert_allclose(got.reshape(-1).numpy()[idx], golden[f"{tag}.{key}.val"], rtol=0, atol=1e-5 * scale, err_msg=key)


def test_oracle_eval_matches_the_reference(golden):
    sd = ol.with_tables(om.deterministic_state_dict())
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        check_outputs(golden, "fwd_eval", ol.forward(sd, images, calibs, sizes, training=False), 2e-4, 2e-5)


@pytest.mark.parametrize("B", [1, 2])
def test_oracle_train_and_gradients_match_the_reference(B, golden):
    sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in ol.with_tables(om.deterministic_state_dict()).items()}
    images, calibs, sizes = om.synthetic_inputs(B, 0, H=96, W=320)
    out = ol.forward(sd, images, calibs, sizes, training=True)
    tag = f"b{B}"
    check_outputs(golden, f"{tag}.fwd_train", out, 2e-4, 2e-5)
    om.surrogate_loss(out).backward()
    names = json.loads(golden[f"{tag}.grad_names"].tobytes())
    assert len(names) == 315 and ol.ROW in names and ol.COL in names
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
    for name in (ol.ROW, ol.COL):
        if B == 1:
            continue                                          # the whole table gradients are stored for batch 2 only
        full = golden[f"{tag}.grad_full.{name}"]
        l2 = float(np.linalg.norm(sd[name].grad.numpy() - full) / np.linalg.norm(full))
        assert l2 < 2e-2, (name, l2)
