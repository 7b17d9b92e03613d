"""CPU: the reference's other transformer sizes (cfg `enc_layers` / `dec_layers` / `num_queries` / `dim_feedforward` /
`aux_loss`) -- the product model's state_dict contract against the unmodified reference (tests/golden/sizes.npz, written by
tools/gen_golden_sizes.py), the oracle (tests/oracle_sizes.py) against the reference's outputs and gradients, the oracle
criterion (scipy) against the reference criterion at 6 layers and up to 300 queries per group (tests/golden/criterion_sizes.npz),
and the sizes the product refuses."""
import json
import os
import re
import sys

import numpy as np
import pytest
import torch

from oracle import criterion as oc
from oracle import monodetr_torch as om
import oracle_sizes as osz      # tests/oracle_sizes.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import grad_index  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sizes.npz"))


@pytest.fixture(scope="module")
def crit_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "criterion_sizes.npz"))


def _build(**kw):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    return build_monodetr(dict(DEFAULT_MODEL_CFG, device="cpu", **kw))[0]


@pytest.mark.parametrize("tag", list(osz.VARIANTS))
def test_state_dict_matches_the_reference(tag, golden):
    v = osz.VARIANTS[tag]
    m = _build(**v)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    shapes = {k: tuple(s) for k, s, _ in spec}
    assert shapes == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n for n, p in m.named_parameters() if p.requires_grad}
    cfg = osz.sizes_cfg(tag)
    enc = {int(x) for x in re.findall(r"encoder\.layers\.(\d+)\.", " ".join(shapes))}
    dec = {int(x) for x in re.findall(r"^depthaware_transformer\.decoder\.layers\.(\d+)\.", "\n".join(shapes), re.M)}
    assert enc == set(range(cfg["enc_layers"])) and dec == set(range(cfg["dec_layers"]))
    assert shapes["depthaware_transformer.encoder.layers.0.linear1.weight"] == (cfg["dim_feedforward"], 256)
    assert shapes["depthaware_transformer.decoder.layers.0.linear2.weight"] == (256, cfg["dim_feedforward"])
    q = "tgt_embed.weight" if cfg["use_dab"] else "query_embed.weight"
    assert shapes[q][0] == cfg["num_queries"] * 11
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in osz.state_dict_spec(cfg).items()})
    assert {k: tuple(t.shape) for k, t in oracle_spec.items()} == shapes


@pytest.mark.parametrize("kw", [dict(enc_layers=6, dec_layers=6, dim_feedforward=1024), dict(num_queries=300, dim_feedforward=2048),
                                dict(enc_layers=1, dec_layers=1, aux_loss=False), dict(enc_layers=2, dec_layers=5, num_queries=1),
                                dict(use_dab=True, num_queries=100, dec_layers=4)])
def test_reference_shaped_checkpoint_loads_strictly(kw):
    m = _build(**kw)
    cfg = {**om.CFG, "use_dab": False, "aux_loss": True, **kw}
    m.load_state_dict(om.with_aliases(osz.deterministic_state_dict(cfg)), strict=True)
    assert len(m.depthaware_transformer.encoder.layers) == cfg["enc_layers"]
    assert len(m.depthaware_transformer.decoder.layers) == cfg["dec_layers"]


@pytest.mark.parametrize("kw", [dict(backbone="resnet101"), dict(dilation=True), dict(use_dab=True), dict(position_embedding="learned"),
                                dict(nheads=4), dict(nheads=16), dict(enc_n_points=8, dec_n_points=2)])
def test_sizes_combine_with_the_other_model_options(kw):
    m = _build(enc_layers=5, dec_layers=6, num_queries=300, dim_feedforward=2048, **kw)
    assert len(m.depthaware_transformer.decoder.layers) == 6 and len(m.class_embed) == 6
    assert m.num_queries == 300


@pytest.mark.parametrize("kw,match", [
    (dict(enc_layers=0), "enc_layers=0: 1 to 6"), (dict(enc_layers=7), "enc_layers=7: 1 to 6"),
    (dict(dec_layers=0), "dec_layers=0: 1 to 6"), (dict(dec_layers=7), "dec_layers=7: 1 to 6"),
    (dict(num_queries=0), "num_queries=0"), (dict(num_queries=301), "num_queries=301"),
    (dict(dim_feedforward=0), "dim_feedforward=0"), (dict(dim_feedforward=1026), "dim_feedforward=1026"),
    (dict(return_intermediate_dec=False), "reference itself fails"), (dict(hidden_dim=128), "reference itself fails")])
def test_unsupported_sizes_raise_before_the_device(monkeypatch, kw, match):
    def no_device(*a, **k):
        raise AssertionError("the device was touched")
    monkeypatch.setattr(torch.Tensor, "cuda", no_device)
    monkeypatch.setattr(torch.nn.Module, "cuda", no_device)
    from monodetr_b200 import _lib
    monkeypatch.setattr(_lib, "call", no_device)
    with pytest.raises(NotImplementedError, match=match):
        _build(**kw)


def test_criterion_layer_limit_is_the_header_constant():
    from monodetr_b200 import criterion
    with open(os.path.join(ROOT, "include", "monodetr_b200.h")) as f:
        header = f.read()
    assert int(re.search(r"#define MDB_CRITERION_MAX_LAYERS (\d+)", header).group(1)) == criterion.MAX_LAYERS == 6
    assert int(re.search(r"#define MDB_CRITERION_NUM_LOSSES (\d+)", header).group(1)) == criterion.NUM_LOSSES


def test_criterion_takes_the_queries_of_its_model():
    """build_criterion(cfg) accepts cfg["num_queries"] queries per group, and never fewer than the 64 it always took."""
    from monodetr_b200.criterion import SetCriterion, build_criterion
    from bench_extras import CRIT_CFG
    assert build_criterion(CRIT_CFG).max_queries == 64
    assert [build_criterion(dict(CRIT_CFG, num_queries=n)).max_queries for n in (1, 50, 64, 65, 100, 300)] == [64, 64, 64, 65, 100, 300]
    for n in (63, 301):
        with pytest.raises(NotImplementedError, match="max_queries"):
            SetCriterion(3, None, {}, 0.25, ["labels"], max_queries=n)


def test_stream_indices_are_distinct_up_to_six_layers():
    """Every branch of a 6-layer decoder has its own stream; layers 0-2 keep the default schedule's indices."""
    from monodetr_b200.depthaware_transformer import ahead_streams
    from monodetr_b200.monodetr import head_stream
    assert [ahead_streams(l) for l in range(3)] == [(9, 12), (10, 13), (11, 14)]
    assert [head_stream(l) for l in range(3)] == [1, 2, 3]
    fixed = [0, 5, 6, 7, 8, 15, 16, 17, 18]       # depth predictor, box / dim heads, self-attention k / v, neck
    used = fixed + [i for l in range(6) for i in ahead_streams(l)] + [head_stream(l) for l in range(6)]
    assert len(used) == len(set(used)), sorted(used)


def _check_outputs(golden, prefix, out, rtol, atol, n_aux):
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_{k}", out[k].detach().numpy()), rtol=rtol, atol=atol,
                                   err_msg=prefix + " " + k)
    assert len(out.get("aux_outputs", [])) == n_aux
    assert not any(k.startswith(f"{prefix}_aux{n_aux}_") for k in golden.files)
    for i, a in enumerate(out.get("aux_outputs", [])):
        for k in a:
            np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_aux{i}_{k}", a[k].detach().numpy()), rtol=rtol,
                                       atol=atol, err_msg=f"{prefix} aux{i} {k}")


def n_aux_of(cfg):
    return cfg["dec_layers"] - 1 if cfg["aux_loss"] else 0


@pytest.mark.parametrize("tag", list(osz.VARIANTS))
def test_oracle_matches_the_reference(tag, golden):
    """Eval outputs at 192 x 640 and train outputs + every parameter gradient at 96 x 320, with the bars
    tests/test_points_host.py holds the point-count oracle to."""
    cfg = osz.sizes_cfg(tag)
    sd = osz.deterministic_state_dict(cfg)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        _check_outputs(golden, f"{tag}.fwd_eval", osz.forward(sd, images, calibs, sizes, training=False, cfg=cfg), 2e-4, 2e-5,
                       n_aux_of(cfg))

    if f"{tag}.grad_names" not in golden.files:
        assert cfg["num_queries"] != 50                       # the reference trains at 50 queries per group only
        return
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    sdg = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    out = osz.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
    _check_outputs(golden, f"{tag}.fwd_train", out, 2e-4, 2e-5, n_aux_of(cfg))
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
    assert len(rels) > 100
    assert sorted(rels)[len(rels) // 2] < 1e-3


def run_oracle_criterion(name):
    seed, counts, nq, group, L = osz.CRITERION_CASES[name]
    out, padded = osz.criterion_case(name)
    leaves = {}
    for layer, d in [("main", out)] + [(f"aux{i}", a) for i, a in enumerate(out.get("aux_outputs", []))]:
        for k in list(d):
            if torch.is_tensor(d[k]):
                d[k] = d[k].clone().requires_grad_(True)
                leaves[f"{layer}.{k}"] = d[k]
    losses, indices = oc.set_criterion(out, padded, training=group > 1, group_num=group)
    w = oc.weight_dict(L)
    total = sum(losses[k] * w[k] for k in losses if k in w)
    total.backward()
    return losses, indices, total, leaves


@pytest.mark.parametrize("name", list(osz.CRITERION_CASES))
def test_oracle_criterion_matches_the_reference(name, crit_golden):
    seed, counts, nq, group, L = osz.CRITERION_CASES[name]
    losses, indices, total, leaves = run_oracle_criterion(name)
    keys = [k[len(name) + 6:] for k in crit_golden.files if k.startswith(f"{name}.loss.")]
    assert sorted(keys) == sorted(losses)
    assert len(indices) == L
    for k in keys:
        np.testing.assert_allclose(float(losses[k]), float(crit_golden[f"{name}.loss.{k}"]), rtol=2e-6, atol=1e-7, err_msg=k)
    np.testing.assert_allclose(float(total), float(crit_golden[f"{name}.total"]), rtol=2e-6)
    for l, ind in enumerate(indices):
        for b, (i, j) in enumerate(ind):
            assert len(j) == min(counts[b], nq) * group
            assert np.array_equal(i.numpy(), crit_golden[f"{name}.match.{l}.{b}.src"])
            assert np.array_equal(j.numpy(), crit_golden[f"{name}.match.{l}.{b}.tgt"])
    for k, t in leaves.items():
        full = t.grad.numpy() if t.grad is not None else np.zeros(tuple(t.shape), np.float32)
        got, g, gmax = oc.golden_grad(crit_golden, f"{name}.grad.{k}", full)
        np.testing.assert_allclose(got, g, rtol=1e-5, atol=1e-9 + 1e-6 * gmax, err_msg=k)
