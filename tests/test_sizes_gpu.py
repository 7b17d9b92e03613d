"""H100: the reference's other transformer sizes (tests/oracle_sizes.VARIANTS) -- the device matcher against scipy at up to 300
queries per group and 6 decoder layers, the device criterion against the unmodified reference (tests/golden/criterion_sizes.npz),
the model against the reference (tests/golden/sizes.npz) and per-stage gradients against the oracle, reproducible training
iterations eager and as a CUDA graph at the deep and 300-query sizes, Tester inference at 300 queries, and the default
configuration's training iteration byte for byte against the build before the matcher took its dynamic shared memory."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import criterion as oc
from oracle import monodetr_torch as om
import oracle_sizes as osz      # tests/oracle_sizes.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sizes import crit_cfg, default_iteration_digests, make_iteration  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

pytestmark = pytest.mark.gpu
OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


# ---- the matcher --------------------------------------------------------------------------------------------------------------
def _device_pairs(match, l, b, n):
    """(group, Gmax) matched queries of one image -> (query indices, target indices) in the order scipy's result is stored."""
    src, tgt = [], []
    for g in range(match.shape[2]):
        pairs = sorted((int(match[l, b, g, j]), j) for j in range(n) if match[l, b, g, j] >= 0)
        src += [q for q, _ in pairs]
        tgt += [j for _, j in pairs]
    return np.array(src, np.int64), np.array(tgt, np.int64)


@pytest.mark.parametrize("L", [1, 6])
@pytest.mark.parametrize("nq", [1, 63, 64, 65, 100, 300])
def test_matcher_equals_scipy(nq, L):
    """Every (layer, image, group) assignment index for index against scipy's on the oracle's cost matrices.  The images have
    0, 1, 50 and 64 targets, so that both the targets (nt <= nq) and the queries (nt > nq) are the rows."""
    from monodetr_b200 import criterion as mc
    counts, group = (0, 1, 50, 64), 2
    B = len(counts)
    out, padded = oc.synthetic_case(40 + nq + L, B, nq * group, Gmax=64, n_aux=L - 1, max_gt=1, empty_image=False)
    g = torch.Generator().manual_seed(nq)
    padded["mask_2d"] = torch.zeros(B, 64, dtype=torch.bool)
    for b, n in enumerate(counts):
        padded["mask_2d"][b, torch.randperm(64, generator=g)[:n]] = True
    layers = [out] + out["aux_outputs"]
    dev_layers = [{k: v.cuda() for k, v in d.items() if torch.is_tensor(v)} for d in layers]
    tgt = mc.pack_targets({k: v.cuda() for k, v in padded.items()}, torch.device("cuda"))
    st = mc._prepare(tgt)
    matcher = mc.build_matcher(crit_cfg({}))
    match, tclass = mc._match(matcher, dev_layers, tgt, st, group)
    match, tclass = match.cpu().numpy(), tclass.cpu().numpy()
    targets = oc.prepare_targets(padded)
    for l, d in enumerate(layers):
        ref = oc.hungarian_match({k: v for k, v in d.items() if k != "aux_outputs"}, targets, group)
        for b, (i, j) in enumerate(ref):
            src, tg = _device_pairs(match, l, b, counts[b])
            assert len(src) == min(counts[b], nq) * group, (l, b)
            assert np.array_equal(src, i.numpy()) and np.array_equal(tg, j.numpy()), (l, b)
            want = np.full(nq * group, 3)
            want[i.numpy()] = targets[b]["labels"][j].numpy()
            assert np.array_equal(tclass[l, b], want), (l, b)


def test_matcher_refuses_beyond_its_limits():
    from monodetr_b200 import criterion as mc
    out, padded = oc.synthetic_case(3, 2, 301, Gmax=64, n_aux=6, max_gt=5)
    tgt = mc.pack_targets({k: v.cuda() for k, v in padded.items()}, torch.device("cuda"))
    st = mc._prepare(tgt)
    matcher = mc.build_matcher(crit_cfg({}))
    layers = [{k: v.cuda() for k, v in d.items() if torch.is_tensor(v)} for d in [out] + out["aux_outputs"]]
    with pytest.raises(RuntimeError, match="mdb_criterion_match_f32"):
        mc._match(matcher, layers[:1], tgt, st, 1)                  # 301 queries per group
    with pytest.raises(RuntimeError, match="mdb_criterion_match_f32"):
        mc._match(matcher, layers, tgt, st, 7)                      # 7 layers (43 queries per group)
    crit = mc.build_criterion(crit_cfg({})).cuda()
    o = dict(layers[0], aux_outputs=layers[1:])
    with pytest.raises(ValueError, match="at most 5 auxiliary outputs"):
        crit(o, tgt)


def test_criterion_takes_the_queries_of_the_model_it_is_built_for():
    """build_criterion(cfg) with num_queries 100 matches 100 queries in one group as scipy does; one built from the loss settings
    alone keeps its 64-query limit; the library refuses more than 300 whatever the criterion allows."""
    from monodetr_b200.criterion import SetCriterion, build_criterion
    big, pb = oc.synthetic_case(43, 1, 100, n_aux=0)
    o = {k: v.cuda().requires_grad_(True) for k, v in big.items() if torch.is_tensor(v)}
    p = {k: v.cuda() for k, v in pb.items()}
    crit = build_criterion(crit_cfg({"num_queries": 100})).cuda().eval()
    assert crit.max_queries == 100
    crit(o, p)
    ref = oc.hungarian_match({k: v for k, v in big.items() if k != "aux_outputs"}, oc.prepare_targets(pb), 1)
    src, tgt = _device_pairs(crit.last_indices.cpu().numpy(), 0, 0, int(pb["mask_2d"][0].sum()))
    assert np.array_equal(src, ref[0][0].numpy()) and np.array_equal(tgt, ref[0][1].numpy())
    assert build_criterion(crit_cfg({})).max_queries == 64
    with pytest.raises(RuntimeError, match="at most 64"):
        build_criterion(crit_cfg({})).cuda().eval()(o, p)
    with pytest.raises(NotImplementedError):
        SetCriterion(3, None, {}, 0.25, ["labels"], max_queries=301)


# ---- the criterion against the reference ----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def crit_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "criterion_sizes.npz"))


@pytest.mark.parametrize("name", list(osz.CRITERION_CASES))
def test_criterion_matches_the_reference(name, crit_golden):
    from monodetr_b200.criterion import build_criterion
    seed, counts, nq, group, L = osz.CRITERION_CASES[name]
    out, padded = osz.criterion_case(name)
    cfg = crit_cfg({"dec_layers": L, "aux_loss": L > 1, "num_queries": nq})
    crit = build_criterion(cfg).cuda().train(group > 1)

    def mv(d):
        return {k: v.cuda().requires_grad_(True) for k, v in d.items() if k != "aux_outputs"}
    o = mv(out)
    if L > 1:
        o["aux_outputs"] = [mv(a) for a in out["aux_outputs"]]
    p = {k: v.cuda() for k, v in padded.items()}
    losses = crit(o, p)
    total = sum(losses[k] * crit.weight_dict[k] for k in losses if k in crit.weight_dict)
    total.backward()
    torch.cuda.synchronize()
    keys = [k[len(name) + 6:] for k in crit_golden.files if k.startswith(f"{name}.loss.")]
    assert sorted(keys) == sorted(losses)
    m = crit.last_indices.cpu().numpy()
    assert m.shape[0] == L
    for l in range(L):
        for b, n in enumerate(counts):
            src, tgt = _device_pairs(m, l, b, n)
            assert np.array_equal(src, crit_golden[f"{name}.match.{l}.{b}.src"]), (l, b)
            assert np.array_equal(tgt, crit_golden[f"{name}.match.{l}.{b}.tgt"]), (l, b)
    for k in keys:
        np.testing.assert_allclose(float(losses[k]), float(crit_golden[f"{name}.loss.{k}"]), rtol=2e-5, atol=1e-6, err_msg=k)
    np.testing.assert_allclose(float(total), float(crit_golden[f"{name}.total"]), rtol=2e-5)
    for layer, d in [("main", o)] + [(f"aux{i}", a) for i, a in enumerate(o.get("aux_outputs", []))]:
        for k, t in d.items():
            if not torch.is_tensor(t):
                continue
            full = t.grad.cpu().numpy() if t.grad is not None else np.zeros(tuple(t.shape), np.float32)
            got, g, gmax = oc.golden_grad(crit_golden, f"{name}.grad.{layer}.{k}", full)
            np.testing.assert_allclose(got, g, rtol=2e-4, atol=1e-9 + 2e-5 * gmax, err_msg=f"{layer}.{k}")


# ---- the model ----------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "sizes.npz"))


def _model(tag, load=True):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, dropout=0.0, **osz.VARIANTS[tag]))
    if load:
        m.load_state_dict(om.with_aliases(osz.deterministic_state_dict(osz.sizes_cfg(tag))))
    for mod in m.modules():              # the depth encoder hard-codes dropout 0.1 (depth_predictor.py:49-50)
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return m.cuda()


def _check(golden, prefix, out):
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_{k}", out[k].detach().float().cpu().numpy()), rtol=2e-2,
                                   atol=2e-3, err_msg=k)
    for i, a in enumerate(out.get("aux_outputs", [])):
        for k in a:
            np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_aux{i}_{k}", a[k].detach().float().cpu().numpy()),
                                       rtol=2e-2, atol=2e-3, err_msg=f"aux{i} {k}")


@pytest.mark.parametrize("tag", list(osz.VARIANTS))
def test_model_matches_the_reference(tag, golden):
    """Eval outputs at 192 x 640 (and, where the reference trains, train outputs at 96 x 320) against the unmodified reference."""
    cfg = osz.sizes_cfg(tag)
    m = _model(tag).eval()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
    assert len(out.get("aux_outputs", [])) == (cfg["dec_layers"] - 1 if cfg["aux_loss"] else 0)
    _check(golden, f"{tag}.fwd_eval", out)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
    assert out["pred_logits"].shape[1] == 11 * cfg["num_queries"]
    if f"{tag}.grad_names" in golden.files:
        _check(golden, f"{tag}.fwd_train", out)
    om.surrogate_loss(out).backward()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)


STAGES = ("backbone", "input_proj", "depth_predictor", "depthaware_transformer.encoder", "depthaware_transformer.decoder.layers",
          "depthaware_transformer.decoder", "depthaware_transformer", "query_embed", "tgt_embed", "refpoint_embed", "class_embed",
          "bbox_embed", "dim_embed_3d", "angle_embed", "depth_embed")


@pytest.mark.parametrize("tag", list(osz.VARIANTS))
def test_gradients_per_stage(tag):
    """Frozen sampling locations, 192 x 640, B = 2: every gradient against the CPU oracle, with the bars of
    tests/test_points_gpu.py (median < 1e-3; every tensor < 2e-2, query_embed < 5e-2; max-norm and L2)."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    cfg = osz.sizes_cfg(tag)
    sd0 = osz.deterministic_state_dict(cfg)
    m = _model(tag, load=False)
    m.load_state_dict(om.with_aliases(sd0))
    m.train()
    images, calibs, sizes = om.synthetic_inputs(2, 11, H=192, W=640)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd0.items()}
        om.surrogate_loss(osz.forward(sd, images, calibs, sizes, training=True, cfg=cfg)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    params = dict(m.named_parameters())
    for name, p in params.items():        # analytically zero (see tests/test_backbone_variants_gpu.py)
        if name.endswith(("sa_kcontent_proj.bias", "sa_kpos_proj.bias")) and p.grad is not None:
            wmax = float(params[name[:-len("bias")] + "weight"].grad.abs().max())
            assert float(p.grad.abs().max()) <= 5e-3 * wmax and float(sd[name].grad.abs().max()) <= 1e-4 * wmax, name
            p.grad = None
    by_name = om.with_aliases(sd)
    per_stage, rel_max, rel_l2 = {}, [], []
    for name, p in m.named_parameters():
        if not p.requires_grad or p.grad is None:
            continue
        gref = by_name[name].grad
        assert gref is not None, name
        scale = float(gref.abs().max())
        if scale < 1e-7:
            continue
        d = p.grad.cpu() - gref
        r, l2 = float(d.abs().max()) / scale, float(d.norm() / gref.norm())
        rel_max.append(r)
        rel_l2.append(l2)
        stage = "query_embed" if name.startswith("depthaware_transformer.decoder.query_scale.") else \
            next(s for s in STAGES if name.startswith(s))
        cur = per_stage.get(stage, (0.0, 0.0, ""))
        per_stage[stage] = (max(cur[0], r), max(cur[1], l2), name if r > cur[0] else cur[2])
    print(tag, {k: f"{v[0]:.1e} {v[1]:.1e}" for k, v in per_stage.items()},
          "median", f"{float(np.median(rel_max)):.2e} {float(np.median(rel_l2)):.2e}", "tensors", len(rel_max))
    assert len(rel_max) > 100
    assert float(np.median(rel_max)) < 1e-3 and float(np.median(rel_l2)) < 1e-3
    for stage, (r, l2, name) in per_stage.items():
        assert r < (5e-2 if stage == "query_embed" else 2e-2) and l2 < 2e-2, (stage, name, r, l2)


# ---- training iterations ------------------------------------------------------------------------------------------------------
def _assert_equal(a, b):
    for name, xs, ys in zip(("outputs", "losses", "gradients", "parameters"), a, b):
        assert len(xs) == len(ys), name
        assert all(bool(torch.isfinite(x).all()) for x in xs), name
        bad = [i for i, (x, y) in enumerate(zip(xs, ys)) if not torch.equal(x, y)]
        assert not bad, (name, len(bad), len(xs))


@pytest.mark.parametrize("tag", ["deep", "q300"])
def test_training_iteration_as_a_cuda_graph_is_bit_identical(tag):
    """Reproducible mode: a replayed CUDA graph of the training iteration (forward with dropout, the device criterion over every
    decoder layer, backward, FusedAdamW) gives the bits of the same iteration run eagerly."""
    import monodetr_b200
    from monodetr_b200 import kernels as K, tc
    dev = torch.device("cuda", torch.cuda.current_device())
    prev, prev_prec = monodetr_b200.set_deterministic(True), tc.get_precision()
    tc.set_precision("bf16x3")
    kw = osz.VARIANTS[tag]
    try:
        _, it_a, snap_a = make_iteration(dev, kw)
        bucket_b, it_b, snap_b = make_iteration(dev, kw)
        K.reseed(dev, 99)
        for _ in range(3):
            it_a()
        eager = snap_a()
        K.reseed(dev, 99)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                it_b()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            it_b()
        bucket_b.freeze_sources()
        graph.replay()
        torch.cuda.synchronize()
        got = snap_b()
        _assert_equal(eager, got)
        assert len(eager[1]) == 10 + 8 * (kw.get("dec_layers", 3) - 1)       # the loss dict covers every decoder layer
        assert eager[0][0].shape[1] == 11 * kw.get("num_queries", 50)
    finally:
        tc.set_precision(prev_prec)
        monodetr_b200.set_deterministic(prev)


def test_default_iteration_is_byte_identical_to_the_fixed_size_matcher():
    """At the default configuration the training iteration's outputs, losses, gradients and updated parameters are the bytes
    recorded with the build whose matcher held a fixed 64 x 64 double cost matrix (tests/golden/sizes_default_step.json, written
    by `tools/bench_sizes.py --child digests` on an H100 80GB HBM3 with that build): the dynamic shared-memory matcher and the
    new stream indices leave the default path unchanged."""
    with open(os.path.join(os.path.dirname(__file__), "golden", "sizes_default_step.json")) as f:
        want = json.load(f)
    got = default_iteration_digests(torch.device("cuda", torch.cuda.current_device()))
    assert got == want


# ---- inference at 300 queries -----------------------------------------------------------------------------------------------
def test_tester_at_300_queries(tmp_path, monkeypatch):
    """Tester.inference() + evaluate() at num_queries 300 (900 decode candidates per image) against decode_detections +
    the reference-format files + kitti_eval.evaluate, as tests/test_validation_gpu.py checks the default model."""
    import types
    from monodetr_b200 import decode, tester
    from monodetr_b200 import kitti_eval as ke
    from test_validation_gpu import NAMES, Log, _Loader, labels_near, write_file_path
    model = _model("q300").eval()
    n_img, B = 4, 2
    images, calibs, sizes = om.synthetic_inputs(n_img, 3, H=192, W=640)
    ids = [2, 5, 9, 11]
    batches = [(images[b:b + B], calibs[b:b + B], {}, {"img_id": torch.tensor(ids[b:b + B]), "img_size": sizes[b:b + B]})
               for b in range(0, n_img, B)]
    with torch.no_grad():
        outs = [model(x.cuda(), c.cuda(), None, s["img_size"].cuda()) for x, c, _, s in batches]
    assert outs[0]["pred_logits"].shape[1:] == (300, 3)
    mean = np.zeros((3, 3), np.float32)
    write_file_path(str(tmp_path / "ref"), [(o, s["img_size"].cuda(), c.cuda()) for o, (_, c, _, s) in zip(outs, batches)],
                    [ids[b:b + B] for b in range(0, n_img, B)], mean, thr=0.0)
    os.makedirs(tmp_path / "label_2")
    for i, text in zip(ids, labels_near(ke.get_label_annos(str(tmp_path / "ref")), np.random.default_rng(4))):
        (tmp_path / "label_2" / ("%06d.txt" % i)).write_text(text)
    ds = types.SimpleNamespace(idx_list=["%06d" % i for i in ids], label_dir=str(tmp_path / "label_2"), writelist=["Car"],
                               class_name=NAMES, cls_mean_size=mean, split="val", max_objs=50)
    monkeypatch.chdir(tmp_path)
    log = Log()
    t = tester.Tester({"topk": 50, "threshold": 0.0}, model, _Loader(ds, batches), log, {"save_path": "out/"})
    was = torch.is_grad_enabled()
    try:
        t.inference()
    finally:
        torch.set_grad_enabled(was)
    car = t.evaluate()
    ref_log = Log()
    ref = ke.evaluate(str(tmp_path / "ref"), ds.label_dir, ids, ["Car"], ref_log)
    assert car == ref and log.lines == ["==> Saving ..."] + ref_log.lines
    for i in ids:
        name = "%06d.txt" % i
        assert (tmp_path / "out" / "monodetr" / "outputs" / "data" / name).read_bytes() == (tmp_path / "ref" / name).read_bytes()
    dets = decode.extract_dets_from_outputs(outs[0], topk=50)
    assert dets.shape[:2] == (B, 50)
