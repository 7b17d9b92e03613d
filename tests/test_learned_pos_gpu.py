"""GPU: the learned position embedding (`position_embedding: 'learned'`) -- its kernels (csrc/pos_embed.cu) against the unmodified
reference (tests/golden/learned_pos.npz) and fp64, the whole model against the fixture, per-stage gradients against the CPU oracle
(tests/oracle_learned_pos.py) alone and with use_dab / DC5, a bit-reproducible training iteration, eager and as a replayed CUDA
graph, and `Trainer` / `Tester` on a learned-embedding model."""
import os
import sys
import types

import numpy as np
import pytest
import torch

import monodetr_b200
from oracle import monodetr_torch as om
import oracle_backbones as ob    # tests/oracle_backbones.py
import oracle_dab as od          # tests/oracle_dab.py
import oracle_learned_pos as ol  # tests/oracle_learned_pos.py

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from gen_golden_reference_pins import sampled_forward  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "learned_pos.npz"))


def _upstream(h, w):
    """The fixture's seeded upstream gradient (oracle_learned_pos.upstream_grad) in the (h*w, 256) layout."""
    return ol.upstream_grad(h, w)[0].permute(1, 2, 0).reshape(h * w, 256).contiguous()


# ---- kernels -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w", ol.SHAPES)
def test_kernels_against_the_reference_and_fp64(h, w, golden):
    """Forward bit-identical to the reference's table (its SHA-256 per axis); backward within 1e-5 of max|grad| of the fp64
    gradient and of the reference's fp32 one at the stored positions, and the same bits on a second run.  One launch each way."""
    from monodetr_b200 import _lib, functional as Fn
    col_cpu, row_cpu = ol.module_tables()
    col, row = col_cpu.cuda().requires_grad_(True), row_cpu.cuda().requires_grad_(True)
    tag = f"mod.{h}x{w}"
    n0 = _lib.launch_count()
    out = Fn.pos_learned(col, row, h, w)
    assert _lib.launch_count() - n0 == 1
    assert out.shape == (h * w, 256)
    t = out.detach().cpu().view(h, w, 256)
    x_emb, y_emb = t[0, :, :128], t[:, 0, 128:]
    assert torch.equal(t, torch.cat([x_emb.unsqueeze(0).expand(h, -1, -1), y_emb.unsqueeze(1).expand(-1, w, -1)], -1))
    want_x, want_y = ol.axis_embeds(col_cpu, row_cpu, h, w)        # the CPU oracle: equal to the fixture's digests on the CPU
    assert np.array_equal(ol.digest(x_emb), golden[tag + ".x_sha"]), float((x_emb - want_x).abs().max())
    assert np.array_equal(ol.digest(y_emb), golden[tag + ".y_sha"]), float((y_emb - want_y).abs().max())
    g = _upstream(h, w).cuda()
    out.backward(g)
    assert _lib.launch_count() - n0 == 2
    c64 = col.detach().double().requires_grad_(True)
    r64 = row.detach().double().requires_grad_(True)
    ol.table_nhwc(c64, r64, h, w).backward(g.double())
    for got, ref64, key in ((col.grad, c64.grad, "dcol"), (row.grad, r64.grad, "drow")):
        scale = float(ref64.abs().max())
        assert float((got.double() - ref64).abs().max()) <= 1e-5 * scale, key
        idx = torch.from_numpy(golden[f"{tag}.{key}.idx"]).long()
        ref32 = torch.from_numpy(golden[f"{tag}.{key}.val"])
        assert idx.numel() > 0 and float((got.reshape(-1).cpu()[idx] - ref32).abs().max()) <= 1e-5 * scale, key
    first = (col.grad.clone(), row.grad.clone())
    col.grad = row.grad = None
    Fn.pos_learned(col, row, h, w).backward(g)
    assert torch.equal(col.grad, first[0]) and torch.equal(row.grad, first[1])
    with torch.no_grad():
        assert Fn.pos_learned(col, row, h, w).grad_fn is None


# ---- the whole model ---------------------------------------------------------------------------------------------------------
def _model(dropout=0.0, **kw):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, position_embedding="learned", dropout=dropout, **kw))
    if kw.get("use_dab"):
        sd = ol.with_tables(od.deterministic_state_dict())
    else:
        sd = ol.with_tables(ob.deterministic_state_dict(ob.variant_cfg("resnet50", kw.get("dilation", False))))
    m.load_state_dict(om.with_aliases(sd))
    if dropout == 0.0:
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
            if isinstance(mod, torch.nn.MultiheadAttention):
                mod.dropout = 0.0
    return m.cuda(), sd


def _flat(out):
    items = [(k, out[k]) for k in ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")]
    items += [(f"aux{i}_{k}", v) for i, a in enumerate(out["aux_outputs"]) for k, v in a.items()]
    return items


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
def test_model_matches_the_reference(precision, golden):
    """Eval at 1 x 192 x 640, train mode (dropout off) at 1 and 2 x 96 x 320: every output incl. aux within 1e-3
    (max|a - b| / max|b| over the stored elements)."""
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(precision)
    try:
        m, _ = _model()
        for training, B, (H, W), prefix in ((False, 1, (192, 640), "fwd_eval"), (True, 1, (96, 320), "b1.fwd_train"),
                                            (True, 2, (96, 320), "b2.fwd_train")):
            m.train(training)
            images, calibs, sizes = om.synthetic_inputs(B, 0, H=H, W=W)
            with torch.no_grad():
                out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
            worst = []
            for k, v in _flat(out):
                a, b = sampled_forward(golden, f"{prefix}_{k}", v.float().cpu().numpy())
                rel = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))
                worst.append((rel, k))
                assert rel < 1e-3, (prefix, k, rel)
            print(precision, prefix, "worst", max(worst))
    finally:
        tc.set_precision(prev)


STAGES = ("backbone.1", "backbone.0", "input_proj", "depth_predictor", "depthaware_transformer.encoder",
          "depthaware_transformer.decoder", "depthaware_transformer.level_embed", "depthaware_transformer.reference_points",
          "query_embed", "tgt_embed", "refpoint_embed", "class_embed", "bbox_embed", "dim_embed_3d", "angle_embed", "depth_embed")


def _per_stage(m, sd, oracle_forward, B, H, W, **kw):
    """Frozen sampling locations: every gradient of the surrogate loss against the CPU oracle's -> {stage: (max-norm, L2, worst
    name)}, with the median max-norm / L2 errors, as tests/test_dab_gpu.py measures them."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    m.train()
    images, calibs, sizes = om.synthetic_inputs(B, 11, H=H, W=W)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sdg = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
        om.surrogate_loss(ol.forward(sdg, images, calibs, sizes, training=True, base=oracle_forward, **kw)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    params = dict(m.named_parameters())
    for name, p in params.items():        # analytically zero (see tests/test_backbone_variants_gpu.py)
        if name.endswith(("sa_kcontent_proj.bias", "sa_kpos_proj.bias")) and p.grad is not None:
            wmax = float(params[name[:-len("bias")] + "weight"].grad.abs().max())
            assert float(p.grad.abs().max()) <= 5e-3 * wmax and float(sdg[name].grad.abs().max()) <= 1e-4 * wmax, name
            p.grad = None
    per_stage, rel_max, rel_l2 = {}, [], []
    for name, p in m.named_parameters():
        if name.startswith(("depthaware_transformer.decoder.bbox_embed", "depthaware_transformer.decoder.dim_embed")):
            continue
        if not p.requires_grad or p.grad is None:
            continue
        gref = sdg[name].grad
        assert gref is not None, name
        scale = float(gref.abs().max())
        if scale < 1e-7:
            continue
        d = p.grad.cpu() - gref
        r, l2 = float(d.abs().max()) / scale, float(d.norm() / gref.norm())
        rel_max.append(r)
        rel_l2.append(l2)
        stage = next(s for s in STAGES if name.startswith(s))
        cur = per_stage.get(stage, (0.0, 0.0, ""))
        per_stage[stage] = (max(cur[0], r), max(cur[1], l2), name if r > cur[0] else cur[2])
    print(B, {k: f"{v[0]:.1e} {v[1]:.1e}" for k, v in per_stage.items()},
          "median", f"{float(np.median(rel_max)):.2e} {float(np.median(rel_l2)):.2e}", "tensors", len(rel_max))
    return per_stage, float(np.median(rel_max)), float(np.median(rel_l2))


def _assert_bars(per_stage, med_max, med_l2):
    assert "backbone.1" in per_stage
    assert med_max < 1e-3 and med_l2 < 1e-3
    for stage, (r, l2, name) in per_stage.items():
        assert r < 2e-2 and l2 < 2e-2, (stage, name, r, l2)


@pytest.mark.parametrize("B", [1, 2])
def test_gradients_per_stage(B):
    """The bars of tests/test_model_grad_gpu.py (median < 1e-3, every tensor < 2e-2, max-norm and L2), both tables included."""
    m, sd = _model()
    _assert_bars(*_per_stage(m, sd, om.forward, B, 192, 640))
    for name in (ol.ROW, ol.COL):
        assert dict(m.named_parameters())[name].grad is not None


@pytest.mark.parametrize("variant", ["use_dab", "dc5"])
def test_with_anchor_boxes_and_with_dc5(variant):
    """use_dab + learned and DC5 + learned against the oracle composed the same way, at 1 x 192 x 640 (the size of the suite's
    per-stage bars: at 96 x 320 a few ResNet weight gradients exceed 2e-2, the tail DESIGN.md attributes to ReLU / max-pool
    selections flipping on 1e-6 forward noise)."""
    if variant == "use_dab":
        m, sd = _model(use_dab=True)
        per_stage, med_max, med_l2 = _per_stage(m, sd, od.forward, 1, 192, 640)
        # with both branches the worst max-norm error sits in the decoder's query_scale weight (3.1e-2 on an H100, L2 5e-3):
        # that stage is held to the L2 bar and to 5e-2 in max-norm, the tables and every other stage to the full bars
        r, l2, name = per_stage.pop("depthaware_transformer.decoder")
        assert r < 5e-2 and l2 < 2e-2, (name, r, l2)
    else:
        m, sd = _model(dilation=True)
        per_stage, med_max, med_l2 = _per_stage(m, sd, ob.forward, 1, 192, 640, cfg=ob.variant_cfg("resnet50", True))
    _assert_bars(per_stage, med_max, med_l2)


# ---- reproducible mode and graph capture ---------------------------------------------------------------------------------------
def _setup(dev, B=2):
    from bench_extras import CRIT_CFG, synthetic_targets
    from monodetr_b200 import build_monodetr, tc
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, position_embedding="learned", dropout=0.1))
    model = model.to(dev).train()
    crit = build_criterion(CRIT_CFG).to(dev).train()
    bucket = FlatGradBucket(model)
    opt = FusedAdamW(model, bucket, lr=2e-4, weight_decay=1e-4, device_step=True)
    images, calibs, sizes = (t.to(dev) for t in synthetic_batch(B, seed=77))
    tg = {k: v.to(dev) for k, v in synthetic_targets(77, B).items()}
    state = {}

    def it():
        bucket.zero()
        out = model(images, calibs, None, sizes)
        losses = crit(out, tg)
        crit.weighted_sum().backward()
        opt.step()
        state["out"], state["losses"] = out, losses

    def snapshot():
        out = state["out"]
        flat = [v for _, v in _flat(out)]
        losses = [state["losses"][k] for k in sorted(state["losses"])]
        grads = [p.grad for p in model.parameters() if p.grad is not None]
        return [t.detach().clone() for t in flat], [t.detach().clone() for t in losses], [t.clone() for t in grads], \
            [p.detach().clone() for p in model.parameters()]
    return model, bucket, it, snapshot


def _assert_equal(a, b):
    for name, xs, ys in zip(("outputs", "losses", "gradients", "parameters"), a, b):
        assert len(xs) == len(ys), name
        bad = [i for i, (x, y) in enumerate(zip(xs, ys)) if not torch.equal(x, y)]
        assert not bad, (name, len(bad), len(xs))


def test_training_iteration_is_bit_reproducible_eager_and_as_a_cuda_graph():
    """Reproducible mode: forward with dropout, the device criterion, backward and FusedAdamW give identical bits twice eagerly,
    and a replayed CUDA graph of the whole iteration (captured without a host synchronisation) gives the eager bits."""
    from monodetr_b200 import kernels as K
    dev = torch.device("cuda", torch.cuda.current_device())
    prev = monodetr_b200.set_deterministic(True)
    try:
        runs = []
        for _ in range(2):
            model, bucket, it, snap = _setup(dev)
            K.reseed(dev, 4242)
            it()
            runs.append(snap())
        assert len(bucket.names) == 315
        assert model.backbone[1].row_embed.weight.grad is not None and model.backbone[1].col_embed.weight.grad is not None
        _assert_equal(runs[0], runs[1])

        _, _, it_a, snap_a = _setup(dev)
        _, bucket_b, it_b, snap_b = _setup(dev)
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
        torch.cuda.set_sync_debug_mode("error")
        try:
            with torch.cuda.graph(graph):
                it_b()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        bucket_b.freeze_sources()
        graph.replay()
        torch.cuda.synchronize()
        _assert_equal(eager, snap_b())
    finally:
        monodetr_b200.set_deterministic(prev)


# ---- Trainer and Tester --------------------------------------------------------------------------------------------------------
def _trainer(max_graphs=None):
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr, kernels as K, tc
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    from monodetr_b200.trainer import Trainer
    import trainer_stubs as S
    from test_trainer_gpu import CFG, H, SCHED, W, _loader
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, position_embedding="learned", dropout=0.1))
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    crit.depth_map_scale = (W // 16, H // 16)
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler(SCHED, opt, last_epoch=-1)
    tr = Trainer(CFG, model, opt, _loader(), None, sched, warm, S.ListLogger(), crit, "m")
    if max_graphs is not None:
        tr.MAX_GRAPHS = max_graphs
    tr.PRINT_EVERY = 1
    K.reseed(torch.device("cuda", torch.cuda.current_device()), 4242)
    return tr


def test_trainer_graph_path_and_tester(tmp_path, monkeypatch):
    """Reproducible mode: an epoch of four batches through Trainer's replayed graphs leaves every parameter, both tables included,
    equal to the same epoch run eagerly (the suite's bar for this comparison is bit equality); Tester then validates the trained
    model on a small labelled set."""
    from monodetr_b200 import kitti_eval as ke, tester, trainer as T
    from test_validation_gpu import NAMES, Log, _Loader, labels_near, write_file_path
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(T, "print_losses", lambda i, log: None)
    prev = monodetr_b200.set_deterministic(True)
    try:
        trained = {}
        for name, max_graphs in (("graph", None), ("eager", 0)):
            tr = _trainer(max_graphs)
            init = {n: p.detach().clone() for n, p in tr.model.named_parameters() if n in (ol.ROW, ol.COL)}
            tr.train_one_epoch(0)
            torch.cuda.synchronize()
            assert tr.graph_path and (tr.live_graphs > 0) == (max_graphs is None)
            for n, p in tr.model.named_parameters():
                if n in init:
                    assert not torch.equal(p.detach(), init[n]), n                            # the tables trained
            trained[name] = tr
        pg = dict(trained["graph"].model.named_parameters())
        pe = dict(trained["eager"].model.named_parameters())
        bad = [n for n in pg if not torch.equal(pg[n], pe[n])]
        assert not bad, bad[:5]
    finally:
        monodetr_b200.set_deterministic(prev)

    model = trained["graph"].model.eval()
    ids, B = [1, 5, 9, 12], 2
    images, calibs, sizes = om.synthetic_inputs(len(ids), 3, H=96, W=320)
    batches = [(images[b:b + B].cuda(), calibs[b:b + B].cuda(), {}, {"img_id": torch.tensor(ids[b:b + B]), "img_size": sizes[b:b + B].cuda()})
               for b in range(0, len(ids), B)]
    with torch.no_grad():
        outs = [model(x, c, None, s["img_size"]) for x, c, _, s in batches]
    mean = np.zeros((3, 3), np.float32)
    write_file_path(str(tmp_path / "ref"), [(o, s["img_size"], c) for o, (_, c, _, s) in zip(outs, batches)],
                    [ids[b:b + B] for b in range(0, len(ids), B)], mean, thr=0.0)
    os.makedirs(tmp_path / "label_2")
    for i, text in zip(ids, labels_near(ke.get_label_annos(str(tmp_path / "ref")), np.random.default_rng(2))):
        (tmp_path / "label_2" / ("%06d.txt" % i)).write_text(text)
    ds = types.SimpleNamespace(idx_list=["%06d" % i for i in ids], label_dir=str(tmp_path / "label_2"), writelist=["Car"],
                               class_name=NAMES, cls_mean_size=mean, split="val", max_objs=50)
    log = Log()
    t = tester.Tester({"topk": 50, "threshold": 0.0}, model, _Loader(ds, batches), log, {"save_path": "out/"})
    was = torch.is_grad_enabled()
    try:
        t.inference()
    finally:
        torch.set_grad_enabled(was)
    car = t.evaluate()
    ref_log = Log()
    assert car == ke.evaluate(str(tmp_path / "ref"), ds.label_dir, ids, ["Car"], ref_log)
    assert log.lines == ["==> Saving ..."] + ref_log.lines
