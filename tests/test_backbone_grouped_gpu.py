"""GPU: the reference's ResNeXt and wide-ResNet backbones on the sm_90a kernels (grouped 3x3s on the channel-banded GEMM).

- resnext50_32x4d, resnext50_32x4d + DC5 and wide_resnet50_2 against the unmodified reference
  (tests/golden/backbones_grouped.npz) at the whole-model 1e-3 bar;
- resnext101_32x8d, resnext101_64x4d and wide_resnet101_2 against the CPU oracle;
- per-stage gradients with frozen sampling locations at the bars of tests/test_model_grad_gpu.py;
- a reproducible-mode resnext50_32x4d training iteration twice, and as a replayed CUDA graph, bit for bit;
- one training iteration of every new (backbone, dilation).
"""
import os
import sys

import numpy as np
import pytest
import torch

import oracle_backbones_grouped as obg     # tests/oracle_backbones_grouped.py
from oracle import monodetr_torch as om

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sizes import make_iteration  # noqa: E402
from gen_golden_backbones_grouped import NAMES, VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402


def _model(backbone, dilation):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, backbone=backbone, dilation=dilation, dropout=0.0))
    m.load_state_dict(om.with_aliases(obg.deterministic_state_dict(obg.variant_cfg(backbone, dilation))))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return m.cuda()


def _flat(out):
    items = [(k, out[k]) for k in ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")]
    items += [(f"aux{i}_{k}", v) for i, a in enumerate(out["aux_outputs"]) for k, v in a.items()]
    return items


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "backbones_grouped.npz"))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
@pytest.mark.parametrize("tag", list(VARIANTS))
def test_model_matches_the_reference(tag, precision, golden):
    """Eval outputs at 192 x 640 and train-mode outputs (dropout off) at 96 x 320, every output incl. aux within 1e-3."""
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(precision)
    try:
        m = _model(*VARIANTS[tag])
        for training, (H, W) in ((False, (192, 640)), (True, (96, 320))):
            m.train(training)
            images, calibs, sizes = om.synthetic_inputs(1, 0, H=H, W=W)
            with torch.no_grad():
                out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
            prefix = f"{tag}.fwd_{'train' if training else 'eval'}"
            worst = []
            for k, v in _flat(out):
                a, b = sampled_forward(golden, f"{prefix}_{k}", v.float().cpu().numpy())
                rel = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))
                worst.append((rel, k))
                assert rel < 1e-3, (prefix, k, rel)
            print(tag, precision, prefix, "worst", max(worst))
    finally:
        tc.set_precision(prev)


@pytest.mark.parametrize("backbone", ["resnext101_32x8d", "resnext101_64x4d", "wide_resnet101_2"])
def test_deep_variants_match_the_oracle(backbone):
    cfg = obg.variant_cfg(backbone, False)
    m = _model(backbone, False).eval()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        ref = obg.forward(obg.deterministic_state_dict(cfg), images, calibs, sizes, training=False, cfg=cfg)
    for (k, a), (_, b) in zip(_flat(out), _flat(ref)):
        rel = float((a.float().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-12))
        assert rel < 1e-3, (k, rel)


@pytest.mark.parametrize("backbone,dilation", [("resnext50_32x4d", False), ("resnext50_32x4d", True), ("wide_resnet50_2", False)])
def test_gradients_per_stage(backbone, dilation):
    """Frozen sampling locations, 192 x 640, B = 1: the bars of tests/test_model_grad_gpu.py."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    from test_model_grad_gpu import _grad_report
    cfg = obg.variant_cfg(backbone, dilation)
    m = _model(backbone, dilation).train()
    images, calibs, sizes = om.synthetic_inputs(1, 11, H=192, W=640)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in obg.deterministic_state_dict(cfg).items()}
        om.surrogate_loss(obg.forward(sd, images, calibs, sizes, training=True, cfg=cfg)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    # analytically zero key-bias gradients: cancellation noise on both sides, held against the weight's gradient (as in
    # tests/test_backbone_variants_gpu.py)
    params = dict(m.named_parameters())
    for name, p in params.items():
        if name.endswith(("sa_kcontent_proj.bias", "sa_kpos_proj.bias")) and p.grad is not None:
            wmax = float(params[name[:-len("bias")] + "weight"].grad.abs().max())
            assert float(p.grad.abs().max()) <= 5e-3 * wmax and float(sd[name].grad.abs().max()) <= 1e-4 * wmax, name
            p.grad = None
    per_stage, rel_max, rel_l2 = _grad_report(m, sd)
    print(backbone, dilation, {k: f"{v[0]:.1e} {v[1]:.1e}" for k, v in per_stage.items()},
          "median", f"{float(np.median(rel_max)):.2e} {float(np.median(rel_l2)):.2e}", "tensors", len(rel_max))
    assert len(rel_max) > 240
    assert float(np.median(rel_max)) < 1e-3 and float(np.median(rel_l2)) < 1e-3
    for stage, (r, l2, name) in per_stage.items():
        assert r < (5e-2 if stage == "query_embed" else 2e-2) and l2 < 2e-2, (stage, name, r, l2)


def _assert_equal(a, b):
    for name, xs, ys in zip(("outputs", "losses", "gradients", "parameters"), a, b):
        assert len(xs) == len(ys), name
        assert all(bool(torch.isfinite(x).all()) for x in xs), name
        bad = [i for i, (x, y) in enumerate(zip(xs, ys)) if not torch.equal(x, y)]
        assert not bad, (name, len(bad), len(xs))


def test_training_iteration_is_bit_reproducible_and_graph_replayable():
    """Reproducible mode, resnext50_32x4d: two eager runs of the training iteration (forward with dropout, the device
    criterion, backward, FusedAdamW) give the same bits, and so does the iteration captured and replayed as a CUDA graph
    (what the Trainer replays)."""
    import monodetr_b200
    from monodetr_b200 import kernels as K, tc
    dev = torch.device("cuda", torch.cuda.current_device())
    prev, prev_prec = monodetr_b200.set_deterministic(True), tc.get_precision()
    tc.set_precision("bf16x3")
    kw = {"backbone": "resnext50_32x4d"}
    try:
        runs = []
        for _ in range(2):
            _, it, snap = make_iteration(dev, kw)
            K.reseed(dev, 99)
            for _ in range(3):
                it()
            runs.append(snap())
        _assert_equal(runs[0], runs[1])
        assert len(runs[0][2]) == 313
        bucket_b, it_b, snap_b = make_iteration(dev, kw)
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
        _assert_equal(runs[0], snap_b())
    finally:
        tc.set_precision(prev_prec)
        monodetr_b200.set_deterministic(prev)


@pytest.mark.parametrize("dilation", [False, True])
@pytest.mark.parametrize("backbone", NAMES)
def test_training_iteration_runs(backbone, dilation):
    """Every new backbone, with and without DC5: two training iterations at batch 2, finite outputs, losses and gradients,
    and every trainable backbone weight gets a gradient."""
    dev = torch.device("cuda", torch.cuda.current_device())
    _, it, snap = make_iteration(dev, {"backbone": backbone, "dilation": dilation}, hw=(192, 640))
    it()
    it()
    outs, losses, grads, _ = snap()
    for t in outs + losses + grads:
        assert bool(torch.isfinite(t).all())
    assert len(grads) == (313 if "50" in backbone else 364)
