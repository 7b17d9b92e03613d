"""GPU: the reference's other head counts (cfg `nheads` 4 and 16: attention head widths 64 and 16) on the sm_90a kernels --
both models against the unmodified reference (tests/golden/nheads.npz) at the bars of tests/test_backbone_variants_gpu.py,
per-stage gradients against the CPU oracle (tests/oracle_nheads.py), and two reproducible-mode training iterations giving
the same bits."""
import os
import sys

import numpy as np
import pytest
import torch

import oracle_nheads as on      # tests/oracle_nheads.py
from oracle import monodetr_torch as om

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_nheads import VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402


def _model(nheads, dropout=0.0):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, nheads=nheads, dropout=dropout))
    m.load_state_dict(om.with_aliases(on.deterministic_state_dict(on.heads_cfg(nheads))))
    if dropout == 0.0:
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
    return np.load(os.path.join(golden_dir, "nheads.npz"))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
@pytest.mark.parametrize("tag", list(VARIANTS))
def test_model_matches_the_reference(tag, precision, golden):
    """Eval outputs at 192 x 640 and train-mode outputs (dropout off) at 96 x 320, every output incl. aux within 1e-3
    (max|a - b| / max|b| over the stored elements)."""
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(precision)
    try:
        m = _model(VARIANTS[tag])
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


@pytest.mark.parametrize("nheads", [4, 16])
def test_gradients_per_stage(nheads):
    """Frozen sampling locations, 192 x 640, B = 1: the bars of tests/test_model_grad_gpu.py."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    from test_model_grad_gpu import _grad_report
    cfg = on.heads_cfg(nheads)
    m = _model(nheads).train()
    images, calibs, sizes = om.synthetic_inputs(1, 11, H=192, W=640)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in on.deterministic_state_dict(cfg).items()}
        om.surrogate_loss(on.forward(sd, images, calibs, sizes, training=True, cfg=cfg)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    # The key-projection biases of the decoder's self-attention have an analytically zero gradient: both sides give
    # cancellation noise there, held against the weight's gradient (as tests/test_backbone_variants_gpu.py does).
    params = dict(m.named_parameters())
    for name, p in params.items():
        if name.endswith(("sa_kcontent_proj.bias", "sa_kpos_proj.bias")) and p.grad is not None:
            wmax = float(params[name[:-len("bias")] + "weight"].grad.abs().max())
            assert float(p.grad.abs().max()) <= 5e-3 * wmax and float(sd[name].grad.abs().max()) <= 1e-4 * wmax, name
            p.grad = None
    per_stage, rel_max, rel_l2 = _grad_report(m, sd)
    print(nheads, {k: f"{v[0]:.1e} {v[1]:.1e}" for k, v in per_stage.items()},
          "median", f"{float(np.median(rel_max)):.2e} {float(np.median(rel_l2)):.2e}", "tensors", len(rel_max))
    assert len(rel_max) > 240
    assert float(np.median(rel_max)) < 1e-3 and float(np.median(rel_l2)) < 1e-3
    for stage, (r, l2, name) in per_stage.items():
        assert r < (5e-2 if stage == "query_embed" else 2e-2) and l2 < 2e-2, (stage, name, r, l2)


@pytest.mark.parametrize("nheads", [4, 16])
def test_training_iteration_is_bit_reproducible(nheads):
    """Reproducible mode: forward with dropout, the device criterion, backward and FusedAdamW, twice from the same state."""
    import monodetr_b200
    from bench_extras import CRIT_CFG, synthetic_targets
    from monodetr_b200 import build_monodetr, kernels as K, tc
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW
    dev = torch.device("cuda", torch.cuda.current_device())
    prev = monodetr_b200.set_deterministic(True)
    prev_prec = tc.get_precision()
    tc.set_precision("bf16x3")
    try:
        runs = []
        for _ in range(2):
            torch.manual_seed(0)
            model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, nheads=nheads, dropout=0.1))
            model = model.to(dev).train()
            crit = build_criterion(CRIT_CFG).to(dev).train()
            bucket = FlatGradBucket(model)
            opt = FusedAdamW(model, bucket, lr=2e-4, weight_decay=1e-4, device_step=True)
            images, calibs, sizes = (t.to(dev) for t in synthetic_batch(2, seed=77))
            tg = {k: v.to(dev) for k, v in synthetic_targets(77, 2).items()}
            K.reseed(dev, 4242)
            for _ in range(2):
                bucket.zero()
                out = model(images, calibs, None, sizes)
                losses = crit(out, tg)
                crit.weighted_sum().backward()
                opt.step()
            runs.append(([v.detach().clone() for _, v in _flat(out)], [losses[k].detach().clone() for k in sorted(losses)],
                         [p.grad.clone() for p in model.parameters() if p.grad is not None],
                         [p.detach().clone() for p in model.parameters()]))
        assert len(runs[0][2]) == 313
        for name, xs, ys in zip(("outputs", "losses", "gradients", "parameters"), runs[0], runs[1]):
            assert all(bool(torch.isfinite(x).all()) for x in xs), name
            bad = [i for i, (a, b) in enumerate(zip(xs, ys)) if not torch.equal(a, b)]
            assert not bad, (name, len(bad), len(xs))
    finally:
        tc.set_precision(prev_prec)
        monodetr_b200.set_deterministic(prev)
