"""GPU: the reference's other backbones on the sm_90a kernels.

1. The dilated 3x3 convolution of the tensor-core family (the `*_dilated` entry points, dilation 2, padding 2, stride 1: the
   dilated C5 stage of torchvision's ResNets) against fp64 torch convolutions at the per-element bound of
   tests/tc_error_model.py, in all three precision modes: forward with bias / residual / ReLU (TMA epilogue) and with a
   width that is not a multiple of 4 (register epilogue), data gradient with residual + ReLU mask, weight gradient + bias.
   Shapes cover partial row / column tiles, batches 1, 3 and 8, and both BF16x3 tile widths (256 -> 256 and 512 -> 512 at
   24 x 80, batch 8: 128 x 256 tiles).  Forward and data gradient are bit-reproducible and batch-independent; a dilated
   entry point with dilation 1 gives the plain entry point's bits; unsupported geometries raise.
2. Whole models: resnet50 + DC5, resnet101 and resnet101 + DC5 against the unmodified reference
   (tests/golden/backbones.npz), resnet152 against the CPU oracle; per-stage gradients against the oracle; and two
   reproducible-mode training iterations of resnet50 + DC5 give the same bits.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import oracle_backbones as ob     # tests/oracle_backbones.py
import tc_error_model as em
from oracle_backbones import variant_cfg
from oracle import monodetr_torch as om

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

MODES = ("bf16x3", "tf32x3", "tf32")
D = 2               # the DC5 dilation (padding = dilation, stride 1)


@pytest.fixture(params=MODES)
def mode(request):
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(request.param)
    yield request.param
    tc.set_precision(prev)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _pack(w):
    O, I, kh, kw = w.shape
    return w.permute(2, 3, 0, 1).reshape(kh * kw, O, I).contiguous()


def _operand(w, mode):
    from monodetr_b200 import tc
    return tc.split_weights([w])[0] if mode == "bf16x3" else _pack(w)


def _conv_f(a, b):
    taps, O, I = b.shape
    return F.conv2d(a.permute(0, 3, 1, 2), b.view(3, 3, O, I).permute(2, 3, 0, 1), padding=D, dilation=D).permute(0, 2, 3, 1)


def _dgrad_f(shape):
    def f(a, b):
        taps, O, I = b.shape
        B, H, W, C = shape
        return torch.nn.grad.conv2d_input((B, C, H, W), b.view(3, 3, O, I).permute(2, 3, 0, 1), a.permute(0, 3, 1, 2),
                                          padding=D, dilation=D).permute(0, 2, 3, 1)
    return f


def _wgrad_f(shape):
    def f(a, b):                                   # a = dy (B, H, W, Cout), b = x (B, H, W, Cin) -> (taps, Cout, Cin)
        Cout, Cin = a.shape[-1], b.shape[-1]
        g = torch.nn.grad.conv2d_weight(b.permute(0, 3, 1, 2), (Cout, Cin, 3, 3), a.permute(0, 3, 1, 2), padding=D, dilation=D)
        return g.permute(2, 3, 0, 1).reshape(9, Cout, Cin)
    return f


def _wide(N, B, H, W, kblocks):
    """pick_bn of conv_gemm.cu for a stride-1 'same' convolution (tests/test_gemm_wide_tile_gpu.py restates it in full)."""
    from test_gemm_wide_tile_gpu import _m_tiles, _wide as wide
    return wide(N, _m_tiles(W, H, B), kblocks)


# B, H, W, Cin, Cout: partial row tiles (13 x 29) and column tiles (200 = 128 + 72), batch 1 / 3 / 8, the model's layer-4
# width at the DC5 resolution (512 -> 512 at 24 x 80, batch 8: 144 k-blocks, 128 x 256 tiles in bf16x3) and a 256 -> 256
# that also runs wide.  Output widths that are not a multiple of 4 go through the register epilogue (forward only).
CONVS = [
    (1, 13, 29, 64, 200),
    (3, 24, 80, 128, 132),
    (8, 24, 80, 256, 256),
    (8, 24, 80, 512, 512),
]
RAGGED = [(3, 13, 29, 128, 250), (1, 24, 80, 512, 6)]


@pytest.mark.parametrize("cfg", CONVS + RAGGED)
def test_dilated_forward(mode, cfg):
    from monodetr_b200 import tc
    B, H, W, Cin, Cout = cfg
    if mode == "bf16x3" and cfg in ((8, 24, 80, 256, 256), (8, 24, 80, 512, 512)):
        assert _wide(Cout, B, H, W, 9 * Cin // 32)
    g = _gen(sum(cfg))
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (Cin * 9) ** 0.5
    bias = torch.randn(Cout, device="cuda", generator=g)
    t, s = em.target(_conv_f, x, _pack(w), mode)
    res = torch.randn(t.shape, device="cuda", generator=g)
    wo = _operand(w, mode)
    y = tc.conv2d_forward(x, wo, bias, res, 3, 3, 1, D, relu=True, dilation=D)
    assert y.shape == (B, H, W, Cout)
    em.assert_gemm(f"fwd d2 {cfg} +b+r+relu", y, torch.relu(t + bias.double() + res.double()), s, mode,
                   epi=em.epi_mag(t, bias, res))
    y = tc.conv2d_forward(x, wo, None, None, 3, 3, 1, D, dilation=D)
    em.assert_gemm(f"fwd d2 {cfg}", y, t, s, mode)


@pytest.mark.parametrize("cfg", CONVS)
def test_dilated_dgrad(mode, cfg):
    """Data gradient of a layer Cin -> Cout with residual + ReLU mask; cfg's last two entries are (Cout, Cin), so that the
    data gradient's output width Cin takes the widths the forward's Cout takes."""
    from monodetr_b200 import tc
    B, H, W, Cout, Cin = cfg
    if mode == "bf16x3" and cfg in ((8, 24, 80, 256, 256), (8, 24, 80, 512, 512)):
        assert _wide(Cin, B, H, W, 9 * Cout // 32)
    g = _gen(sum(cfg) + 1)
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (Cin * 9) ** 0.5
    x_shape = (B, H, W, Cin)
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    t, s = em.target(_dgrad_f(x_shape), dy, _pack(w), mode)
    r = torch.randn(x_shape, device="cuda", generator=g)
    mask = torch.randn(x_shape, device="cuda", generator=g)
    mask[..., ::3] = -0.0
    gate = (mask > 0).double()
    wo = _operand(w, mode)
    dx = tc.conv2d_dgrad(dy, wo, x_shape, r, mask, 3, 3, 1, D, dilation=D)
    em.assert_gemm(f"dgrad d2 {cfg} +r*mask", dx, (t + r.double()) * gate, s * gate, mode, epi=em.epi_mag(t, None, r) * gate)
    dx = tc.conv2d_dgrad(dy, wo, x_shape, None, None, 3, 3, 1, D, dilation=D)
    em.assert_gemm(f"dgrad d2 {cfg}", dx, t, s, mode)


@pytest.mark.parametrize("cfg", CONVS)
def test_dilated_wgrad(mode, cfg):
    from monodetr_b200 import tc
    B, H, W, Cin, Cout = cfg
    g = _gen(sum(cfg) + 2)
    x = torch.randn(B, H, W, Cin, device="cuda", generator=g)
    dy = torch.randn(B, H, W, Cout, device="cuda", generator=g)
    t, s = em.target(_wgrad_f(x.shape), dy, x, mode)
    dw, db = tc.conv2d_wgrad(dy, x, None, 3, 3, 1, D, with_bias_grad=True, dilation=D)
    em.assert_gemm(f"wgrad d2 {cfg}", dw, t, s, mode)
    ref_db = dy.double().sum((0, 1, 2))
    assert float((db.double() - ref_db).abs().max()) <= 1e-5 * float(dy.double().abs().sum((0, 1, 2)).max())


def test_dilated_bits():
    """Forward and data gradient: run to run, an image alone against the same image in batches of 3 and 8 (at batch 8 the
    512 -> 512 runs 128 x 256 tiles, alone 128-wide ones), and every _dilated entry point with dilation 1 against the plain
    entry point (the weight gradient in reproducible mode, where it is summed in one fixed order)."""
    import monodetr_b200
    from monodetr_b200 import _lib, tc
    g = _gen(9)
    prev_mode = tc.get_precision()
    for mode in MODES:
        tc.set_precision(mode)
        try:
            B, H, W, C = 8, 24, 80, 512
            x = torch.randn(B, H, W, C, device="cuda", generator=g)
            w = torch.randn(C, C, 3, 3, device="cuda", generator=g) / (C * 9) ** 0.5
            bias = torch.randn(C, device="cuda", generator=g)
            res = torch.randn(B, H, W, C, device="cuda", generator=g)
            mask = torch.randn(B, H, W, C, device="cuda", generator=g)
            wo = _operand(w, mode)
            fwd = lambda n: tc.conv2d_forward(x[:n].contiguous(), wo, bias, res[:n].contiguous(), 3, 3, 1, D, relu=True, dilation=D)
            bwd = lambda n: tc.conv2d_dgrad(x[:n].contiguous(), wo, (n, H, W, C), res[:n].contiguous(), mask[:n].contiguous(), 3, 3,
                                            1, D, dilation=D)
            y8, dx8 = fwd(8), bwd(8)
            assert torch.equal(y8, fwd(8)) and torch.equal(dx8, bwd(8)), mode
            for n in (1, 3):
                assert torch.equal(y8[:n], fwd(n)) and torch.equal(dx8[:n], bwd(n)), (mode, n)

            # dilation 1 through the _dilated entry points == the plain entry points (pad 1)
            split = mode == "bf16x3"
            y_plain = tc.conv2d_forward(x, wo, bias, res, 3, 3, 1, 1, relu=True)
            y_d1 = torch.empty_like(y_plain)
            _lib.call("mdb_conv2d_forward_dilated_bf16x3" if split else "mdb_conv2d_forward_dilated_f32", x,
                      wo.wf if split else wo, bias, res, y_d1, B, H, W, C, C, 3, 3, 1, 1, 1, 1)
            assert torch.equal(y_plain, y_d1), mode
            dx_plain = tc.conv2d_dgrad(x, wo, x.shape, res, mask, 3, 3, 1, 1)
            dx_d1 = torch.empty_like(dx_plain)
            _lib.call("mdb_conv2d_dgrad_dilated_bf16x3" if split else "mdb_conv2d_dgrad_dilated_f32", x, wo.wd if split else wo,
                      res, mask, dx_d1, B, H, W, C, C, 3, 3, 1, 1, 1, 0)
            assert torch.equal(dx_plain, dx_d1), mode
            prev = monodetr_b200.set_deterministic(True)
            try:
                dw_plain = tc.conv2d_wgrad(res, x, None, 3, 3, 1, 1)
                dw_d1 = torch.empty_like(dw_plain)
                _lib.call("mdb_conv2d_wgrad_bias_dilated_f32", res, x, None, dw_d1, None, B, H, W, C, C, 3, 3, 1, 1, 1, 0)
                assert torch.equal(dw_plain, dw_d1), mode
                assert torch.equal(tc.conv2d_wgrad(res, x, None, 3, 3, 1, D, dilation=D),
                                   tc.conv2d_wgrad(res, x, None, 3, 3, 1, D, dilation=D)), mode
            finally:
                monodetr_b200.set_deterministic(prev)
            assert _lib.lib().mdb_conv2d_forward_workspace_bytes_dilated(B, H, W, C, C, 3, 3, 1, 1, 1, 0, 0, int(split)) == \
                _lib.lib().mdb_conv2d_forward_workspace_bytes(B, H, W, C, C, 3, 3, 1, 1, 0, 0, int(split))
        finally:
            tc.set_precision(prev_mode)


def test_unsupported_dilated_geometries_raise():
    from monodetr_b200 import _lib, tc
    g = _gen(4)
    x = torch.randn(1, 24, 80, 64, device="cuda", generator=g)
    w3 = _pack(torch.randn(64, 64, 3, 3, device="cuda", generator=g))
    w1 = _pack(torch.randn(64, 64, 1, 1, device="cuda", generator=g))
    with pytest.raises(RuntimeError, match="conv2d_forward"):
        tc.conv2d_forward(x, w3, None, None, 3, 3, 2, D, dilation=D)               # stride 2 with dilation 2
    with pytest.raises(RuntimeError, match="mdb_conv2d_dgrad_dilated"):
        tc.conv2d_dgrad(torch.randn(1, 12, 40, 64, device="cuda", generator=g), w3, x.shape, None, None, 3, 3, 2, D, dilation=D)
    with pytest.raises(RuntimeError, match="mdb_conv2d_wgrad_bias_dilated"):
        tc.conv2d_wgrad(torch.randn(1, 12, 40, 64, device="cuda", generator=g), x, None, 3, 3, 2, D, dilation=D)
    with pytest.raises(RuntimeError, match="conv2d_forward"):
        tc.conv2d_forward(x, w1, None, None, 1, 1, 1, 0, dilation=D)                # 1x1 with dilation 2
    with pytest.raises(RuntimeError, match="mdb_conv2d_wgrad_bias_dilated"):      # weight gradient: pad % dilation != 0
        tc.conv2d_wgrad(torch.randn(1, 22, 78, 64, device="cuda", generator=g), x, None, 3, 3, 1, 1, dilation=D)
    for dil in (0, -1):
        assert _lib.lib().mdb_conv2d_forward_workspace_bytes_dilated(1, 24, 80, 64, 64, 3, 3, 1, 1, dil, 0, 0, 0) < 0
    assert _lib.lib().mdb_conv2d_forward_workspace_bytes_dilated(1, 24, 80, 64, 64, 3, 3, 2, 2, 2, 0, 0, 0) < 0


# ---- whole models ------------------------------------------------------------------------------------------------------------
def _model(backbone, dilation, dropout=0.0):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, backbone=backbone, dilation=dilation, dropout=dropout))
    m.load_state_dict(om.with_aliases(ob.deterministic_state_dict(variant_cfg(backbone, dilation))))
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
    return np.load(os.path.join(golden_dir, "backbones.npz"))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
@pytest.mark.parametrize("tag", list(VARIANTS))
def test_model_matches_the_reference(tag, precision, golden):
    """Eval outputs at 192 x 640 and train-mode outputs (dropout off) at 96 x 320, every output incl. aux within 1e-3
    (max|a - b| / max|b| over the stored elements)."""
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


def test_resnet152_matches_the_oracle():
    cfg = variant_cfg("resnet152", False)
    m = _model("resnet152", False).eval()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        ref = ob.forward(ob.deterministic_state_dict(cfg), images, calibs, sizes, training=False, cfg=cfg)
    for (k, a), (_, b) in zip(_flat(out), _flat(ref)):
        rel = float((a.float().cpu() - b).abs().max() / b.abs().max().clamp_min(1e-12))
        assert rel < 1e-3, (k, rel)


@pytest.mark.parametrize("backbone,dilation", [("resnet50", True), ("resnet101", False)])
def test_gradients_per_stage(backbone, dilation):
    """Frozen sampling locations, 192 x 640, B = 1: the bars of tests/test_model_grad_gpu.py."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    from test_model_grad_gpu import _grad_report
    cfg = variant_cfg(backbone, dilation)
    m = _model(backbone, dilation).train()
    images, calibs, sizes = om.synthetic_inputs(1, 11, H=192, W=640)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in ob.deterministic_state_dict(cfg).items()}
        om.surrogate_loss(ob.forward(sd, images, calibs, sizes, training=True, cfg=cfg)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    # The key-projection biases of the decoder's self-attention have an analytically zero gradient (a softmax does not see a
    # constant added to every key's score): both sides give cancellation noise there -- on the device that of the attention
    # backward's single-pass TF32 contractions (tests/tc_error_model.C_ATT_BWD) --, held against the weight's gradient.
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
        # query_embed: each row is the gradient of ONE of the 550 queries, not a sum over pixels or queries, so its max-norm is
        # a single query's worst case of the ReLU / max-pool selection noise, which grows with the backbone's depth (resnet101:
        # 3.6e-2 max-norm at 8.1e-3 L2 on an H100); the L2 bar stays.
        assert r < (5e-2 if stage == "query_embed" else 2e-2) and l2 < 2e-2, (stage, name, r, l2)


def test_dc5_training_iteration_is_bit_reproducible():
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
    tc.set_precision("bf16x3")
    try:
        runs = []
        for _ in range(2):
            torch.manual_seed(0)
            model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, backbone="resnet50", dilation=True, dropout=0.1))
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
            bad = [i for i, (a, b) in enumerate(zip(xs, ys)) if not torch.equal(a, b)]
            assert not bad, (name, len(bad), len(xs))
    finally:
        monodetr_b200.set_deterministic(prev)
