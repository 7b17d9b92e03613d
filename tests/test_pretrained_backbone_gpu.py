"""GPU: backbones loaded through `pretrained_backbone` with ImageNet-scale FrozenBN statistics (tests/imagenet_checkpoints.py:
running_var over eight decades, negative and zero BN weights, shifts up to ~1e3), where the folded BN scale reaches ~1e3.

- Every kernel call of the backbone, in both compensated precision modes, for all 8 bodies with and without the dilated C5
  stage at 2 x 3 x 96 x 320: the stem against float64 at tests/heads_error_model.C_STEM, the max-pool exactly, every
  convolution of every block (so every stage output), and in the backward every data gradient and every weight gradient of
  layer2-4, each against the float64 sum of its split operands at the bound of tests/tc_error_model.py.  Each call is held
  to the target of its own device inputs, so the bound is per kernel, not per network.
- The default resnet50 forward the same way at 384 x 1280.
- Weights loaded into a model that has already run a forward give the bits of a model built pretrained.
- A Trainer epoch (CUDA graph path) on the synthetic KITTI tree from a pretrained file: finite losses and parameters.
"""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import heads_error_model as hem
import imagenet_checkpoints as ic
import tc_error_model as em
from monodetr_b200 import backbone as bb

pytestmark = pytest.mark.gpu
F64 = torch.float64
MODES = ["bf16x3", "tf32x3"]     # ('tf32' rounds the block outputs to TF32 for their consumer: not the targets below)


@pytest.fixture(scope="module")
def hub(tmp_path_factory):
    """ensure(name): the hub directory holds `name`'s ImageNet-statistics file (one at a time: the deep ones are large)."""
    prev = torch.hub.get_dir()
    d = str(tmp_path_factory.mktemp("hub"))
    torch.hub.set_dir(d)
    current = []

    def ensure(name):
        if current != [name]:
            for old in current:
                os.remove(bb.imagenet_checkpoint_path(old))
            ic.write(ic.synthetic_checkpoint(name, seed=len(name), statistics="imagenet"), bb.imagenet_checkpoint_path(name))
            current[:] = [name]
    try:
        yield ensure
    finally:
        torch.hub.set_dir(prev)


@pytest.fixture
def mode(request):
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(request.param)
    yield request.param
    tc.set_precision(prev)


class _Record:
    """Every backbone call of the GEMM family, the stem and the max-pool, with arguments and result."""

    def __init__(self, monkeypatch):
        from monodetr_b200 import _lib, tc
        self.fwd, self.dgrad, self.wgrad, self.stem, self.pool = [], [], [], [], []
        fwd0, dgrad0, wgrad0, call0 = tc.conv2d_forward, tc.conv2d_dgrad, tc.conv2d_wgrad, _lib.call

        def fwd(x, w, bias=None, residual=None, kh=1, kw=1, stride=1, pad=0, relu=False, round_out=False, dilation=1, groups=1):
            y = fwd0(x, w, bias, residual, kh, kw, stride, pad, relu, round_out, dilation, groups)
            self.fwd.append((x, w, bias, residual, stride, pad, relu, dilation, groups, y))
            return y

        def dgrad(dy, w, x_shape, residual=None, relu_mask=None, kh=1, kw=1, stride=1, pad=0, round_out=False, dilation=1,
                  groups=1):
            dx = dgrad0(dy, w, x_shape, residual, relu_mask, kh, kw, stride, pad, round_out, dilation, groups)
            self.dgrad.append((dy, w, residual, relu_mask, stride, pad, dilation, groups, dx))
            return dx

        def wgrad(dy, x, rowscale=None, kh=1, kw=1, stride=1, pad=0, with_bias_grad=False, dilation=1, groups=1):
            self.wgrad.append((dy, x, rowscale, stride, pad, dilation, groups))
            return wgrad0(dy, x, rowscale, kh, kw, stride, pad, with_bias_grad, dilation, groups)

        def call(name, *args, **kw):
            r = call0(name, *args, **kw)
            if name == "mdb_stem_conv7x7_bn_relu_f32":
                self.stem.append(args[:5])
            elif name == "mdb_maxpool3x3s2_nhwc_f32":
                self.pool.append(args[:2])
            return r
        monkeypatch.setattr(tc, "conv2d_forward", fwd)
        monkeypatch.setattr(tc, "conv2d_dgrad", dgrad)
        monkeypatch.setattr(tc, "conv2d_wgrad", wgrad)
        monkeypatch.setattr(_lib, "call", call)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _epilogue32(shape, bias, res, relu):
    """The fp32 epilogue of an exact zero accumulator, as the kernel computes it."""
    z = torch.zeros(shape, device="cuda") + bias
    if res is not None:
        z = z + res
    return torch.relu(z) if relu else z


def _check_stem(rec):
    (images, w, scale, shift, y), = rec.stem
    ref, mag = hem.stem(images, w, scale, shift)
    err = (y.to(F64) - ref).abs()
    pos = mag > 0
    ratio = float((err[pos] / mag[pos]).max())
    print(f"stem: worst |y-ref|/mag = {ratio:.2f} (bound {hem.C_STEM})")
    assert bool(torch.isfinite(y).all()) and ratio <= hem.C_STEM and bool((err[~pos] == 0).all())
    (y2, pooled), = rec.pool
    assert y2 is y and torch.equal(_nchw(pooled), F.max_pool2d(_nchw(y), 3, 2, 1))


def _check_forward(rec, convs, sc, sh, mode):
    """Every convolution against float64; returns conv index -> (folded weight, output)."""
    of_shift = {t.data_ptr(): j for j, t in enumerate(sh)}
    seen = {}
    for x, w, bias, res, stride, pad, relu, dil, groups, y in rec.fwd:
        j = of_shift[bias.data_ptr()]
        wf = convs[j].weight.detach() * sc[j].view(-1, 1, 1, 1)

        def f(a, b):
            return _nhwc(F.conv2d(_nchw(a), b, stride=stride, padding=pad, dilation=dil, groups=groups))
        t, s = em.target(f, x, wf, mode)
        pre = t + bias.double() + (res.double() if res is not None else 0)
        em.assert_gemm(f"conv {j} {tuple(wf.shape)} s{stride} d{dil} g{groups}", y, torch.relu(pre) if relu else pre, s, mode,
                       epi=em.epi_mag(t, bias, res), exact_zero=_epilogue32(y.shape, bias, res, relu))
        seen[id(w)] = (j, wf)
    assert len(seen) == len(convs) - 1
    return seen


def _run_backbone(name, dilation, H, W, backward, seed):
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(seed)
    joiner = bb.build_backbone(dict(DEFAULT_MODEL_CFG, backbone=name, dilation=dilation, pretrained_backbone=True))
    net = joiner[0].cuda()
    sd = torch.load(bb.imagenet_checkpoint_path(name), weights_only=True)
    for k, v in net.body.state_dict().items():
        assert torch.equal(v.cpu(), sd[k]), k
    g = torch.Generator(device="cuda").manual_seed(seed)
    images = torch.randn(2 if backward else 1, 3, H, W, device="cuda", generator=g)
    feats = net(images)
    if backward:
        torch.autograd.backward(feats, [torch.randn(f.shape, device="cuda", generator=g) for f in feats])
    torch.cuda.synchronize()
    return net, feats


def _check(rec, net, feats, mode, backward):
    convs = net._convs()
    sc, sh = net._bn_tensors()
    _check_stem(rec)
    seen = _check_forward(rec, convs, sc, sh, mode)
    outs = {r[-1].data_ptr() for r in rec.fwd}
    assert len(feats) == 3 and all(f.data_ptr() in outs for f in feats)          # the stage outputs are checked outputs
    for f in feats:
        print(f"stage output {tuple(f.shape)}: max |y| {float(f.abs().max()):.3e}")
    if not backward:
        return
    for dy, w, res, mask, stride, pad, dil, groups, dx in rec.dgrad:
        j, wf = seen[id(w)]

        def f(a, b):
            return _nhwc(torch.nn.grad.conv2d_input(_nchw(dx).shape, b, _nchw(a), stride=stride, padding=pad, dilation=dil,
                                                    groups=groups))
        t, s = em.target(f, dy, wf, mode)
        gate = (mask > 0).double() if mask is not None else torch.ones((), dtype=F64, device="cuda")
        ref = (t + (res.double() if res is not None else 0)) * gate
        exact = (res if res is not None else torch.zeros((), device="cuda")) * (mask > 0 if mask is not None else 1)
        em.assert_gemm(f"dgrad conv {j} s{stride} d{dil} g{groups}", dx, ref, s * gate, mode,
                       epi=em.epi_mag(t, None, res) * gate, exact_zero=exact)
    of_scale = {t.data_ptr(): j for j, t in enumerate(sc)}
    checked = set()
    for dy, x, rowscale, stride, pad, dil, groups in rec.wgrad:
        j = of_scale[rowscale.data_ptr()]
        wgt = convs[j].weight

        def f(a, b):
            return torch.nn.grad.conv2d_weight(_nchw(b), wgt.shape, _nchw(a), stride=stride, padding=pad, dilation=dil,
                                               groups=groups)
        t, s = em.target(f, dy, x, mode)
        scv = rowscale.double().view(-1, 1, 1, 1)
        em.assert_gemm(f"wgrad conv {j} s{stride} d{dil} g{groups}", wgt.grad, t * scv, s * scv.abs(), mode,
                       epi=t.abs() * scv.abs())
        checked.add(j)
    trainable = {j for j, c in enumerate(convs) if c.weight.requires_grad}
    # every trainable conv gets a data gradient except conv1 and the downsample of layer2's first block (its input is frozen)
    assert checked == trainable and len(rec.dgrad) == len(trainable) - 2


@pytest.mark.parametrize("mode", MODES, indirect=True)
@pytest.mark.parametrize("dilation", [False, True])
@pytest.mark.parametrize("name", ic.NAMES)
def test_every_backbone_kernel_within_its_bound(name, dilation, mode, hub, monkeypatch):
    hub(name)
    rec = _Record(monkeypatch)
    net, feats = _run_backbone(name, dilation, 96, 320, True, seed=len(name) + dilation)
    monkeypatch.undo()
    with torch.no_grad():
        _check(rec, net, feats, mode, True)


def test_resnet50_forward_full_size(hub, monkeypatch):
    hub("resnet50")
    rec = _Record(monkeypatch)
    net, feats = _run_backbone("resnet50", False, 384, 1280, False, seed=5)
    monkeypatch.undo()
    from monodetr_b200 import tc
    with torch.no_grad():
        _check(rec, net, feats, tc.get_precision(), False)


def _model(pretrained, seed=0):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(seed)
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, pretrained_backbone=pretrained))
    return m.cuda().eval()


@pytest.mark.parametrize("mode", MODES, indirect=True)
def test_loading_after_a_forward_matches_a_pretrained_build(mode, hub):
    """The folded BN tensors and weight splits of a model that already ran are rebuilt from the loaded values."""
    import monodetr_b200
    from oracle import monodetr_torch as om
    hub("resnet50")
    images, calibs, sizes = (t.cuda() for t in om.synthetic_inputs(1, 3, H=96, W=320))
    prev = monodetr_b200.set_deterministic(True)
    try:
        with torch.no_grad():
            late = _model(False)
            before = late(images, calibs, None, sizes)["pred_logits"].clone()
            bb.load_imagenet_weights(late.backbone[0].body, "resnet50")
            got = late(images, calibs, None, sizes)
            want = _model(True)(images, calibs, None, sizes)
    finally:
        monodetr_b200.set_deterministic(prev)
    assert not torch.equal(before, got["pred_logits"])
    for k in ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits"):
        assert torch.equal(got[k], want[k]), k


def test_trainer_epoch_from_a_pretrained_file(hub, tmp_path, monkeypatch):
    import synthetic_kitti as sk
    import trainer_stubs as S
    from bench_extras import CRIT_CFG
    from monodetr_b200 import build_monodetr, dataset as ds, kernels as K, tc, trainer as T
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    hub("resnet50")
    logs = []
    monkeypatch.setattr(T, "print_losses", lambda i, log: logs.append(dict(log)))
    root = str(tmp_path / "kitti")
    sk.write_tree(root)
    cfg = dict(json.loads(str(np.load(os.path.join(os.path.dirname(__file__), "golden", "loader.npz"))["cfg"])), root_dir=root)
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, pretrained_backbone=True))
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler({"warmup": False, "decay_rate": 0.5, "decay_list": [1]}, opt, last_epoch=-1)
    sk.set_random_seed(444)
    train_loader, val_loader = ds.build_dataloader(cfg, workers=0)
    tr = T.Trainer({"max_epoch": 1, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": str(tmp_path / "out")},
                   model, opt, train_loader, val_loader, sched, warm, S.ListLogger(), crit, "m")
    assert tr.graph_path
    tr.PRINT_EVERY = 1
    K.reseed(torch.device("cuda", torch.cuda.current_device()), 4242)
    tr.train_one_epoch(0)
    assert tr.live_graphs >= 1
    assert len(logs) == len(train_loader)
    print({k: f"{v:.4g}" for k, v in logs[-1].items()})
    assert all(log and all(np.isfinite(v) for v in log.values()) for log in logs)
    assert all(bool(torch.isfinite(p).all()) for p in model.parameters())
