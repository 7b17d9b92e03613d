"""CPU: the reference's other backbones (cfg `backbone` in resnet50 / resnet101 / resnet152, `dilation` True = the dilated C5
stage) -- the product model's state_dict contract against the unmodified reference (tests/golden/backbones.npz, written by
tools/gen_golden_backbones.py), the oracle against the reference's outputs and gradients, and the whole product model's host
logic through the stand-in device library (tests/fake_device_lib.py, extended here by the dilated convolution entry points)
against the oracle."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import f32
import oracle_backbones as ob     # tests/oracle_backbones.py
from oracle_backbones import variant_cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import VARIANTS, grad_index  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "backbones.npz"))


def _model_cfg(backbone, dilation, **kw):
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    return dict(DEFAULT_MODEL_CFG, backbone=backbone, dilation=dilation, **kw)


def _build(backbone, dilation):
    from monodetr_b200 import build_monodetr
    torch.manual_seed(0)
    return build_monodetr(_model_cfg(backbone, dilation))[0]


# ---- state_dict contract ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", list(VARIANTS))
def test_state_dict_matches_the_reference(tag, golden):
    backbone, dilation = VARIANTS[tag]
    m = _build(backbone, dilation)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    assert {k: tuple(s) for k, s, _ in spec} == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n for n, p in m.named_parameters() if p.requires_grad}
    assert len(spec) == {"resnet50": 582, "resnet101": 837}[backbone]
    # the oracle's statement of the same variant
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in ob.state_dict_spec(variant_cfg(backbone, dilation)).items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == {k: tuple(s) for k, s, _ in spec}


@pytest.mark.parametrize("backbone,dilation", [("resnet50", True), ("resnet101", False), ("resnet101", True),
                                               ("resnet152", False), ("resnet152", True)])
def test_reference_shaped_checkpoint_loads_strictly(backbone, dilation):
    m = _build(backbone, dilation)
    sd = om.with_aliases(ob.deterministic_state_dict(variant_cfg(backbone, dilation)))
    sd["backbone.0.body.bn1.num_batches_tracked"] = torch.tensor(0)           # dropped like the reference (backbone.py:41-50)
    m.load_state_dict(sd, strict=True)
    assert m.backbone.strides == ([8, 16, 16] if dilation else [8, 16, 32])
    assert m.backbone.num_channels == [512, 1024, 2048]


def test_resnet152_state_dict():
    """ResNet-152: the oracle's spec (torchvision's layer names, 3-8-36-3 blocks) and the reference's trainability rule."""
    m = _build("resnet152", False)
    sd = m.state_dict()
    spec = om.with_aliases({k: torch.empty(s) for k, s in ob.state_dict_spec(variant_cfg("resnet152", False)).items()})
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in spec.items()}
    assert len(sd) == 1092
    assert sum(p.numel() for p in m.parameters()) == 72_212_692
    for name, p in m.named_parameters():
        if name.startswith("backbone.0.body."):
            assert p.requires_grad == any(s in name for s in ("layer2", "layer3", "layer4")), name
    assert len(m.backbone[0].body.layer2) == 8 and len(m.backbone[0].body.layer3) == 36


def test_dc5_block_geometry():
    """torchvision's replace_stride_with_dilation=[False, False, True]: layer4 block 0 is stride 1 / dilation 1 (its 1x1
    downsample stride 1 too), blocks 1.. are 3x3 with dilation 2 and padding 2."""
    body = _build("resnet50", True).backbone[0].body
    b0 = body.layer4[0]
    assert (b0.stride, b0.dilation, b0.conv2.stride, b0.conv2.dilation, b0.conv2.padding) == (1, 1, (1, 1), (1, 1), (1, 1))
    assert b0.downsample[0].stride == (1, 1)
    for blk in body.layer4[1:]:
        assert (blk.stride, blk.dilation, blk.conv2.dilation, blk.conv2.padding) == (1, 2, (2, 2), (2, 2))
    assert all(blk.dilation == 1 for name, blk in body.blocks() if name != "layer4")


@pytest.mark.parametrize("name", ["resnet18", "resnet34", "resnext50_32x4d", "wide_resnet50_2", "resnet200"])
def test_unsupported_backbones_raise(name):
    from monodetr_b200.backbone import Backbone
    for dilation in (False, True):
        with pytest.raises(NotImplementedError, match="resnet50, resnet101, resnet152"):
            Backbone(name, True, True, dilation)


# ---- oracle against the reference ------------------------------------------------------------------------------------------
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
    """Eval outputs at 192 x 640 and train outputs + every parameter gradient at 96 x 320, as tests/test_oracle_model.py
    checks resnet50 (same bars)."""
    cfg = variant_cfg(*VARIANTS[tag])
    sd = ob.deterministic_state_dict(cfg)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        _check_outputs(golden, f"{tag}.fwd_eval", ob.forward(sd, images, calibs, sizes, training=False, cfg=cfg), 2e-4, 2e-5)

    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    sdg = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    out = ob.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
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
        # (tests/test_oracle_model.py); everything else agrees to ~1e-4
        rel = float(np.abs(gm[grad_index(gm.numel(), name)].numpy() - golden[f"{tag}.grad_val"][offs[j]:offs[j + 1]]).max()) / scale
        assert rel <= 5e-2, (name, rel)
        assert abs(float(gm.abs().max()) - scale) <= 5e-2 * scale, name
        rels.append(rel)
    assert len(rels) > 250
    assert sorted(rels)[len(rels) // 2] < 1e-3


# ---- the product model's host logic, through the stand-in library ----------------------------------------------------------
class DilatedFakeLib(fake_device_lib.FakeLib):
    """FakeLib plus the dilated convolution entry points (include/monodetr_b200.h, "*_dilated"), each restated with torch's
    dilated convolution; every convolution call is logged as (entry point, kh, stride, pad, dilation)."""

    def __init__(self, precision):
        super().__init__(precision)
        self.conv_log = []

    @staticmethod
    def _size(n, k, stride, pad, d):
        return (n + 2 * pad - d * (k - 1) - 1) // stride + 1

    # the undilated entry points, logged
    def mdb_conv2d_forward_f32(self, x, w, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, stream):
        self.conv_log.append(("forward", kh, stride, pad, 1))
        return self._fwd(x, w, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, flags)

    def mdb_conv2d_dgrad_f32(self, dy, w, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, flags, stream):
        self.conv_log.append(("dgrad", kh, stride, pad, 1))
        return self._dgrad(dy, w, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, 1)

    def mdb_conv2d_wgrad_bias_f32(self, dy, x, rowscale, dw, db, B, H, W, Cin, Cout, kh, kw, stride, pad, accumulate, stream):
        self.conv_log.append(("wgrad", kh, stride, pad, 1))
        return self._wgrad(dy, x, rowscale, dw, db, B, H, W, Cin, Cout, kh, kw, stride, pad, 1, accumulate)

    # the dilated twins
    def mdb_conv2d_forward_workspace_bytes_dilated(self, *a):
        return 0

    def mdb_conv2d_forward_dilated_f32(self, x, w, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, flags, stream):
        self.conv_log.append(("forward_dilated", kh, stride, pad, dil))
        return self._fwd(x, w, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, flags)

    def mdb_conv2d_dgrad_dilated_f32(self, dy, w, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, flags,
                                     stream):
        self.conv_log.append(("dgrad_dilated", kh, stride, pad, dil))
        return self._dgrad(dy, w, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil)

    def mdb_conv2d_wgrad_bias_dilated_f32(self, dy, x, rowscale, dw, db, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, accumulate,
                                          stream):
        self.conv_log.append(("wgrad_dilated", kh, stride, pad, dil))
        return self._wgrad(dy, x, rowscale, dw, db, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, accumulate)

    def mdb_conv2d_forward_dilated_bf16x3(self, x, w_split, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, flags,
                                          stream):
        self.conv_log.append(("forward_dilated", kh, stride, pad, dil))
        w = self._decode_split(w_split, kh * kw, Cout, Cin).contiguous()
        return self._fwd(x, w.data_ptr(), bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, flags)

    def mdb_conv2d_dgrad_dilated_bf16x3(self, dy, w_split_t, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil,
                                        flags, stream):
        self.conv_log.append(("dgrad_dilated", kh, stride, pad, dil))
        w = self._decode_split(w_split_t, kh * kw, Cin, Cout).transpose(1, 2).contiguous()
        return self._dgrad(dy, w.data_ptr(), residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil)

    # (FakeLib's bf16x3 forward / dgrad decode the split weights and call the _f32 methods above, which log them)
    def _fwd(self, x, w, bias, residual, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, flags):
        Ho, Wo = self._size(H, kh, stride, pad, dil), self._size(W, kw, stride, pad, dil)
        out = F.conv2d(f32(x, B, H, W, Cin).permute(0, 3, 1, 2), self._w_oihw(w, Cout, Cin, kh, kw), f32(bias, Cout), stride=stride,
                       padding=pad, dilation=dil).permute(0, 2, 3, 1)
        if residual:
            out = out + f32(residual, B, Ho, Wo, Cout)
        if flags & 1:
            out = torch.relu(out)
        f32(y, B, Ho, Wo, Cout).copy_(out)
        return 0

    def _dgrad(self, dy, w, residual, relu_mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil):
        Ho, Wo = self._size(H, kh, stride, pad, dil), self._size(W, kw, stride, pad, dil)
        g = torch.nn.grad.conv2d_input((B, Cin, H, W), self._w_oihw(w, Cout, Cin, kh, kw).contiguous(),
                                       f32(dy, B, Ho, Wo, Cout).permute(0, 3, 1, 2), stride=stride, padding=pad,
                                       dilation=dil).permute(0, 2, 3, 1)
        if residual:
            g = g + f32(residual, B, H, W, Cin)
        if relu_mask:
            g = g * (f32(relu_mask, B, H, W, Cin) > 0)
        f32(dx, B, H, W, Cin).copy_(g)
        return 0

    def _wgrad(self, dy, x, rowscale, dw, db, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, accumulate):
        Ho, Wo = self._size(H, kh, stride, pad, dil), self._size(W, kw, stride, pad, dil)
        dyt = f32(dy, B, Ho, Wo, Cout)
        g = torch.nn.grad.conv2d_weight(f32(x, B, H, W, Cin).permute(0, 3, 1, 2), (Cout, Cin, kh, kw), dyt.permute(0, 3, 1, 2),
                                        stride=stride, padding=pad, dilation=dil)
        if rowscale:
            g = g * f32(rowscale, Cout).view(-1, 1, 1, 1)
        g = g.permute(2, 3, 0, 1).reshape(kh * kw, Cout, Cin)
        out = f32(dw, kh * kw, Cout, Cin)
        out.copy_(out + g if accumulate else g)
        if db:
            s = dyt.sum((0, 1, 2))
            o = f32(db, Cout)
            o.copy_(o + s if accumulate else s)
        return 0


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
@pytest.mark.parametrize("backbone,dilation", [("resnet50", True), ("resnet101", False)])
def test_whole_model_matches_the_oracle(monkeypatch, backbone, dilation, precision):
    """Train mode at 96 x 320: every output within 1e-4 and every parameter gradient at the bars of
    tests/test_model_host_logic.py; the dilation-2 convolutions go through the _dilated entry points, all others through the
    plain ones with the arguments they always had."""
    from monodetr_b200 import _lib
    from monodetr_b200.bench_model import surrogate_loss
    fake_device_lib.install(monkeypatch, {"tf32x3": 1, "bf16x3": 2}[precision])
    fake = DilatedFakeLib({"tf32x3": 1, "bf16x3": 2}[precision])
    monkeypatch.setattr(_lib, "_lib", fake)
    from monodetr_b200 import build_monodetr, tc
    assert tc.get_precision() == precision
    cfg = variant_cfg(backbone, dilation)
    m, _ = build_monodetr(_model_cfg(backbone, dilation, dropout=0.0, device="cpu"))
    sd = ob.deterministic_state_dict(cfg)
    m.load_state_dict(om.with_aliases(sd))
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    m.train()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    out = m(images, calibs, None, sizes)
    surrogate_loss(out).backward()

    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = ob.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
    om.surrogate_loss(ref).backward()
    for k in OUT_KEYS:
        assert out[k].shape == ref[k].shape, k
        assert _rel(out[k].detach(), ref[k].detach()) < 1e-4, (k, _rel(out[k].detach(), ref[k].detach()))
    for a, b in zip(out["aux_outputs"], ref["aux_outputs"]):
        for k in a:
            assert _rel(a[k].detach(), b[k].detach()) < 1e-4, ("aux", k)

    by_name = om.with_aliases(sdg)
    errs = []
    for name, p in m.named_parameters():
        want = by_name[name].grad
        if not p.requires_grad:
            assert p.grad is None, name
            continue
        if p.grad is None:
            assert want is None or not want.any(), name
            continue
        assert want is not None, name
        errs.append((_rel(p.grad, want), name, float(want.abs().max())))
    errs.sort()
    assert len(errs) == (313 if backbone == "resnet50" else 364)
    med_bar, worst_bar = (1e-3, 1e-1) if precision == "bf16x3" else (3e-4, 3e-2)
    assert errs[len(errs) // 2][0] < med_bar, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < worst_bar or scale < 1e-6, (name, err, scale)

    # layer4's blocks 1 and 2 under DC5: one dilated forward, dgrad and wgrad each; nothing else is dilated
    dilated = [c for c in fake.conv_log if c[0].endswith("_dilated")]
    n_d2 = 2 if dilation else 0
    assert sorted(dilated) == sorted([(kind + "_dilated", 3, 1, 2, 2) for kind in ("forward", "dgrad", "wgrad")] * n_d2)
    assert all(pad == kh // 2 for kind, kh, _, pad, _ in fake.conv_log if not kind.endswith("_dilated"))
    assert any(kind == "forward" and kh == 3 for kind, kh, _, _, _ in fake.conv_log)
