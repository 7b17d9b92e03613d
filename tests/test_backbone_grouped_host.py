"""CPU: the reference's ResNeXt and wide-ResNet backbones (cfg `backbone` in resnext50_32x4d / resnext101_32x8d /
resnext101_64x4d / wide_resnet50_2 / wide_resnet101_2, each with `dilation` False and True) -- the product model's
state_dict contract against the unmodified reference (tests/golden/backbones_grouped.npz, written by
tools/gen_golden_backbones_grouped.py), the oracle against the reference's outputs and gradients, the grouped entry points'
geometry checks, and the whole product model's host logic through the stand-in device library (tests/fake_device_lib.py,
extended here by the grouped convolution entry points) against the oracle."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import monodetr_torch as om
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import _ptrs, bf16, f32
import oracle_backbones_grouped as obg     # tests/oracle_backbones_grouped.py

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from gen_golden_backbones import grad_index  # noqa: E402
from gen_golden_backbones_grouped import SPEC_VARIANTS, VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "backbones_grouped.npz"))


def _model_cfg(backbone, dilation, **kw):
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    return dict(DEFAULT_MODEL_CFG, backbone=backbone, dilation=dilation, **kw)


def _build(backbone, dilation):
    from monodetr_b200 import build_monodetr
    torch.manual_seed(0)
    return build_monodetr(_model_cfg(backbone, dilation))[0]


# ---- state_dict contract ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", list(SPEC_VARIANTS))
def test_state_dict_matches_the_reference(tag, golden):
    backbone, dilation = SPEC_VARIANTS[tag]
    m = _build(backbone, dilation)
    spec = json.loads(golden[f"{tag}.spec"].tobytes())
    assert [k for k, _, _ in spec] == list(m.state_dict().keys())
    assert {k: tuple(s) for k, s, _ in spec} == {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert {k for k, _, t in spec if t} == {n for n, p in m.named_parameters() if p.requires_grad}
    oracle_spec = om.with_aliases({k: torch.empty(s) for k, s in obg.state_dict_spec(obg.variant_cfg(backbone, dilation)).items()})
    assert {k: tuple(v.shape) for k, v in oracle_spec.items()} == {k: tuple(s) for k, s, _ in spec}
    assert m.backbone.strides == ([8, 16, 16] if dilation else [8, 16, 32])
    assert m.backbone.num_channels == [512, 1024, 2048]


@pytest.mark.parametrize("tag", list(SPEC_VARIANTS))
def test_reference_shaped_checkpoint_loads_strictly(tag):
    backbone, dilation = SPEC_VARIANTS[tag]
    m = _build(backbone, dilation)
    sd = om.with_aliases(obg.deterministic_state_dict(obg.variant_cfg(backbone, dilation)))
    sd["backbone.0.body.bn1.num_batches_tracked"] = torch.tensor(0)
    m.load_state_dict(sd, strict=True)


@pytest.mark.parametrize("name", ["resnet18", "resnet34", "resnet200", "resnext50_32x8d", "resnet50"])
def test_unsupported_backbones_raise(name):
    """The model section's names that build nothing raise, listing every name that builds; each backbone class refuses the
    other's names."""
    from monodetr_b200.backbone import ResNeXtBackbone
    msg = ("resnet50, resnet101, resnet152 and ResNeXtBackbone builds resnext50_32x4d, resnext101_32x8d, resnext101_64x4d, "
           "wide_resnet50_2, wide_resnet101_2")
    for dilation in (False, True):
        if name != "resnet50":
            with pytest.raises(NotImplementedError, match=msg):
                _build(name, dilation)
        with pytest.raises(NotImplementedError, match=msg):
            ResNeXtBackbone(name, True, True, dilation)


@pytest.mark.parametrize("name", ["resnext50_32x4d", "wide_resnet101_2"])
def test_build_backbone_picks_the_class_by_name(name):
    from monodetr_b200.backbone import Backbone, ResNeXtBackbone
    assert isinstance(_build(name, False).backbone[0], ResNeXtBackbone)
    assert isinstance(_build("resnet50", False).backbone[0], Backbone)


# ---- the C ABI's geometry checks (they return before touching a pointer) ---------------------------------------------------
# (B, H, W, Cin, Cout, kh, kw, stride, pad, dilation, groups)
_BAD = [
    (1, 8, 8, 96, 96, 3, 3, 1, 1, 1, 32),        # C % 128
    (1, 8, 8, 384, 384, 3, 3, 1, 1, 1, 2),       # 192 channels per group do not divide 128
    (1, 8, 8, 256, 256, 3, 3, 1, 1, 1, 3),       # C % groups
    (1, 8, 8, 256, 128, 3, 3, 1, 1, 1, 32),      # Cin != Cout
    (1, 8, 8, 256, 256, 1, 1, 1, 0, 1, 32),      # 1x1
    (1, 8, 8, 256, 256, 3, 3, 2, 2, 2, 32),      # dilation at stride 2
    (1, 8, 8, 256, 256, 3, 3, 3, 1, 1, 32),      # stride 3
]


@pytest.mark.parametrize("geom", _BAD)
@pytest.mark.parametrize("entry", ["mdb_conv2d_forward_grouped_f32", "mdb_conv2d_forward_grouped_bf16x3",
                                   "mdb_conv2d_dgrad_grouped_f32", "mdb_conv2d_dgrad_grouped_bf16x3",
                                   "mdb_conv2d_wgrad_grouped_f32"])
def test_unsupported_grouped_geometry_is_refused(entry, geom):
    from monodetr_b200 import _lib
    nptr = 4 if entry.startswith("mdb_conv2d_wgrad") else 5
    assert getattr(_lib.lib(), entry)(*([None] * nptr), *geom, 0, None) == -2


def test_grouped_weight_gradient_needs_pad_multiple_of_dilation():
    from monodetr_b200 import _lib
    assert _lib.lib().mdb_conv2d_wgrad_grouped_f32(None, None, None, None, 1, 8, 8, 256, 256, 3, 3, 1, 1, 2, 32, 0, None) == -2
    # the same geometry is a valid forward (it fails only on the NULL pointers)
    assert _lib.lib().mdb_conv2d_forward_grouped_f32(None, None, None, None, None, 1, 8, 8, 256, 256, 3, 3, 1, 1, 2, 32, 0,
                                                     None) == -1


def test_grouped_pack_refuses_bad_widths():
    from monodetr_b200 import _lib
    w = (ctypes.c_void_p * 1)(16)
    for C, g in ((96, 32), (384, 2), (256, 0)):
        rc = _lib.lib().mdb_pack_conv_weights_grouped_multi_f32(1, w, None, w, None, (ctypes.c_int * 1)(C), (ctypes.c_int * 1)(g),
                                                                None)
        assert rc == (-1 if g == 0 else -2)


# ---- oracle against the reference ------------------------------------------------------------------------------------------
def _check_outputs(golden, prefix, out, rtol, atol):
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_{k}", out[k].detach().numpy()), rtol=rtol, atol=atol,
                                   err_msg=prefix + " " + k)
    for i, a in enumerate(out["aux_outputs"]):
        for k in a:
            np.testing.assert_allclose(*sampled_forward(golden, f"{prefix}_aux{i}_{k}", a[k].detach().numpy()), rtol=rtol,
                                       atol=atol, err_msg=f"{prefix} aux{i} {k}")


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_oracle_matches_the_reference(tag, golden):
    """Eval outputs at 192 x 640, train outputs and sampled parameter gradients at 96 x 320 (the bars of
    tests/test_backbone_variants_host.py)."""
    cfg = obg.variant_cfg(*VARIANTS[tag])
    sd = obg.deterministic_state_dict(cfg)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        _check_outputs(golden, f"{tag}.fwd_eval", obg.forward(sd, images, calibs, sizes, training=False, cfg=cfg), 2e-4, 2e-5)
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    sdg = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd.items()}
    out = obg.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
    _check_outputs(golden, f"{tag}.fwd_train", out, 2e-4, 2e-5)
    om.surrogate_loss(out).backward()
    names = json.loads(golden[f"{tag}.grad_names"].tobytes())
    offs = np.concatenate([[0], np.cumsum(golden[f"{tag}.grad_len"])])
    rels = []
    for j, name in enumerate(names):
        if name not in sdg:
            continue
        gm = sdg[name].grad
        assert gm is not None, name
        scale = float(golden[f"{tag}.grad_max"][j])
        if scale < 1e-6:
            continue
        gm = gm.reshape(-1)
        rel = float(np.abs(gm[grad_index(gm.numel(), name)].numpy() - golden[f"{tag}.grad_val"][offs[j]:offs[j + 1]]).max()) / scale
        assert rel <= 5e-2, (name, rel)
        assert abs(float(gm.abs().max()) - scale) <= 5e-2 * scale, name
        rels.append(rel)
    assert len(rels) > 250
    assert sorted(rels)[len(rels) // 2] < 1e-3


# ---- the product model's host logic, through the stand-in library ----------------------------------------------------------
def _bands(C):
    return torch.arange(C).view(C, 1) // 128 * 128 + torch.arange(128).view(1, 128)


def _band_from_oihw(w, C, groups):
    """(C, C/g, 3, 3) -> (wf, wd) band-local (9, C, 128) as include/monodetr_b200.h states them."""
    gc = C // groups
    dense = torch.zeros(C, C, 9, dtype=w.dtype)
    for q in range(groups):
        dense[q * gc:(q + 1) * gc, q * gc:(q + 1) * gc] = w[q * gc:(q + 1) * gc].reshape(gc, gc, 9)
    b = _bands(C).expand(9, C, 128)
    return dense.permute(2, 0, 1).gather(2, b), dense.permute(2, 1, 0).gather(2, b)


def _oihw_from_band(band, C, groups, transposed):
    full = torch.zeros(9, C, C, dtype=band.dtype)
    full.scatter_(2, _bands(C).expand(9, C, 128), band)
    if transposed:
        full = full.transpose(1, 2)
    gc = C // groups
    return torch.stack([full[:, o, (o // gc) * gc:(o // gc + 1) * gc] for o in range(C)]).permute(0, 2, 1).reshape(C, gc, 3, 3)


class GroupedFakeLib(fake_device_lib.FakeLib):
    """FakeLib plus the dilated and the grouped convolution entry points, restated with torch; every grouped call is logged
    as (entry point, C, groups, stride, pad, dilation)."""

    def __init__(self, precision):
        super().__init__(precision)
        self.grouped_log = []

    def mdb_conv2d_forward_workspace_bytes_dilated(self, *a):
        return 0

    def _band(self, ptr, C, split):
        if split:
            t = bf16(ptr, 9, C, 4, 2, 32).float()
            return (t[:, :, :, 0] + t[:, :, :, 1]).reshape(9, C, 128)
        return f32(ptr, 9, C, 128)

    def _pack(self, n, w, scale, wf, wd, C, groups, split):
        ws, ss = _ptrs(w, n), (_ptrs(scale, n) if scale else [0] * n)
        fs, ds = _ptrs(wf, n), (_ptrs(wd, n) if wd else [0] * n)
        for j in range(n):
            c, g = int(C[j]), int(groups[j])
            src = f32(ws[j], c, c // g, 3, 3)
            if ss[j]:
                src = src * f32(ss[j], c).view(-1, 1, 1, 1)
            for dst, band in zip((fs[j], ds[j]), _band_from_oihw(src, c, g)):
                if not dst:
                    continue
                if split:
                    hi = band.to(torch.bfloat16)
                    lo = (band - hi.float()).to(torch.bfloat16)
                    out = bf16(dst, 9, c, 4, 2, 32)
                    out[:, :, :, 0].copy_(hi.view(9, c, 4, 32))
                    out[:, :, :, 1].copy_(lo.view(9, c, 4, 32))
                else:
                    f32(dst, 9, c, 128).copy_(band)
        return 0

    def mdb_pack_conv_weights_grouped_multi_f32(self, n, w, scale, wf, wd, C, groups, stream):
        return self._pack(n, w, scale, wf, wd, C, groups, False)

    def mdb_pack_conv_weights_grouped_multi_bf16x3(self, n, w, scale, wf, wd, C, groups, stream):
        return self._pack(n, w, scale, wf, wd, C, groups, True)

    def mdb_unpack_conv_wgrads_grouped_multi_f32(self, n, dw, out, C, groups, stream):
        ds, os_ = _ptrs(dw, n), _ptrs(out, n)
        for j in range(n):
            c, g = int(C[j]), int(groups[j])
            f32(os_[j], c, c // g, 3, 3).copy_(_oihw_from_band(f32(ds[j], 9, c, 128), c, g, False))
        return 0

    @staticmethod
    def _size(n, stride, pad, d):
        return (n + 2 * pad - 2 * d - 1) // stride + 1

    def _fwd(self, x, w, bias, residual, y, B, H, W, C, stride, pad, dil, groups, flags, split):
        self.grouped_log.append(("forward", C, groups, stride, pad, dil))
        wt = _oihw_from_band(self._band(w, C, split), C, groups, False)
        Ho, Wo = self._size(H, stride, pad, dil), self._size(W, stride, pad, dil)
        out = F.conv2d(f32(x, B, H, W, C).permute(0, 3, 1, 2), wt, f32(bias, C), stride=stride, padding=pad, dilation=dil,
                       groups=groups).permute(0, 2, 3, 1)
        if residual:
            out = out + f32(residual, B, Ho, Wo, C)
        if flags & 1:
            out = torch.relu(out)
        f32(y, B, Ho, Wo, C).copy_(out)
        return 0

    def mdb_conv2d_forward_grouped_f32(self, x, w, bias, res, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, groups, flags, st):
        return self._fwd(x, w, bias, res, y, B, H, W, Cin, stride, pad, dil, groups, flags, False)

    def mdb_conv2d_forward_grouped_bf16x3(self, x, w, bias, res, y, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, groups, flags,
                                          st):
        return self._fwd(x, w, bias, res, y, B, H, W, Cin, stride, pad, dil, groups, flags, True)

    def _dgrad(self, dy, w, residual, relu_mask, dx, B, H, W, C, stride, pad, dil, groups, split):
        self.grouped_log.append(("dgrad", C, groups, stride, pad, dil))
        wt = _oihw_from_band(self._band(w, C, split), C, groups, True)
        Ho, Wo = self._size(H, stride, pad, dil), self._size(W, stride, pad, dil)
        g = torch.nn.grad.conv2d_input((B, C, H, W), wt, f32(dy, B, Ho, Wo, C).permute(0, 3, 1, 2), stride=stride, padding=pad,
                                       dilation=dil, groups=groups).permute(0, 2, 3, 1)
        if residual:
            g = g + f32(residual, B, H, W, C)
        if relu_mask:
            g = g * (f32(relu_mask, B, H, W, C) > 0)
        f32(dx, B, H, W, C).copy_(g)
        return 0

    def mdb_conv2d_dgrad_grouped_f32(self, dy, w, res, mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, groups, flags, st):
        return self._dgrad(dy, w, res, mask, dx, B, H, W, Cin, stride, pad, dil, groups, False)

    def mdb_conv2d_dgrad_grouped_bf16x3(self, dy, w, res, mask, dx, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, groups, flags,
                                        st):
        return self._dgrad(dy, w, res, mask, dx, B, H, W, Cin, stride, pad, dil, groups, True)

    def mdb_conv2d_wgrad_grouped_f32(self, dy, x, rowscale, dw, B, H, W, Cin, Cout, kh, kw, stride, pad, dil, groups, accumulate,
                                     st):
        self.grouped_log.append(("wgrad", Cin, groups, stride, pad, dil))
        C = Cin
        Ho, Wo = self._size(H, stride, pad, dil), self._size(W, stride, pad, dil)
        g = torch.nn.grad.conv2d_weight(f32(x, B, H, W, C).permute(0, 3, 1, 2), (C, C // groups, 3, 3),
                                        f32(dy, B, Ho, Wo, C).permute(0, 3, 1, 2), stride=stride, padding=pad, dilation=dil,
                                        groups=groups)
        if rowscale:
            g = g * f32(rowscale, C).view(-1, 1, 1, 1)
        band = _band_from_oihw(g, C, groups)[0]
        out = f32(dw, 9, C, 128)
        out.copy_(out + band if accumulate else band)
        return 0


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
@pytest.mark.parametrize("dilation", [False, True])
def test_whole_model_matches_the_oracle(monkeypatch, dilation, precision):
    """resnext50_32x4d in train mode at 96 x 320: every output within 1e-4 and every parameter gradient at the bars of
    tests/test_backbone_variants_host.py; every grouped 3x3 -- and nothing else -- goes through the grouped entry points."""
    from monodetr_b200 import _lib
    from monodetr_b200.bench_model import surrogate_loss
    fake_device_lib.install(monkeypatch, {"tf32x3": 1, "bf16x3": 2}[precision])
    fake = GroupedFakeLib({"tf32x3": 1, "bf16x3": 2}[precision])
    monkeypatch.setattr(_lib, "_lib", fake)
    from monodetr_b200 import build_monodetr, tc
    assert tc.get_precision() == precision
    cfg = obg.variant_cfg("resnext50_32x4d", dilation)
    m, _ = build_monodetr(_model_cfg("resnext50_32x4d", dilation, dropout=0.0, device="cpu"))
    sd = obg.deterministic_state_dict(cfg)
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
    ref = obg.forward(sdg, images, calibs, sizes, training=True, cfg=cfg)
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
    assert len(errs) == 313
    # worst bar 1e-1 in both modes: a few gradients behind the bilinear sampling locations (layer4.0.conv2 under DC5: 3.2e-2
    # in tf32x3) differ by O(1e-2) between two fp32 evaluation orders (tests/test_oracle_model.py)
    med_bar, worst_bar = (1e-3 if precision == "bf16x3" else 3e-4), 1e-1
    assert errs[len(errs) // 2][0] < med_bar, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < worst_bar or scale < 1e-6, (name, err, scale)

    # 16 grouped 3x3s forward (layer1 included), the 13 of layers 2-4 also backward, nothing else grouped; the weights are
    # packed by one call and their gradients unpacked by one
    blocks = obg.resnet_blocks(cfg)
    want_fwd = [("forward", width, 32, stride, dil, dil) for _, _, _, stride, dil, width, _ in blocks]
    want_bwd = [(kind, width, 32, stride, dil, dil) for name, _, _, stride, dil, width, _ in blocks if name != "layer1"
                for kind in ("dgrad", "wgrad")]
    assert sorted(fake.grouped_log) == sorted(want_fwd + want_bwd)
    assert fake.calls.get("mdb_conv2d_forward_dilated_f32", 0) == fake.calls.get("mdb_conv2d_forward_dilated_bf16x3", 0) == 0
    assert fake.calls["mdb_pack_conv_weights_grouped_multi_" + ("bf16x3" if precision == "bf16x3" else "f32")] == 1
    assert fake.calls["mdb_unpack_conv_wgrads_grouped_multi_f32"] == 1
