"""ResNet backbones on the sm_90a kernels -- host-side mirror of the reference's
lib/models/monodetr/backbone.py (FrozenBatchNorm2d :27-64, BackboneBase :67-90, Backbone :93-108, Joiner
:111-126, build_backbone :129-135) with torchvision's bottleneck ResNets (resnet50 / 101 / 152, the ResNeXts resnext50_32x4d / resnext101_32x8d /
resnext101_64x4d and the wide ResNets wide_resnet50_2 / 101_2; v1.5: stride on the 3x3; optionally with layer4's stride
replaced by dilation 2, the "DC5" variant) restated as parameter containers with the same state_dict keys
(`backbone.0.body.*`).

Execution is ONE hand-scheduled autograd Function (no cuDNN, no per-layer autograd nodes):
  * conv1 7x7/2 + FrozenBN + ReLU and max-pool: dedicated forward-only kernels (conv1/layer1 are frozen, :71-73);
  * every other conv is the wgmma implicit-GEMM kernel with FrozenBN folded in: scale into the packed weights,
    shift as the epilogue bias, ReLU / residual-add+ReLU in the epilogue, activations NHWC; a ResNeXt's grouped 3x3
    conv2 runs the channel-banded form of that kernel (tc.conv2d_* with groups);
  * backward: dgrad kernels apply the previous ReLU's mask (and add the identity-branch gradient) in their
    epilogue, wgrad kernels multiply by the BN scale per output row; layer1 and the stem get no backward.
"""
import os
from typing import List

import torch
from torch import nn
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from . import _lib, tc
from .position_encoding import build_position_encoding

# (stage, planes, stride) of torchvision's ResNet, and the blocks per stage of each bottleneck depth it builds
_STAGES = [("layer1", 64, 1), ("layer2", 128, 2), ("layer3", 256, 2), ("layer4", 512, 2)]
RESNET_DEPTHS = {"resnet50": (3, 4, 6, 3), "resnet101": (3, 4, 23, 3), "resnet152": (3, 8, 36, 3)}
# torchvision's ResNeXts and wide ResNets by name: (blocks per stage, groups, width_per_group); the 3x3 of a block with
# `planes` has width = planes * width_per_group / 64 * groups channels
RESNEXT_BODIES = {
    "resnext50_32x4d": (RESNET_DEPTHS["resnet50"], 32, 4),
    "resnext101_32x8d": (RESNET_DEPTHS["resnet101"], 32, 8),
    "resnext101_64x4d": (RESNET_DEPTHS["resnet101"], 64, 4),
    "wide_resnet50_2": (RESNET_DEPTHS["resnet50"], 1, 128),
    "wide_resnet101_2": (RESNET_DEPTHS["resnet101"], 1, 128),
}
# torchvision's IMAGENET1K_V1 checkpoint of each body, which the reference's `pretrained=True` loads: (file name under
# torch.hub.get_dir()/checkpoints, torchvision weights enum).  A dilated C5 stage has the same weights.
IMAGENET1K_V1 = {
    "resnet50": ("resnet50-0676ba61.pth", "ResNet50_Weights"),
    "resnet101": ("resnet101-63fe2227.pth", "ResNet101_Weights"),
    "resnet152": ("resnet152-394f9c45.pth", "ResNet152_Weights"),
    "resnext50_32x4d": ("resnext50_32x4d-7cdf4587.pth", "ResNeXt50_32X4D_Weights"),
    "resnext101_32x8d": ("resnext101_32x8d-8ba56ff5.pth", "ResNeXt101_32X8D_Weights"),
    "resnext101_64x4d": ("resnext101_64x4d-173b62eb.pth", "ResNeXt101_64X4D_Weights"),
    "wide_resnet50_2": ("wide_resnet50_2-95faca4d.pth", "Wide_ResNet50_2_Weights"),
    "wide_resnet101_2": ("wide_resnet101_2-32ee1156.pth", "Wide_ResNet101_2_Weights"),
}


class FrozenBatchNorm2d(nn.Module):
    """Buffers only (never trained): y = x * scale + shift with scale = w * rsqrt(rv + eps) (reference :54-64)."""

    def __init__(self, n, eps=1e-5):
        super().__init__()
        self.register_buffer("weight", torch.ones(n))
        self.register_buffer("bias", torch.zeros(n))
        self.register_buffer("running_mean", torch.zeros(n))
        self.register_buffer("running_var", torch.ones(n))
        self.eps = eps

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        state_dict.pop(prefix + "num_batches_tracked", None)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs)

    def scale_shift(self):
        scale = self.weight * (self.running_var + self.eps).rsqrt()
        return scale.contiguous(), (self.bias - self.running_mean * scale).contiguous()


def _conv(cin, cout, k, stride=1, dilation=1, groups=1):
    m = nn.Conv2d(cin, cout, k, stride=stride, padding=dilation * (k // 2), dilation=dilation, groups=groups,
                  bias=False)   # parameter container only
    nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
    return m


class Bottleneck(nn.Module):
    expansion = 4

    def __init__(self, inplanes, planes, stride, downsample, dilation=1, groups=1, width_per_group=64):
        super().__init__()
        width = int(planes * (width_per_group / 64.0)) * groups      # torchvision's Bottleneck
        self.conv1 = _conv(inplanes, width, 1)
        self.bn1 = FrozenBatchNorm2d(width)
        self.conv2 = _conv(width, width, 3, stride, dilation, groups)
        self.bn2 = FrozenBatchNorm2d(width)
        self.conv3 = _conv(width, planes * 4, 1)
        self.bn3 = FrozenBatchNorm2d(planes * 4)
        self.downsample = None
        if downsample:
            self.downsample = nn.Sequential(_conv(inplanes, planes * 4, 1, stride), FrozenBatchNorm2d(planes * 4))
        self.stride = stride
        self.dilation = dilation
        self.groups = groups


class ResNetBody(nn.Module):
    """Parameter tree with torchvision's names: conv1, bn1, layer1..layer4 (what IntermediateLayerGetter keeps).
    `depths` = blocks per stage (RESNET_DEPTHS); `dilate_c5` = torchvision's replace_stride_with_dilation=[False, False, True]:
    layer4's block 0 keeps dilation 1 with stride 1 (its 1x1 downsample too), blocks 1.. are 3x3 with dilation 2 / padding 2.
    `groups` / `width_per_group`: torchvision's ResNeXt / wide ResNet arguments (RESNEXT_BODIES)."""

    def __init__(self, depths=RESNET_DEPTHS["resnet50"], dilate_c5=False, groups=1, width_per_group=64):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 64, 7, stride=2, padding=3, bias=False)
        nn.init.kaiming_normal_(self.conv1.weight, mode="fan_out", nonlinearity="relu")
        self.bn1 = FrozenBatchNorm2d(64)
        inplanes = 64
        for (name, planes, stride), blocks in zip(_STAGES, depths):
            dilated = dilate_c5 and name == "layer4"
            layers = []
            for i in range(blocks):
                if dilated:      # (stride, dilation): torchvision's _make_layer with dilate=True
                    blk_stride, blk_dil = 1, (1 if i == 0 else stride)
                else:
                    blk_stride, blk_dil = (stride if i == 0 else 1), 1
                layers.append(Bottleneck(inplanes, planes, blk_stride, downsample=(i == 0), dilation=blk_dil, groups=groups,
                                         width_per_group=width_per_group))
                inplanes = planes * 4
            setattr(self, name, nn.Sequential(*layers))

    def blocks(self):
        for name, _, _ in _STAGES:
            for blk in getattr(self, name):
                yield name, blk


# ------------------------------------------------------------------------------------------------------------
class _ResNetFn(Function):
    """images NCHW -> (layer2, layer3, layer4) NHWC.  args = (images, n_params, *conv_weights, *bn_scale_shift)."""

    @staticmethod
    def forward(ctx, images, meta, *tensors):
        nconv = meta["nconv"]
        weights = tensors[:nconv]
        scales = tensors[nconv:2 * nconv]
        shifts = tensors[2 * nconv:3 * nconv]
        B, _, H, W = images.shape
        dev = images.device
        # ---- stem (frozen) --------------------------------------------------------------------------------
        H1, W1 = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        y = torch.empty((B, H1, W1, 64), dtype=torch.float32, device=dev)
        _lib.call("mdb_stem_conv7x7_bn_relu_f32", images.contiguous(), weights[0].contiguous(), scales[0], shifts[0], y, B, H, W)
        H2, W2 = (H1 + 2 - 3) // 2 + 1, (W1 + 2 - 3) // 2 + 1
        x = torch.empty((B, H2, W2, 64), dtype=torch.float32, device=dev)
        _lib.call("mdb_maxpool3x3s2_nhwc_f32", y, x, B, H1, W1, 64)
        del y
        # ---- bottlenecks ----------------------------------------------------------------------------------
        saved, packed, feats = [], [], []
        # all bottleneck weights re-laid-out to [tap][O][I] with the BN scale folded in by ONE launch per 64 tensors (52 tensors).
        # (Running this re-layout on a branch stream beside the stem was measured: 332.6 vs 332.1 img/s, within noise -- the stem
        # fills every SM, the memory-bound re-layout only finds room in its tail; not kept.)
        # A ResNeXt's grouped conv2 weights go to the band-local layout instead, all of them by one more launch.
        grouped = meta["grouped"]                                    # conv index -> groups
        dense = [j for j in range(1, nconv) if j not in grouped]
        if tc.get_precision() == "bf16x3":      # (hi, lo) bf16 operands for fprop and dgrad, BN scale folded before the split
            dense_wp = tc.split_weights([weights[j].detach() for j in dense], [scales[j] for j in dense])
        else:
            dense_wp = tc.pack_weights_multi([weights[j] for j in dense], [scales[j] for j in dense])
        all_wp = [None] * nconv
        for j, w in zip(dense, dense_wp):
            all_wp[j] = w
        gj = list(grouped)
        for j, w in zip(gj, tc.pack_grouped_multi([weights[j].detach() for j in gj], [scales[j] for j in gj],
                                                  [grouped[j] for j in gj])):
            all_wp[j] = w
        ci = 1
        for bi, (stage, stride, dil, has_ds, trainable, groups) in enumerate(meta["blocks"]):
            idx = [ci, ci + 1, ci + 2] + ([ci + 3] if has_ds else [])
            ci += len(idx)
            wp = [all_wp[j] for j in idx]
            o1 = tc.conv2d_forward(x, wp[0], shifts[idx[0]], None, 1, 1, 1, 0, relu=True, round_out=True)
            o2 = tc.conv2d_forward(o1, wp[1], shifts[idx[1]], None, 3, 3, stride, dil, relu=True, round_out=True, dilation=dil,
                                   groups=groups)
            if has_ds:
                idn = tc.conv2d_forward(x, wp[3], shifts[idx[3]], None, 1, 1, stride, 0, relu=False)
            else:
                idn = x
            out = tc.conv2d_forward(o2, wp[2], shifts[idx[2]], idn, 1, 1, 1, 0, relu=True, round_out=True)
            if trainable:
                saved.append((x, o1, o2, out))
                packed.append(wp)
            x = out
            if meta["stage_end"][bi] and stage != "layer1":
                feats.append(out)
        ctx.meta = meta
        ctx.saved = saved           # plain python refs: these are never exposed to autograd users
        ctx.packed = packed
        ctx.scales = scales
        return tuple(feats)

    @staticmethod
    @once_differentiable
    def backward(ctx, *gfeats):
        meta = ctx.meta
        nconv = meta["nconv"]
        blocks = [b for b in meta["blocks"] if b[4]]                 # trainable blocks, in forward order
        ends = [e for b, e in zip(meta["blocks"], meta["stage_end"]) if b[4]]
        conv_idx = meta["train_conv_idx"]                            # per trainable block: indices into weights
        grads = [None] * (3 * nconv)
        # which feature gradient enters after which trainable block
        feat_of_block = {}
        f = 0
        for k, e in enumerate(ends):
            if e:
                feat_of_block[k] = f
                f += 1
        g = None                                                      # grad wrt block output, already ReLU-masked
        pending = []                                                  # 3x3 weight gradients still in packed layout
        pending_grouped = []                                          # ... in band-local layout (grouped conv2)
        for k in range(len(blocks) - 1, -1, -1):
            stage, stride, dil, has_ds, _, groups = blocks[k]
            x, o1, o2, out = ctx.saved[k]
            wp = ctx.packed[k]
            idx = conv_idx[k]
            sc = [ctx.scales[j] for j in idx]
            if g is None:                                             # last block: only the neck's gradient
                g = _relu_mask(gfeats[feat_of_block[k]].contiguous(), out)
            # conv3
            grads[idx[2]] = tc.conv2d_wgrad(g, o2, sc[2], 1, 1, 1, 0).view_as(_w(ctx, idx[2]))
            g2 = tc.conv2d_dgrad(g, wp[2], o2.shape, None, o2, 1, 1, 1, 0, round_out=True)
            # conv2 (3x3, maybe strided or dilated; padding = dilation)
            dw2 = tc.conv2d_wgrad(g2, o1, sc[1], 3, 3, stride, dil, dilation=dil, groups=groups)
            (pending if groups == 1 else pending_grouped).append((idx[1], groups, dw2))   # -> OIHW at the end
            g1 = tc.conv2d_dgrad(g2, wp[1], o1.shape, None, o1, 3, 3, stride, dil, round_out=True, dilation=dil, groups=groups)
            # conv1
            grads[idx[0]] = tc.conv2d_wgrad(g1, x, sc[0], 1, 1, 1, 0).view_as(_w(ctx, idx[0]))
            if has_ds:
                grads[idx[3]] = tc.conv2d_wgrad(g, x, sc[3], 1, 1, stride, 0).view_as(_w(ctx, idx[3]))
            if k == 0:
                break                                                 # input of the first trainable block is frozen
            # gradient wrt this block's input = conv1 path + identity/downsample path (+ the neck's gradient if the
            # input is a returned feature), masked by the input's own ReLU -> it is the previous block's `g`.
            extra = gfeats[feat_of_block[k - 1]].contiguous() if (k - 1) in feat_of_block else None
            if has_ds:
                side = tc.conv2d_dgrad(g, wp[3], x.shape, extra, None, 1, 1, stride, 0)
            else:
                side = g if extra is None else g + extra
            g = tc.conv2d_dgrad(g1, wp[0], x.shape, side, x, 1, 1, 1, 0, round_out=True)
            ctx.saved[k] = None
        ctx.saved = ctx.packed = None
        for (j, _, _), dw in zip(pending, tc.unpack_wgrads_multi([d for _, _, d in pending], [(3, 3)] * len(pending))):
            grads[j] = dw
        for (j, _, _), dw in zip(pending_grouped, tc.unpack_grouped_wgrads_multi([d for _, _, d in pending_grouped],
                                                                                  [g for _, g, _ in pending_grouped])):
            grads[j] = dw
        return (None, None) + tuple(grads)


def _w(ctx, j):
    return ctx.meta["weight_shapes"][j]


def _relu_mask(dy, y):
    from .functional import relu_backward
    return relu_backward(dy, y)


class BackboneBase(nn.Module):
    def __init__(self, body: nn.Module, train_backbone: bool, return_interm_layers: bool):
        super().__init__()
        for name, parameter in body.named_parameters():
            if not train_backbone or ("layer2" not in name and "layer3" not in name and "layer4" not in name):
                parameter.requires_grad_(False)
        assert return_interm_layers, "MonoDETR uses the 3 intermediate levels (num_feature_levels = 4)"
        self.strides = [8, 16, 32]
        self.num_channels = [512, 1024, 2048]
        self.body = body
        self._bn_cache = None

    def _bn_tensors(self):
        """The frozen BatchNorms folded into per-channel scale / shift, recomputed when a buffer has changed.  On the same
        device the new values are written into the tensors already handed out, so that a CUDA graph captured with them (the
        Detector's) reads the buffers as they are after a load_state_dict."""
        key = tuple(b._version for b in self.body.buffers()) + (str(next(self.body.buffers()).device),)
        if self._bn_cache is None or self._bn_cache[0] != key:
            sc, sh = [], []
            with torch.no_grad():
                for bn in self._bns():
                    a, b = bn.scale_shift()
                    sc.append(a)
                    sh.append(b)
                old = self._bn_cache
                if old is not None and old[0][-1] == key[-1]:
                    for dst, src in zip(old[1] + old[2], sc + sh):
                        dst.copy_(src)
                    sc, sh = old[1], old[2]
            self._bn_cache = (key, sc, sh)
        return self._bn_cache[1], self._bn_cache[2]

    def _convs(self):
        convs = [self.body.conv1]
        for _, blk in self.body.blocks():
            convs += [blk.conv1, blk.conv2, blk.conv3] + ([blk.downsample[0]] if blk.downsample is not None else [])
        return convs

    def _bns(self):
        bns = [self.body.bn1]
        for _, blk in self.body.blocks():
            bns += [blk.bn1, blk.bn2, blk.bn3] + ([blk.downsample[1]] if blk.downsample is not None else [])
        return bns

    def forward(self, images):
        """images (B, 3, H, W) NCHW -> list of 3 NHWC feature maps (layer2, layer3, layer4)."""
        if not images.is_cuda:
            raise RuntimeError("monodetr_b200 backbone: CUDA tensors required (there is no CPU path)")
        convs = self._convs()
        sc, sh = self._bn_tensors()
        blocks, stage_end, train_idx, grouped = [], [], [], {}
        ci = 1
        names = [n for n, _ in self.body.blocks()]
        for i, (name, blk) in enumerate(self.body.blocks()):
            has_ds = blk.downsample is not None
            trainable = blk.conv1.weight.requires_grad
            blocks.append((name, blk.stride, blk.dilation, has_ds, trainable, blk.groups))
            stage_end.append(i + 1 == len(names) or names[i + 1] != name)
            idx = [ci, ci + 1, ci + 2] + ([ci + 3] if has_ds else [])
            if blk.groups != 1:
                grouped[ci + 1] = blk.groups
            if trainable:
                train_idx.append(idx)
            ci += len(idx)
        meta = {"nconv": len(convs), "blocks": blocks, "stage_end": stage_end, "train_conv_idx": train_idx, "grouped": grouped,
                "weight_shapes": [torch.empty(c.weight.shape, device="meta") for c in convs]}
        weights = [c.weight for c in convs]
        return list(_ResNetFn.apply(images, meta, *weights, *sc, *sh))


def _unsupported(name):
    # resnet18 / 34 (basic blocks: the reference asserts against them) and unknown names
    return NotImplementedError(f"monodetr_b200 backbone {name!r}: Backbone builds {', '.join(RESNET_DEPTHS)} and ResNeXtBackbone "
                               f"builds {', '.join(RESNEXT_BODIES)}, each with dilation False or True (build_backbone picks the "
                               "class by name)")


class Backbone(BackboneBase):
    """ResNet backbone with frozen BatchNorm (reference :93-108): torchvision's bottleneck ResNets with plain convolutions
    (resnet50 / resnet101 / resnet152), each with or without the dilated C5 stage."""

    def __init__(self, name: str, train_backbone: bool, return_interm_layers: bool, dilation: bool):
        if name not in RESNET_DEPTHS:
            raise _unsupported(name)
        super().__init__(ResNetBody(RESNET_DEPTHS[name], bool(dilation)), train_backbone, return_interm_layers)
        if dilation:
            self.strides[-1] = self.strides[-1] // 2


class ResNeXtBackbone(BackboneBase):
    """The same with torchvision's grouped or widened bottlenecks (RESNEXT_BODIES: resnext50_32x4d / resnext101_32x8d /
    resnext101_64x4d, wide_resnet50_2 / wide_resnet101_2), each with or without the dilated C5 stage."""

    def __init__(self, name: str, train_backbone: bool, return_interm_layers: bool, dilation: bool):
        if name not in RESNEXT_BODIES:
            raise _unsupported(name)
        depths, groups, width_per_group = RESNEXT_BODIES[name]
        super().__init__(ResNetBody(depths, bool(dilation), groups, width_per_group), train_backbone, return_interm_layers)
        if dilation:
            self.strides[-1] = self.strides[-1] // 2


class Joiner(nn.Sequential):
    def __init__(self, backbone, position_embedding):
        super().__init__(backbone, position_embedding)
        self.strides = backbone.strides
        self.num_channels = backbone.num_channels

    def forward(self, images):
        feats: List[torch.Tensor] = self[0](images)
        pos = [self[1](f) for f in feats]
        return feats, pos


def imagenet_checkpoint_path(name):
    """Where torchvision keeps the IMAGENET1K_V1 file of backbone `name`: torch.hub.get_dir()/checkpoints/<file>."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", IMAGENET1K_V1[name][0])


def load_imagenet_weights(body, name, source=True):
    """Copy a torchvision ImageNet state_dict into `body` (a ResNetBody built for backbone `name`), bit for bit.

    source: True reads torchvision's IMAGENET1K_V1 file from the torch hub cache (imagenet_checkpoint_path), a path reads that
    file.  Nothing is downloaded: a missing file raises FileNotFoundError.  `fc.*` and `num_batches_tracked` entries are
    ignored; every other entry must be one of the body's, with its shape and finite values, and every body entry must be
    present (ValueError names the first that is not).  Draws no random numbers, and may run on a body that has already run
    a forward: the folded BN tensors and weight splits are rebuilt from the new values."""
    if source is True:
        path = imagenet_checkpoint_path(name)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"backbone {name!r}: torchvision's ImageNet weights ({IMAGENET1K_V1[name][1]}.IMAGENET1K_V1) "
                                    f"are not at {path}; place the file there (or give its path as pretrained_backbone)")
    else:
        path = os.fspath(source)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"backbone {name!r}: no ImageNet weights file at {path}")
    sd = torch.load(path, map_location="cpu", weights_only=True)
    sd = {k: v for k, v in sd.items() if not k.startswith("fc.") and not k.endswith("num_batches_tracked")}
    own = body.state_dict()
    for k, t in own.items():
        if k not in sd:
            raise ValueError(f"{path}: no entry {k!r} of backbone {name!r}")
        v = sd[k]
        if tuple(v.shape) != tuple(t.shape):
            raise ValueError(f"{path}: {k!r} has shape {tuple(v.shape)}, backbone {name!r} needs {tuple(t.shape)}")
        if not v.is_floating_point() or not bool(torch.isfinite(v).all()):
            raise ValueError(f"{path}: {k!r} holds non-finite or non-floating-point values")
    for k in sd:
        if k not in own:
            raise ValueError(f"{path}: entry {k!r} is not part of backbone {name!r}")
    with torch.no_grad():
        for k, t in own.items():
            t.copy_(sd[k])


def build_backbone(cfg):
    """cfg["pretrained_backbone"] (default False: random initialisation): True or a file path loads torchvision's ImageNet
    weights into the ResNet body (load_imagenet_weights) on the main process only -- rank 0 of an initialised default process
    group, like the reference's `pretrained=is_main_process()`.  The other ranks keep their random weights: `Trainer`
    broadcasts rank 0's parameters and buffers when it is constructed; other callers must broadcast them themselves."""
    position_embedding = build_position_encoding(cfg)
    return_interm_layers = cfg["masks"] or cfg["num_feature_levels"] > 1
    cls = ResNeXtBackbone if cfg["backbone"] in RESNEXT_BODIES else Backbone
    backbone = cls(cfg["backbone"], cfg["train_backbone"], return_interm_layers, cfg["dilation"])
    pretrained = cfg.get("pretrained_backbone", False)
    if pretrained is not False and pretrained is not None and _is_main_process():
        load_imagenet_weights(backbone.body, cfg["backbone"], pretrained)
    return Joiner(backbone, position_embedding)


def _is_main_process():
    import torch.distributed as dist
    return not (dist.is_available() and dist.is_initialized()) or dist.get_rank() == 0
