"""TEST INFRASTRUCTURE: the CPU oracle (oracle/monodetr_torch.py) for the reference's other backbones -- torchvision's
resnet50 / resnet101 / resnet152 (v1.5, stride on the 3x3), each optionally with replace_stride_with_dilation=[False, False,
True] (the dilated C5 stage, "DC5"), selected like the reference's build_backbone (backbone.py:93-135) by cfg["backbone"] /
cfg["dilation"].  oracle/monodetr_torch.py states the resnet50 model; this module restates only the backbone and its
state_dict entries and runs everything else through that module's own functions, so that a variant differs from the
resnet50 oracle in the backbone alone.  Pinned to the unmodified reference by tests/test_backbone_variants_host.py
(tests/golden/backbones.npz)."""
import contextlib

import torch.nn.functional as F

from oracle import monodetr_torch as om

RESNET_DEPTHS = {"resnet50": (3, 4, 6, 3), "resnet101": (3, 4, 23, 3), "resnet152": (3, 8, 36, 3)}
STAGES = [("layer1", 64, 1), ("layer2", 128, 2), ("layer3", 256, 2), ("layer4", 512, 2)]
_resnet50_spec = om.state_dict_spec         # (kept: _variant points om.state_dict_spec at this module's while it runs)


def variant_cfg(backbone, dilation):
    """The oracle's cfg for a variant: om.CFG plus the two backbone keys."""
    return dict(om.CFG, backbone=backbone, dilation=dilation)


def resnet_blocks(cfg):
    """(stage, block index, planes, stride, dilation) of every bottleneck -- torchvision's _make_layer: a dilated layer4
    keeps stride 1, its block 0 dilation 1 (the stage's previous dilation), blocks 1.. dilation 2."""
    out = []
    for (name, planes, stride), blocks in zip(STAGES, RESNET_DEPTHS[cfg["backbone"]]):
        dilated = cfg["dilation"] and name == "layer4"
        for b in range(blocks):
            if dilated:
                out.append((name, b, planes, 1, 1 if b == 0 else stride))
            else:
                out.append((name, b, planes, stride if b == 0 else 1, 1))
    return out


def bottleneck(sd, p, x, stride, dilation):     # torchvision Bottleneck v1.5: stride on the 3x3, padding = dilation
    out = F.relu(om.frozen_bn(sd, p + ".bn1", F.conv2d(x, sd[p + ".conv1.weight"])))
    out = F.relu(om.frozen_bn(sd, p + ".bn2", F.conv2d(out, sd[p + ".conv2.weight"], stride=stride, padding=dilation,
                                                       dilation=dilation)))
    out = om.frozen_bn(sd, p + ".bn3", F.conv2d(out, sd[p + ".conv3.weight"]))
    if (p + ".downsample.0.weight") in sd:
        x = om.frozen_bn(sd, p + ".downsample.1", F.conv2d(x, sd[p + ".downsample.0.weight"], stride=stride))
    return F.relu(out + x)


def backbone(sd, images, cfg):                  # backbone.py:75-90 (returns layer2, layer3, layer4)
    p = "backbone.0.body."
    x = F.relu(om.frozen_bn(sd, p + "bn1", F.conv2d(images, sd[p + "conv1.weight"], stride=2, padding=3)))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    blocks = resnet_blocks(cfg)
    for i, (name, b, _, stride, dilation) in enumerate(blocks):
        x = bottleneck(sd, f"{p}{name}.{b}", x, stride, dilation)
        if name != "layer1" and (i + 1 == len(blocks) or blocks[i + 1][0] != name):
            feats.append(x)
    return feats


def state_dict_spec(cfg):
    """om.state_dict_spec() with the resnet50 body's entries replaced by the variant's (same names and order rules)."""
    b = "backbone.0.body."
    spec = {}

    def bn(p, n):
        for k in ("weight", "bias", "running_mean", "running_var"):
            spec[f"{p}.{k}"] = (n,)
    spec[b + "conv1.weight"] = (64, 3, 7, 7)
    bn(b + "bn1", 64)
    inplanes = 64
    for name, i, planes, _, _ in resnet_blocks(cfg):
        p = f"{b}{name}.{i}"
        spec[p + ".conv1.weight"] = (planes, inplanes, 1, 1); bn(p + ".bn1", planes)
        spec[p + ".conv2.weight"] = (planes, planes, 3, 3); bn(p + ".bn2", planes)
        spec[p + ".conv3.weight"] = (planes * 4, planes, 1, 1); bn(p + ".bn3", planes * 4)
        if i == 0:
            spec[p + ".downsample.0.weight"] = (planes * 4, inplanes, 1, 1); bn(p + ".downsample.1", planes * 4)
        inplanes = planes * 4
    spec.update((k, v) for k, v in _resnet50_spec(cfg).items() if not k.startswith(b))
    return spec


@contextlib.contextmanager
def _variant(cfg):
    """om's model-level functions look their backbone and spec up by module-global name: point them at the variant's."""
    saved = om.backbone, om.state_dict_spec
    om.backbone = lambda sd, images: backbone(sd, images, cfg)
    om.state_dict_spec = lambda c=cfg: state_dict_spec(c)
    try:
        yield
    finally:
        om.backbone, om.state_dict_spec = saved


def deterministic_state_dict(cfg):
    """om.deterministic_state_dict's per-name weights over the variant's names (a name's value does not depend on the
    variant: shared names get the resnet50 oracle's values)."""
    with _variant(cfg):
        return om.deterministic_state_dict(cfg)


def forward(sd, images, calibs, img_sizes, training=False, cfg=None):
    """om.forward with the variant's backbone."""
    with _variant(cfg):
        return om.forward(sd, images, calibs, img_sizes, training=training, cfg=cfg)
