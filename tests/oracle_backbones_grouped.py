"""TEST INFRASTRUCTURE: the CPU oracle for the reference's ResNeXt and wide-ResNet backbones -- torchvision's
resnext50_32x4d / resnext101_32x8d / resnext101_64x4d / wide_resnet50_2 / wide_resnet101_2 (bottleneck width
int(planes * width_per_group / 64) * groups, conv2 grouped), each optionally with the dilated C5 stage.  Like
tests/oracle_backbones.py (which it leaves as it is) it restates only the backbone and its state_dict entries and runs
everything else through oracle/monodetr_torch.py.  Pinned to the unmodified reference by tests/test_backbone_grouped_host.py
(tests/golden/backbones_grouped.npz)."""
import contextlib

import torch.nn.functional as F

from oracle import monodetr_torch as om
import oracle_backbones as ob

# name -> (blocks per stage, groups, width_per_group): torchvision's resnext* / wide_resnet* constructors
BODIES = {
    "resnext50_32x4d": ((3, 4, 6, 3), 32, 4),
    "resnext101_32x8d": ((3, 4, 23, 3), 32, 8),
    "resnext101_64x4d": ((3, 4, 23, 3), 64, 4),
    "wide_resnet50_2": ((3, 4, 6, 3), 1, 128),
    "wide_resnet101_2": ((3, 4, 23, 3), 1, 128),
}
_resnet50_spec = om.state_dict_spec


def variant_cfg(backbone, dilation):
    return dict(om.CFG, backbone=backbone, dilation=dilation)


def resnet_blocks(cfg):
    """(stage, block index, planes, stride, dilation, width, groups) of every bottleneck (torchvision's _make_layer)."""
    depths, groups, wpg = BODIES[cfg["backbone"]]
    out = []
    for (name, planes, stride), blocks in zip(ob.STAGES, depths):
        dilated = cfg["dilation"] and name == "layer4"
        width = int(planes * (wpg / 64.0)) * groups
        for b in range(blocks):
            if dilated:
                out.append((name, b, planes, 1, 1 if b == 0 else stride, width, groups))
            else:
                out.append((name, b, planes, stride if b == 0 else 1, 1, width, groups))
    return out


def bottleneck(sd, p, x, stride, dilation, groups):
    out = F.relu(om.frozen_bn(sd, p + ".bn1", F.conv2d(x, sd[p + ".conv1.weight"])))
    out = F.relu(om.frozen_bn(sd, p + ".bn2", F.conv2d(out, sd[p + ".conv2.weight"], stride=stride, padding=dilation,
                                                       dilation=dilation, groups=groups)))
    out = om.frozen_bn(sd, p + ".bn3", F.conv2d(out, sd[p + ".conv3.weight"]))
    if (p + ".downsample.0.weight") in sd:
        x = om.frozen_bn(sd, p + ".downsample.1", F.conv2d(x, sd[p + ".downsample.0.weight"], stride=stride))
    return F.relu(out + x)


def backbone(sd, images, cfg):
    p = "backbone.0.body."
    x = F.relu(om.frozen_bn(sd, p + "bn1", F.conv2d(images, sd[p + "conv1.weight"], stride=2, padding=3)))
    x = F.max_pool2d(x, 3, 2, 1)
    feats = []
    blocks = resnet_blocks(cfg)
    for i, (name, b, _, stride, dilation, _, groups) in enumerate(blocks):
        x = bottleneck(sd, f"{p}{name}.{b}", x, stride, dilation, groups)
        if name != "layer1" and (i + 1 == len(blocks) or blocks[i + 1][0] != name):
            feats.append(x)
    return feats


def state_dict_spec(cfg):
    b = "backbone.0.body."
    spec = {}

    def bn(p, n):
        for k in ("weight", "bias", "running_mean", "running_var"):
            spec[f"{p}.{k}"] = (n,)
    spec[b + "conv1.weight"] = (64, 3, 7, 7)
    bn(b + "bn1", 64)
    inplanes = 64
    for name, i, planes, _, _, width, groups in resnet_blocks(cfg):
        p = f"{b}{name}.{i}"
        spec[p + ".conv1.weight"] = (width, inplanes, 1, 1); bn(p + ".bn1", width)
        spec[p + ".conv2.weight"] = (width, width // groups, 3, 3); bn(p + ".bn2", width)
        spec[p + ".conv3.weight"] = (planes * 4, width, 1, 1); bn(p + ".bn3", planes * 4)
        if i == 0:
            spec[p + ".downsample.0.weight"] = (planes * 4, inplanes, 1, 1); bn(p + ".downsample.1", planes * 4)
        inplanes = planes * 4
    spec.update((k, v) for k, v in _resnet50_spec(cfg).items() if not k.startswith(b))
    return spec


@contextlib.contextmanager
def _variant(cfg):
    saved = om.backbone, om.state_dict_spec
    om.backbone = lambda sd, images: backbone(sd, images, cfg)
    om.state_dict_spec = lambda c=cfg: state_dict_spec(c)
    try:
        yield
    finally:
        om.backbone, om.state_dict_spec = saved


def deterministic_state_dict(cfg):
    with _variant(cfg):
        return om.deterministic_state_dict(cfg)


def forward(sd, images, calibs, img_sizes, training=False, cfg=None):
    with _variant(cfg):
        return om.forward(sd, images, calibs, img_sizes, training=training, cfg=cfg)
