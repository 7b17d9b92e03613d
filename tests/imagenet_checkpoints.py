"""TEST INFRASTRUCTURE: synthetic checkpoints in the format of torchvision's ImageNet files (what `pretrained_backbone` reads):
the ResNet body's entries without the `backbone.0.body.` prefix (names and shapes from tests/oracle_backbones.py and
tests/oracle_backbones_grouped.py), plus `fc.weight`, `fc.bias` and every BatchNorm's `num_batches_tracked`, which the
loader ignores.  No torchvision and no network involved.

`statistics="imagenet"` draws per-channel FrozenBN statistics far from 1, as trained networks have them: running_var
log-uniform over [1e-6, 1e2], weight uniform over [-1, 3] with every 16th channel exactly 0, running_mean N(0, 2^2), bias
N(0, 1); conv weights are Kaiming-scaled (fan_out, ReLU, as torchvision initialises them) and then multiplied per output
channel by sqrt(running_var + eps) / 4.  That product is what keeps such statistics meaningful: in a trained network
running_var is the variance of the conv's own output, so the raw weights span the same eight decades while the folded
weight (BN scale times conv weight) is O(weight).  Drawn independently of the weights instead, the BN scales (up to ~1e3)
multiply through 16 to 50 blocks and overflow fp32 in the reference as on the device.  The 1/4 keeps the shift terms
(running_mean times scale, up to ~1e3) from growing the activations block over block.
"""
import os

import torch

import oracle_backbones as ob
import oracle_backbones_grouped as obg

NAMES = list(ob.RESNET_DEPTHS) + list(obg.BODIES)
PREFIX = "backbone.0.body."
EPS = 1e-5


def body_spec(name, dilation=False):
    """{torchvision key: shape} of the ResNet body of backbone `name` (dilation does not change it)."""
    mod = ob if name in ob.RESNET_DEPTHS else obg
    spec = mod.state_dict_spec(mod.variant_cfg(name, dilation))
    return {k[len(PREFIX):]: tuple(v) for k, v in spec.items() if k.startswith(PREFIX)}


def synthetic_checkpoint(name, seed=0, statistics="plain"):
    """A torchvision-format state_dict for backbone `name` (fp32; int64 num_batches_tracked).  'plain': N(0, 1) everywhere
    (for load tests: any bit pattern must arrive unchanged); 'imagenet': the statistics of the module docstring."""
    g = torch.Generator().manual_seed(seed)
    spec = body_spec(name)
    sd = {}
    if statistics == "plain":
        for k, shape in spec.items():
            sd[k] = torch.randn(shape, generator=g)
    elif statistics == "imagenet":
        bns = sorted({k.rsplit(".", 1)[0] for k in spec if k.endswith("running_var")})
        for p in bns:
            n = spec[p + ".running_var"][0]
            sd[p + ".running_var"] = 10.0 ** (torch.rand(n, generator=g, dtype=torch.float64) * 8 - 6)
            w = torch.rand(n, generator=g, dtype=torch.float64) * 4 - 1
            w[::16] = 0
            sd[p + ".weight"] = w
            sd[p + ".running_mean"] = torch.randn(n, generator=g, dtype=torch.float64) * 2
            sd[p + ".bias"] = torch.randn(n, generator=g, dtype=torch.float64)
        for k, shape in spec.items():
            if len(shape) != 4:
                continue
            conv = k[:-len(".weight")]
            bn = conv[:-len(".0")] + ".1" if conv.endswith("downsample.0") else conv.replace("conv", "bn")
            fan_out = shape[0] * shape[2] * shape[3]
            w = torch.randn(shape, generator=g, dtype=torch.float64) * (2.0 / fan_out) ** 0.5
            sd[k] = w * ((sd[bn + ".running_var"] + EPS).sqrt() / 4).view(-1, 1, 1, 1)
        sd = {k: sd[k].float() for k in spec}
    else:
        raise ValueError(statistics)
    for k in list(spec):
        if k.endswith("running_var"):
            sd[k[:-len("running_var")] + "num_batches_tracked"] = torch.tensor(seed, dtype=torch.int64)
    sd["fc.weight"] = torch.randn(1000, 2048, generator=g)
    sd["fc.bias"] = torch.randn(1000, generator=g)
    return sd


def write(sd, path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    torch.save(sd, path)
    return path
