"""Golden vectors of the reference model with its ResNeXt and wide-ResNet backbones (torchvision's resnext50_32x4d,
resnext101_32x8d, resnext101_64x4d, wide_resnet50_2, wide_resnet101_2), in the format of tools/gen_golden_backbones.py.
Needs the reference source tree (MONODETR_REFERENCE, see ref_shims):

    python tools/gen_golden_backbones_grouped.py   -> tests/golden/backbones_grouped.npz

Keys prefixed "<tag>.":
  spec            for every variant of SPEC_VARIANTS (each name with dilation False and True)
  fwd_eval_*, fwd_train_*, grad_*
                  for the variants of VARIANTS, as in gen_golden_backbones.py, on the weights of
                  tests/oracle_backbones_grouped.deterministic_state_dict(cfg)
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
warnings.filterwarnings("ignore")

import ref_shims  # noqa: E402
from gen_golden_backbones import build_reference, grad_index, store_outputs  # noqa: E402
import oracle_backbones_grouped as obg  # noqa: E402
from oracle import monodetr_torch as om  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "backbones_grouped.npz")
NAMES = ("resnext50_32x4d", "resnext101_32x8d", "resnext101_64x4d", "wide_resnet50_2", "wide_resnet101_2")
SPEC_VARIANTS = {f"{n}{'_dc5' if d else ''}": (n, d) for n in NAMES for d in (False, True)}
VARIANTS = {"resnext50_32x4d": ("resnext50_32x4d", False), "resnext50_32x4d_dc5": ("resnext50_32x4d", True),
            "wide_resnet50_2": ("wide_resnet50_2", False)}


def main():
    pkg = ref_shims.install()
    res = {}
    for tag, (backbone, dilation) in SPEC_VARIANTS.items():
        model = build_reference(pkg, backbone, dilation, 0.1)
        trainable = {n for n, p in model.named_parameters() if p.requires_grad}
        spec = [[k, list(v.shape), k in trainable] for k, v in model.state_dict().items()]
        res[f"{tag}.spec"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)
        print(f"{tag}: {len(spec)} state_dict entries", flush=True)
        del model
    for tag, (backbone, dilation) in VARIANTS.items():
        sd = om.with_aliases(obg.deterministic_state_dict(obg.variant_cfg(backbone, dilation)))
        model = build_reference(pkg, backbone, dilation, 0.0)
        model.load_state_dict(sd)
        model.eval()
        images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
        with torch.no_grad():
            store_outputs(res, f"{tag}.fwd_eval", model(images, calibs, None, sizes))

        model.train(True)
        images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
        out = model(images, calibs, None, sizes)
        store_outputs(res, f"{tag}.fwd_train", out)
        om.surrogate_loss(out).backward()
        names, gmax, gval = [], [], []
        for name, p in model.named_parameters():
            if p.grad is None:
                continue
            gr = p.grad.reshape(-1)
            names.append(name)
            gmax.append(float(gr.abs().max()))
            gval.append(gr[grad_index(gr.numel(), name)].numpy())
        res[f"{tag}.grad_names"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
        res[f"{tag}.grad_max"] = np.array(gmax, dtype=np.float32)
        res[f"{tag}.grad_val"] = np.concatenate(gval)
        res[f"{tag}.grad_len"] = np.array([len(v) for v in gval], dtype=np.int32)
        print(f"{tag}: {len(names)} gradients", flush=True)

    np.savez_compressed(OUT, **res)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, {len(res)} arrays)")


if __name__ == "__main__":
    main()
