"""Golden vectors of the reference model with anchor-box queries (`use_dab: True`), so that the oracle and the product model can
be checked against the UNMODIFIED reference without it present.  Needs the reference source tree (MONODETR_REFERENCE, see
ref_shims):

    python tools/gen_golden_dab.py   -> tests/golden/dab.npz

Keys (the configs/monodetr.yaml model section with use_dab set, on the weights of tests/oracle_dab.deterministic_state_dict()):
  dab.spec, r101.spec   names (state_dict order), shapes and trainable flags of build_monodetr(cfg), resnet50 and resnet101
  fwd_eval_*            eval-mode outputs (aux included) at 1 x 3 x 192 x 640
  b1.fwd_train_*        train-mode outputs (dropout off) at 1 x 3 x 96 x 320, and for the surrogate loss of that forward
  b1.grad_names         every parameter that gets a gradient, per name in that order max|grad| and the gradient at
  b1.grad_max / val / len   grad_index(numel, name) (as tools/gen_golden_backbones.py)
  b1.grad_full.<name>   the whole gradient of the anchors and of the DAB MLPs' first-layer biases
  b2.*                  the same at batch 2 (pins the batch sum of the anchor gradient)
An output of more than FWD_SAMPLES elements is stored as a seeded sample (gen_golden_reference_pins.sampled_forward).
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
from gen_golden_backbones import grad_index, store_forward, store_outputs  # noqa: E402
import oracle_dab as od  # noqa: E402
from oracle import monodetr_torch as om  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "dab.npz")
FULL_GRADS = ("refpoint_embed.weight", "depthaware_transformer.decoder.ref_point_head.layers.0.bias",
              "depthaware_transformer.decoder.query_scale.layers.0.bias")


def build_reference(pkg, dropout, backbone="resnet50"):
    cfg = ref_shims.load_cfg()["model"]
    cfg.update(use_dab=True, dropout=dropout, backbone=backbone)
    torch.manual_seed(0)
    model, _ = pkg.build_monodetr(cfg)
    if dropout == 0.0:
        # the depth encoder hard-codes dropout=0.1 (depth_predictor.py:49-50): neutralise every dropout in memory
        for m in model.modules():
            if isinstance(m, torch.nn.Dropout):
                m.p = 0.0
            if isinstance(m, torch.nn.MultiheadAttention):
                m.dropout = 0.0
    return model


def spec_of(model):
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    spec = [[k, list(v.shape), k in trainable] for k, v in model.state_dict().items()]
    return np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8), len(spec)


def main():
    pkg = ref_shims.install()
    res = {}
    res["dab.spec"], n = spec_of(build_reference(pkg, 0.1))
    res["r101.spec"], n101 = spec_of(build_reference(pkg, 0.1, "resnet101"))
    print(f"state_dict entries: resnet50 {n}, resnet101 {n101}", flush=True)

    sd = om.with_aliases(od.deterministic_state_dict())
    model = build_reference(pkg, 0.0)
    model.load_state_dict(sd)
    model.eval()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        store_outputs(res, "fwd_eval", model(images, calibs, None, sizes))

    model.train(True)
    for B in (1, 2):
        tag = f"b{B}"
        model.zero_grad(set_to_none=True)
        images, calibs, sizes = om.synthetic_inputs(B, 0, H=96, W=320)
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
            if name in FULL_GRADS:
                res[f"{tag}.grad_full.{name}"] = p.grad.numpy().copy()
        res[f"{tag}.grad_names"] = np.frombuffer(json.dumps(names).encode(), dtype=np.uint8)
        res[f"{tag}.grad_max"] = np.array(gmax, dtype=np.float32)
        res[f"{tag}.grad_val"] = np.concatenate(gval)
        res[f"{tag}.grad_len"] = np.array([len(v) for v in gval], dtype=np.int32)
        print(f"{tag}: {len(names)} gradients", flush=True)

    np.savez_compressed(OUT, **res)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, {len(res)} arrays)")


if __name__ == "__main__":
    main()
