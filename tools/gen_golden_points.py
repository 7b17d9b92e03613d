"""Golden vectors of the reference model with its other sampling-point counts, so that the oracle and the product model can be
checked against the UNMODIFIED reference without it present.  Needs the reference source tree (MONODETR_REFERENCE, see ref_shims):

    python tools/gen_golden_points.py   -> tests/golden/points.npz

For each (enc_n_points, dec_n_points) of VARIANTS (the configs/monodetr.yaml model section with both counts changed): 2 / 2 and
8 / 8 run on the fused kernels, 3 / 6 on the two-step path with different encoder and decoder counts.  Keys prefixed "<tag>.", as
tools/gen_golden_backbones.py stores them:
  spec            names (state_dict order), shapes and trainable flags of the reference's build_monodetr(cfg)
  fwd_eval_*      eval-mode outputs (aux included) at 1 x 3 x 192 x 640
  fwd_train_*     train-mode outputs (dropout off) at 1 x 3 x 96 x 320
  grad_names / grad_max / grad_val / grad_len   sampled gradients of the surrogate loss of that train forward
all on the weights of tests/oracle_points.deterministic_state_dict(cfg).
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(ROOT))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(os.path.dirname(ROOT), "tests"))
warnings.filterwarnings("ignore")

import ref_shims  # noqa: E402
from gen_golden_backbones import grad_index, store_outputs  # noqa: E402
import oracle_points as op  # noqa: E402
from oracle import monodetr_torch as om  # noqa: E402

OUT = os.path.join(os.path.dirname(ROOT), "tests", "golden", "points.npz")
VARIANTS = {"p2": (2, 2), "p8": (8, 8), "p3_6": (3, 6)}


def build_reference(pkg, points, dropout):
    cfg = ref_shims.load_cfg()["model"]
    cfg.update(enc_n_points=points[0], dec_n_points=points[1], dropout=dropout)
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


def main():
    pkg = ref_shims.install()
    res = {}
    for tag, points in VARIANTS.items():
        sd = om.with_aliases(op.deterministic_state_dict(op.points_cfg(*points)))
        model = build_reference(pkg, points, 0.1)
        trainable = {n for n, p in model.named_parameters() if p.requires_grad}
        spec = [[k, list(v.shape), k in trainable] for k, v in model.state_dict().items()]
        res[f"{tag}.spec"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)

        model = build_reference(pkg, points, 0.0)
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
        print(f"{tag}: {len(spec)} state_dict entries, {len(names)} gradients", flush=True)

    np.savez_compressed(OUT, **res)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, {len(res)} arrays)")


if __name__ == "__main__":
    main()
