"""Golden vectors of the reference model at its other transformer sizes, and of the reference criterion at 6 decoder layers and
up to 300 queries per group, so that the oracle and the product can be checked against the UNMODIFIED reference without it
present.  Needs the reference source tree (MONODETR_REFERENCE, see ref_shims):

    python tools/gen_golden_sizes.py   -> tests/golden/sizes.npz, tests/golden/criterion_sizes.npz

sizes.npz: for each variant of tests/oracle_sizes.VARIANTS (the configs/monodetr.yaml model section with the variant's keys),
keys prefixed "<tag>." as tools/gen_golden_points.py stores them:
  spec            names (state_dict order), shapes and trainable flags of the reference's build_monodetr(cfg)
  fwd_eval_*      eval-mode outputs (aux included where aux_loss is on) at 1 x 3 x 192 x 640
  fwd_train_*     train-mode outputs (dropout off) at 1 x 3 x 96 x 320
  grad_names / grad_max / grad_val / grad_len   sampled gradients of the surrogate loss of that train forward
all on the weights of tests/oracle_sizes.deterministic_state_dict(cfg).  The train keys exist only for the variants with 50
queries: the reference's training forward hard-codes 50 queries per group (depthaware_transformer.py:481-482) and fails at
any other count (see tests/oracle_sizes.py).

criterion_sizes.npz: for each case of tests/oracle_sizes.CRITERION_CASES, the reference HungarianMatcher (scipy) + SetCriterion
on tests/oracle_sizes.criterion_case(name), keyed as tools/gen_golden_criterion.py keys criterion.npz, except that a gradient of
more than GRAD_SAMPLES elements is kept at GRAD_SAMPLES seeded positions (oracle/criterion.golden_grad reads either form).
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
import oracle_sizes as osz  # noqa: E402
from oracle import criterion as oc  # noqa: E402
from oracle import monodetr_torch as om  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(ROOT), "tests", "golden")
GRAD_SAMPLES = 1024             # per criterion gradient tensor: 6 layers x 5 heads x 4 cases stay small


def store_grad(res, key, g):
    """oracle/criterion.store_golden_grad's format with GRAD_SAMPLES positions (int32) instead of its 16384."""
    if g.size <= GRAD_SAMPLES:
        res[key] = g
        return
    rng = np.random.default_rng(sum(key.encode()))
    idx = np.sort(rng.choice(g.size, GRAD_SAMPLES, replace=False)).astype(np.int32)
    res[key + ".idx"] = idx
    res[key + ".val"] = g.reshape(-1)[idx].astype(np.float32)
    res[key + ".absmax"] = np.asarray(np.abs(g).max(), np.float64)


def build_reference(pkg, tag, dropout):
    cfg = ref_shims.load_cfg()["model"]
    cfg.update(osz.VARIANTS[tag], dropout=dropout)
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


def model_goldens(pkg):
    res = {}
    for tag in osz.VARIANTS:
        sd = om.with_aliases(osz.deterministic_state_dict(osz.sizes_cfg(tag)))
        model = build_reference(pkg, tag, 0.1)
        trainable = {n for n, p in model.named_parameters() if p.requires_grad}
        spec = [[k, list(v.shape), k in trainable] for k, v in model.state_dict().items()]
        res[f"{tag}.spec"] = np.frombuffer(json.dumps(spec).encode(), dtype=np.uint8)

        model = build_reference(pkg, tag, 0.0)
        model.load_state_dict(sd)
        model.eval()
        images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
        with torch.no_grad():
            store_outputs(res, f"{tag}.fwd_eval", model(images, calibs, None, sizes))

        if osz.sizes_cfg(tag)["num_queries"] != 50:
            print(f"{tag}: {len(spec)} state_dict entries, eval only", flush=True)
            continue
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
    return res


def criterion_goldens():
    # loss_angles / loss_depth_map hard-code the device (monodetr.py:443,462): keep them on the CPU, as gen_golden_criterion does
    torch.Tensor.cuda = lambda self, *a, **k: self
    _tensor = torch.tensor
    torch.tensor = lambda *a, **k: _tensor(*a, **{kk: vv for kk, vv in k.items() if kk != "device"})
    from lib.models.monodetr.matcher import HungarianMatcher
    from lib.models.monodetr.monodetr import SetCriterion
    matcher = HungarianMatcher(cost_class=2, cost_bbox=5, cost_giou=2, cost_3dcenter=10)
    losses = ["labels", "boxes", "cardinality", "depths", "dims", "angles", "center", "depth_map"]
    res = {}
    for name, (seed, counts, nq, group, L) in osz.CRITERION_CASES.items():
        crit = SetCriterion(3, matcher=matcher, weight_dict=oc.weight_dict(L), focal_alpha=0.25, losses=losses, group_num=group)
        o, padded = osz.criterion_case(name)
        layers = [o] + o.get("aux_outputs", [])
        leaves = []
        for li, d in enumerate(layers):
            for k in list(d):
                if torch.is_tensor(d[k]):
                    d[k] = d[k].clone().requires_grad_(True)
                    leaves.append(("main" if li == 0 else f"aux{li - 1}", k, d[k]))
        targets = oc.prepare_targets(padded)
        crit.train(group > 1)
        ld = crit(o, targets)
        total = sum(ld[k] * crit.weight_dict[k] for k in ld if k in crit.weight_dict)
        total.backward()
        for k, v in ld.items():
            res[f"{name}.loss.{k}"] = np.asarray(float(v), np.float64)
        res[f"{name}.total"] = np.asarray(float(total), np.float64)
        for layer, k, t in leaves:
            g = t.grad.numpy() if t.grad is not None else np.zeros(t.shape, np.float32)
            store_grad(res, f"{name}.grad.{layer}.{k}", g)
        for l, od in enumerate(layers):
            ind = matcher({k: v.detach() for k, v in od.items() if k != "aux_outputs"}, targets, group_num=group)
            for b, (i, j) in enumerate(ind):
                res[f"{name}.match.{l}.{b}.src"] = i.numpy()
                res[f"{name}.match.{l}.{b}.tgt"] = j.numpy()
        print(f"{name}: total {float(total):.6f}", flush=True)
    return res


def main():
    pkg = ref_shims.install()
    only = sys.argv[1:] or ["model", "criterion"]
    if "model" in only:
        res = model_goldens(pkg)
        out = os.path.join(GOLDEN, "sizes.npz")
        np.savez_compressed(out, **res)
        print(f"wrote {out} ({os.path.getsize(out)} bytes, {len(res)} arrays)")
    if "criterion" in only:
        res = criterion_goldens()
        out = os.path.join(GOLDEN, "criterion_sizes.npz")
        np.savez_compressed(out, **res)
        print(f"wrote {out} ({os.path.getsize(out)} bytes, {len(res)} arrays)")


if __name__ == "__main__":
    main()
