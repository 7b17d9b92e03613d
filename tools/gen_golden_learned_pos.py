"""Golden vectors of the reference's learned position embedding (`position_embedding: 'learned'`), so that the oracle and the
product model can be checked against the UNMODIFIED reference without it present.  Needs the reference source tree
(MONODETR_REFERENCE, see ref_shims):

    python tools/gen_golden_learned_pos.py   -> tests/golden/learned_pos.npz

Keys:
  learned.spec, dc5.spec    names (state_dict order), shapes and trainable flags of build_monodetr(cfg) with the learned
                            embedding, resnet50 and resnet50 + DC5
  mod.<h>x<w>.x_sha / y_sha the module alone on the seeded tables of oracle_learned_pos.module_tables(), at an h x w map: the
                            SHA-256 (oracle_learned_pos.digest) of x_emb (w, 128) and y_emb (h, 128).  The (1, 256, h, w)
                            output is exactly cat(x_emb[x], y_emb[y]) at every (y, x), which this script asserts, so the two
                            digests pin the whole table bit for bit
  mod.<h>x<w>.dcol.* / drow.*   both tables' gradients for oracle_learned_pos.upstream_grad(h, w): max|grad| (`max`) and the
                            values (`val`) at oracle_learned_pos.grad_sample_index positions (`idx`)
  fwd_eval_*                model eval outputs (aux included) at 1 x 3 x 192 x 640, FWD_SAMPLES seeded elements per tensor
  b1.* / b2.*               train outputs (dropout off) at 96 x 320 for batch 1 / 2 and, for the surrogate loss, every gradient
                            as tools/gen_golden_dab.py stores it; b2 also the whole gradients of both tables in grad_full.<name>
Model weights: tests/oracle_learned_pos.with_tables(om.deterministic_state_dict()).
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
from gen_golden_backbones import grad_index  # noqa: E402
import oracle_learned_pos as ol  # noqa: E402
from oracle import monodetr_torch as om  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "learned_pos.npz")
FWD_SAMPLES = 512              # per output tensor (read back with gen_golden_reference_pins.sampled_forward)


def store_outputs(res, prefix, out):
    """gen_golden_backbones.store_outputs with FWD_SAMPLES seeded positions per output tensor."""
    items = [(f"{prefix}_{k}", v) for k, v in out.items() if k != "aux_outputs"]
    items += [(f"{prefix}_aux{i}_{k}", v) for i, aux in enumerate(out.get("aux_outputs", [])) for k, v in aux.items()]
    for key, v in items:
        a = v.detach().numpy()
        if a.size <= FWD_SAMPLES:
            res[key] = a
            continue
        idx = np.sort(np.random.default_rng(sum(key.encode())).choice(a.size, FWD_SAMPLES, replace=False)).astype(np.int32)
        res[key + ".idx"] = idx
        res[key + ".val"] = a.reshape(-1)[idx]


def build_reference(pkg, dropout, dilation=False):
    cfg = ref_shims.load_cfg()["model"]
    cfg.update(position_embedding="learned", dropout=dropout, dilation=dilation)
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


class _Maps:
    """The NestedTensor fields PositionEmbeddingLearned.forward reads (it ignores the mask)."""

    def __init__(self, x):
        self.tensors, self.mask = x, None


def module_alone(res):
    from lib.models.monodetr.position_encoding import PositionEmbeddingLearned
    m = PositionEmbeddingLearned(128)
    col, row = ol.module_tables()
    with torch.no_grad():
        m.col_embed.weight.copy_(col)
        m.row_embed.weight.copy_(row)
    for h, w in ol.SHAPES:
        m.zero_grad(set_to_none=True)
        pos = m(_Maps(torch.zeros(1, 8, h, w)))
        x_emb, y_emb = pos[0, :128, 0, :].T.contiguous(), pos[0, 128:, :, 0].T.contiguous()
        assert torch.equal(pos[0], torch.cat([x_emb.unsqueeze(0).expand(h, -1, -1), y_emb.unsqueeze(1).expand(-1, w, -1)],
                                             -1).permute(2, 0, 1))
        pos.backward(ol.upstream_grad(h, w))
        tag = f"mod.{h}x{w}"
        res[tag + ".x_sha"] = ol.digest(x_emb)
        res[tag + ".y_sha"] = ol.digest(y_emb)
        for key, g in (("dcol", m.col_embed.weight.grad), ("drow", m.row_embed.weight.grad)):
            idx = ol.grad_sample_index(g, f"{tag}.{key}")
            res[f"{tag}.{key}.idx"] = idx
            res[f"{tag}.{key}.val"] = g.reshape(-1).numpy()[idx].copy()
            res[f"{tag}.{key}.max"] = np.float32(g.abs().max())


def main():
    pkg = ref_shims.install()
    res = {}
    res["learned.spec"], n = spec_of(build_reference(pkg, 0.1))
    res["dc5.spec"], n5 = spec_of(build_reference(pkg, 0.1, dilation=True))
    print(f"state_dict entries: resnet50 {n}, resnet50 + DC5 {n5}", flush=True)
    module_alone(res)

    sd = om.with_aliases(ol.with_tables(om.deterministic_state_dict()))
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
            if B == 2 and name in (ol.ROW, ol.COL):
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
