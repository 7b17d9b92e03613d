"""Times the device criterion and the training step at the reference's other transformer sizes (tests/oracle_sizes.VARIANTS),
and the default configuration's step and matcher against another build of the library, alternated in one call.

    python tools/bench_sizes.py [--batch 8] [--steps 10] [--warmup 3] [--baseline-lib PATH] [--out FILE]

Per configuration (the default model section and each variant), at batch B and 1280 x 384:
  crit_fwd_ms / crit_bwd_ms   the criterion forward (prepare, match, depth map, losses) and backward, on the model's head shapes
                              (Q = num_queries x 11, one layer per decoder layer with aux_loss) and synthetic targets
  match_ms                    the matcher launch alone
  step_ms                     one eager training iteration: forward, criterion, backward, FusedAdamW step
--baseline-lib: the default configuration's step_ms and match_ms are measured by child processes that load this build and the
given one in turn (new, old, new, old, ...), so that both see the same machine state.  The card's name and power limit are read
in the same run and written beside the numbers.
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")
CONFIGS = {"default": {}, "deep": dict(enc_layers=6, dec_layers=6, dim_feedforward=1024),
           "q300": dict(num_queries=300, dim_feedforward=2048), "shallow": dict(enc_layers=1, dec_layers=1, aux_loss=False),
           "dab_q100": dict(use_dab=True, num_queries=100, dec_layers=4)}


def crit_cfg(model_kw):
    from bench_extras import CRIT_CFG
    return dict(CRIT_CFG, dec_layers=model_kw.get("dec_layers", 3), aux_loss=model_kw.get("aux_loss", True),
                num_queries=model_kw.get("num_queries", 50))


def make_iteration(dev, model_kw, B=2, seed=77, hw=None):
    """(bucket, it, snapshot) of one training iteration of the model at `model_kw`: forward with dropout, the device criterion,
    backward, FusedAdamW with the device step -- the iteration the Trainer replays."""
    from bench_extras import synthetic_targets
    from monodetr_b200 import build_monodetr
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, dropout=0.1, **model_kw))
    model = model.to(dev).train()
    crit = build_criterion(crit_cfg(model_kw)).to(dev).train()
    bucket = FlatGradBucket(model)
    opt = FusedAdamW(model, bucket, lr=2e-4, weight_decay=1e-4, device_step=True)
    images, calibs, sizes = synthetic_batch(B, seed=seed)
    if hw is not None:
        images = images[:, :, :hw[0], :hw[1]].contiguous()
    images, calibs, sizes = images.to(dev), calibs.to(dev), sizes.to(dev)
    tg = {k: v.to(dev) for k, v in synthetic_targets(seed, B).items()}
    state = {}

    def it():
        bucket.zero()
        out = model(images, calibs, None, sizes)
        losses = crit(out, tg)
        crit.weighted_sum().backward()
        opt.step()
        state["out"], state["losses"] = out, losses

    def snapshot():
        out = state["out"]
        flat = [out[k] for k in OUT_KEYS] + [v for a in out.get("aux_outputs", []) for _, v in sorted(a.items())]
        losses = [state["losses"][k] for k in sorted(state["losses"])]
        grads = [p.grad for p in model.parameters() if p.grad is not None]
        return [t.detach().clone() for t in flat], [t.detach().clone() for t in losses], [t.clone() for t in grads], \
            [p.detach().clone() for p in model.parameters()]
    return bucket, it, snapshot


def default_iteration_digests(dev):
    """SHA-256 of the outputs, losses, gradients and updated parameters of two reproducible-mode training iterations at the
    default configuration (bf16x3, batch 2, fixed seeds)."""
    import monodetr_b200
    from monodetr_b200 import kernels as K, tc
    prev, prev_prec = monodetr_b200.set_deterministic(True), tc.get_precision()
    tc.set_precision("bf16x3")
    try:
        _, it, snap = make_iteration(dev, {})
        K.reseed(dev, 4242)
        for _ in range(2):
            it()
        torch.cuda.synchronize()
        res = {}
        for name, ts in zip(("outputs", "losses", "gradients", "parameters"), snap()):
            h = hashlib.sha256()
            for t in ts:
                h.update(t.detach().contiguous().cpu().numpy().tobytes())
            res[name] = {"count": len(ts), "sha256": h.hexdigest()}
        return res
    finally:
        tc.set_precision(prev_prec)
        monodetr_b200.set_deterministic(prev)


def _events_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def time_criterion(dev, model_kw, B, steps, warmup):
    from bench_extras import synthetic_heads, synthetic_targets
    from monodetr_b200 import criterion as mc
    nq = model_kw.get("num_queries", 50)
    L = model_kw.get("dec_layers", 3) if model_kw.get("aux_loss", True) else 1
    heads = synthetic_heads(5, B, nq * 11, n_aux=L - 1)
    out = {k: (v.to(dev).requires_grad_(True) if torch.is_tensor(v) else v) for k, v in heads.items() if k != "aux_outputs"}
    out["aux_outputs"] = [{k: v.to(dev).requires_grad_(True) for k, v in a.items()} for a in heads.get("aux_outputs", [])]
    if L == 1:
        del out["aux_outputs"]
    crit = mc.build_criterion(crit_cfg(model_kw)).to(dev).train()
    tg = mc.pack_targets({k: v.to(dev) for k, v in synthetic_targets(9, B).items()}, dev)

    def fwd():
        crit(out, tg)
        return crit._last_losses

    def fwd_bwd():
        crit(out, tg)
        crit.weighted_sum().backward()

    st = mc._prepare(tg)
    layers = [out] + out.get("aux_outputs", [])

    def match():
        mc._match(crit.matcher, layers, tg, st, 11)
    with torch.no_grad():
        f = _events_ms(fwd, steps, warmup)
        m = _events_ms(match, steps, warmup)
    fb = _events_ms(fwd_bwd, steps, warmup)
    return {"crit_fwd_ms": round(f, 4), "crit_bwd_ms": round(fb - f, 4), "match_ms": round(m, 4), "layers": L, "queries": nq * 11}


def time_step(dev, model_kw, B, steps, warmup):
    _, it, _ = make_iteration(dev, model_kw, B=B)
    return round(_events_ms(it, steps, warmup), 3)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def child(args):
    """One process on one library build: the default step and matcher times (or the reproducible-mode digests)."""
    from monodetr_b200 import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    dev = torch.device("cuda", 0)
    if args.child == "digests":
        print(json.dumps(default_iteration_digests(dev)))
        return
    c = time_criterion(dev, {}, args.batch, args.steps * 10, args.warmup)
    print(json.dumps({"lib": _lib.LIB_PATH, "step_ms": time_step(dev, {}, args.batch, args.steps, args.warmup), "match_ms": c["match_ms"]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--only", default=None, help="comma-separated subset of " + ",".join(CONFIGS))
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", default=None, choices=[None, "time", "digests"])
    ap.add_argument("--lib", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sizes: no CUDA device (timings are only taken on the GPU)")
    if args.child:
        return child(args)
    dev = torch.device("cuda", 0)
    res = {"card": card(), "batch": args.batch, "image": "1280x384", "step": "eager, dropout 0.1, FusedAdamW", "configs": {}}
    for name in (args.only.split(",") if args.only else CONFIGS):
        kw = CONFIGS[name]
        r = time_criterion(dev, kw, args.batch, args.steps * 10, args.warmup)
        r["step_ms"] = time_step(dev, kw, args.batch, args.steps, args.warmup)
        res["configs"][name] = r
        print(name, r, flush=True)
        torch.cuda.empty_cache()
    if args.baseline_lib:
        runs = {"new": [], "old": []}
        for _ in range(args.rounds):
            for tag, lib in (("new", None), ("old", args.baseline_lib)):
                cmd = [sys.executable, os.path.abspath(__file__), "--child", "time", "--batch", str(args.batch), "--steps", str(args.steps),
                       "--warmup", str(args.warmup)] + (["--lib", lib] if lib else [])
                out = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout.strip().splitlines()[-1]
                runs[tag].append(json.loads(out))
                print(tag, runs[tag][-1], flush=True)
        res["default_old_vs_new"] = runs
    res["card_after"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
