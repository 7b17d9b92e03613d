"""The fused optimizer steps (`FusedSGD`, `FusedAdam`, `FusedAdamW`) against torch.optim's multi-tensor (`foreach`) steps over
the real model's gradient-receiving parameters, and the `Trainer` iteration with each of them, graph path against eager path.

    python tools/bench_optim.py [--iters 50] [--batch 8] [--steps 20] [--rounds 3]

Optimizer step: one step over the 313 gradient-receiving tensors of the default model (37.06 M parameters) with fixed random
gradients, timed with CUDA events over `--iters` steps after 5 warm-up steps, alternating fused and torch for `--rounds` rounds;
the best round is reported.  torch's side is `torch.optim.SGD(momentum=0.9)` / `torch.optim.Adam` over the reference's two groups
(`foreach` is its default on CUDA); for `adamw` it is `torch.optim.AdamW`, whose decoupled decay is not the reference's AdamW
update but moves the same bytes.  Achieved bandwidth counts algorithmic bytes only: 20 B per parameter for SGD (read p, g, buf;
write p, buf) and 28 B for Adam / AdamW (read p, g, m, v; write p, m, v).

Trainer: ms per iteration at batch 8, 1280x384, as tools/bench_trainer.py measures it (synthetic device-resident batches, epochs
of `--steps` batches timed with the host clock up to a device synchronise, two warm-up epochs).  `eager` is the reference's loop
(MDB_NO_GRAPH) with the same fused optimizer.  Prints one JSON line with the GPU's name and power limit beside the numbers."""
import argparse
import gc
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

KINDS = ("sgd", "adam", "adamw")
BYTES_PER_PARAM = {"sgd": 20, "adam": 28, "adamw": 28}


def fused(kind, model, device_step=False, lr=2e-4, wd=1e-4):
    from monodetr_b200.optim import FusedAdam, FusedAdamW, FusedSGD
    if kind == "sgd":
        return FusedSGD(model, lr=lr, momentum=0.9, weight_decay=wd, device_step=device_step)
    return (FusedAdam if kind == "adam" else FusedAdamW)(model, lr=lr, weight_decay=wd, device_step=device_step)


def torch_optimizer(kind, names, params, lr=2e-4, wd=1e-4):
    groups = [{"params": [p for n, p in zip(names, params) if "bias" in n], "weight_decay": 0},
              {"params": [p for n, p in zip(names, params) if "bias" not in n], "weight_decay": wd}]
    if kind == "sgd":
        return torch.optim.SGD(groups, lr=lr, momentum=0.9)
    return (torch.optim.Adam if kind == "adam" else torch.optim.AdamW)(groups, lr=lr)


def time_steps(opt, iters):
    for _ in range(5):
        opt.step()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        opt.step()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def bench_step(kind, iters, rounds):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    model, _ = build_monodetr(DEFAULT_MODEL_CFG)
    model = model.cuda()
    opt = fused(kind, model)
    b = opt.bucket
    g = torch.Generator(device="cuda").manual_seed(1)
    grads = [torch.randn(p.shape, device="cuda", generator=g) * 1e-3 for p in b.params]
    for p, gr in zip(b.params, grads):
        p.grad = gr
    opt._grads_in_bucket()                       # the gradients now live in the flat bucket, as after bucket.all_reduce()
    for p, v in zip(b.params, b.views):
        p.grad = v
    ref_params = [p.detach().clone().requires_grad_() for p in b.params]
    for p, gr in zip(ref_params, grads):
        p.grad = gr
    ref = torch_optimizer(kind, b.names, ref_params)
    ms = {"fused": [], "torch": []}
    for _ in range(rounds):
        ms["fused"].append(time_steps(opt, iters))
        ms["torch"].append(time_steps(ref, iters))
    best = {k: min(v) for k, v in ms.items()}
    n = b.param_numel
    out = {"tensors": len(b.params), "params": n, "ms_per_step": {k: [round(x, 4) for x in v] for k, v in ms.items()},
           "ms_per_step_best": {k: round(v, 4) for k, v in best.items()},
           "algorithmic_GB_per_s": {k: round(BYTES_PER_PARAM[kind] * n / (v * 1e-3) / 1e9, 1) for k, v in best.items()},
           "speedup": round(best["torch"] / best["fused"], 2)}
    del model, opt, ref, ref_params, grads
    return out


def bench_trainer(kind, batch, steps, rounds):
    from bench_trainer import epoch_ms
    from bench_extras import CRIT_CFG, synthetic_targets
    from monodetr_b200 import build_monodetr
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import build_lr_scheduler
    from monodetr_b200.trainer import Trainer

    class _Logger:
        def info(self, msg):
            pass

    loader = []
    for i in range(steps):
        images, calibs, sizes = synthetic_batch(batch, seed=77 + i)
        targets = {k: v.cuda() for k, v in synthetic_targets(77 + i, batch).items()}
        targets["img_size"] = sizes.cuda()
        loader.append((images.cuda(), calibs.cuda(), targets, {}))
    trainers = {}
    for path in ("graph", "eager"):
        torch.manual_seed(0)
        model, _ = build_monodetr(DEFAULT_MODEL_CFG)
        model = model.cuda().train()
        crit = build_criterion(CRIT_CFG).cuda().train()
        opt = fused(kind, model, device_step=True)
        sched, warm = build_lr_scheduler({"warmup": True, "decay_rate": 0.1, "decay_list": [125, 165]}, opt, last_epoch=-1)
        cfg = {"max_epoch": 1, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": "unused"}
        if path == "eager":
            os.environ["MDB_NO_GRAPH"] = "1"
        try:
            trainers[path] = Trainer(cfg, model, opt, loader, None, sched, warm, _Logger(), crit, "bench")
        finally:
            os.environ.pop("MDB_NO_GRAPH", None)
        assert trainers[path].graph_path == (path == "graph")
    for tr in trainers.values():
        for _ in range(2):
            epoch_ms(tr, steps)
    ms = {name: [] for name in trainers}
    for _ in range(rounds):
        for name, tr in trainers.items():
            ms[name].append(epoch_ms(tr, steps))
    best = {k: min(v) for k, v in ms.items()}
    live = trainers["graph"].live_graphs
    del trainers, loader
    return {"ms_per_iteration": {k: [round(x, 2) for x in v] for k, v in ms.items()},
            "ms_per_iteration_best": {k: round(v, 2) for k, v in best.items()},
            "images_per_sec_best": {k: round(batch / (v * 1e-3), 1) for k, v in best.items()}, "live_graphs": live}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--kinds", default=",".join(KINDS))
    ap.add_argument("--no-trainer", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim: a CUDA device is required (nothing is measured without one)")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True).stdout.strip()
    result = {"gpu": gpu, "optimizer_step": {}, "trainer": {}, "batch": args.batch, "resolution": "1280x384"}
    for kind in args.kinds.split(","):
        result["optimizer_step"][kind] = bench_step(kind, args.iters, args.rounds)
        gc.collect()
        torch.cuda.empty_cache()
        if not args.no_trainer:
            result["trainer"][kind] = bench_trainer(kind, args.batch, args.steps, args.rounds)
            gc.collect()
            torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
