"""ms per iteration of `monodetr_b200.trainer.Trainer`: the graph path against the eager path (the reference's loop: per-image
`prepare_targets`, a Python sum over 26 loss terms and `.item()` on each of them every step), both with this package's model,
device criterion and `FusedAdamW`.  Batch 8 at 1280x384, synthetic batches already on the device, so the loader costs nothing and
the figure is the trainer's own: input copies into the static buffers, the replayed step, the loss log.

    python tools/bench_trainer.py [--batch 8] [--steps 20] [--rounds 3]

Each round times one epoch of `--steps` batches per path, alternating the paths; an epoch is timed with the host clock from its
first batch to a device synchronise after its last.  Epochs before the timed ones warm every shape and capture the graph.  Prints
one JSON line with the GPU's name and power limit beside the numbers."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class _Logger:
    def info(self, msg):
        pass


def build(batch, steps, graph):
    from bench_extras import CRIT_CFG, synthetic_targets
    from monodetr_b200 import build_monodetr
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW, build_lr_scheduler
    from monodetr_b200.trainer import Trainer
    torch.manual_seed(0)
    model, _ = build_monodetr(DEFAULT_MODEL_CFG)
    model = model.cuda().train()
    crit = build_criterion(CRIT_CFG).cuda().train()
    opt = FusedAdamW(model, lr=2e-4, weight_decay=1e-4, device_step=True)
    sched, warm = build_lr_scheduler({"warmup": True, "decay_rate": 0.1, "decay_list": [125, 165]}, opt, last_epoch=-1)
    loader = []
    for i in range(steps):
        images, calibs, sizes = synthetic_batch(batch, seed=77 + i)
        targets = {k: v.cuda() for k, v in synthetic_targets(77 + i, batch).items()}
        targets["img_size"] = sizes.cuda()
        loader.append((images.cuda(), calibs.cuda(), targets, {}))
    cfg = {"max_epoch": 1, "save_frequency": 1, "save_all": False, "use_dn": False, "save_path": "unused"}
    if not graph:
        os.environ["MDB_NO_GRAPH"] = "1"
    try:
        trainer = Trainer(cfg, model, opt, loader, None, sched, warm, _Logger(), crit, "bench")
    finally:
        os.environ.pop("MDB_NO_GRAPH", None)
    assert trainer.graph_path == graph
    return trainer


def epoch_ms(trainer, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
        trainer.train_one_epoch(0)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_trainer: a CUDA device is required (nothing is measured without one)")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                         capture_output=True, text=True).stdout.strip()
    trainers = {"graph": build(args.batch, args.steps, True), "eager": build(args.batch, args.steps, False)}
    for name, tr in trainers.items():
        for _ in range(2):
            epoch_ms(tr, args.steps)                      # warm every shape; the graph path captures in the first of these
    ms = {name: [] for name in trainers}
    for _ in range(args.rounds):
        for name, tr in trainers.items():
            ms[name].append(epoch_ms(tr, args.steps))
    best = {name: min(v) for name, v in ms.items()}
    print(json.dumps({"gpu": gpu, "batch": args.batch, "resolution": "1280x384", "steps_per_epoch": args.steps,
                      "ms_per_iteration": {k: [round(x, 2) for x in v] for k, v in ms.items()},
                      "ms_per_iteration_best": {k: round(v, 2) for k, v in best.items()},
                      "images_per_sec_best": {k: round(args.batch / (v * 1e-3), 1) for k, v in best.items()},
                      "live_graphs": trainers["graph"].live_graphs,
                      "note": "eager = the reference's loop (prepare_targets, Python loss sum, 26 x .item() per step) over the same "
                              "model, device criterion and FusedAdamW; batches are device-resident, the loader is not measured"}))


if __name__ == "__main__":
    main()
