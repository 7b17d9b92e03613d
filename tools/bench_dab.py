"""GPU benchmark of the anchor-box query branch (`use_dab: True`) against the default branch, printed as JSON lines:

  step   the graph-captured training step (forward, surrogate loss of monodetr_b200.bench_model, backward) at batch 8,
         1280 x 384, in images/s
  eval   the eval forward at batch 32, 1280 x 384, in images/s
The two branches alternate within one session, ROUNDS times (the order reversed every other round), each round timing STEPS
replays / forwards per branch; the SM clock is sampled after every round.

    python tools/bench_dab.py [--steps 20] [--rounds 3]

The card's name and power limit are read in the same run (nvidia-smi) and printed first.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_gemm import card, sm_mhz  # noqa: E402
from monodetr_b200 import build_monodetr, tc  # noqa: E402
from monodetr_b200.bench_model import surrogate_loss, synthetic_batch  # noqa: E402
from monodetr_b200.ddp import FlatGradBucket  # noqa: E402
from monodetr_b200.monodetr import DEFAULT_MODEL_CFG  # noqa: E402

BRANCHES = (False, True)          # use_dab


def _model(use_dab, dev):
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, use_dab=use_dab))
    return model.to(dev)


def time_step(use_dab, steps, dev, flush, B=8):
    """Images/s of `steps` replays of the captured training step (256 MiB L2 flush before each, untimed)."""
    model = _model(use_dab, dev).train()
    bucket = FlatGradBucket(model)
    images, calibs, sizes = (t.to(dev) for t in synthetic_batch(B, seed=1000))

    def fwd_bwd():
        bucket.zero()
        surrogate_loss(model(images, calibs, None, sizes)).backward()

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fwd_bwd()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fwd_bwd()
    bucket.freeze_sources()
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    ms = []
    for _ in range(steps):
        flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    del graph, model, bucket
    torch.cuda.empty_cache()
    return B * steps / (sum(ms) * 1e-3), statistics.median(ms)


def time_eval(use_dab, steps, dev, flush, B=32):
    """Images/s of `steps` eager eval forwards (no_grad), each after an untimed L2 flush."""
    model = _model(use_dab, dev).eval()
    images, calibs, sizes = (t.to(dev) for t in synthetic_batch(B, seed=1001))
    with torch.no_grad():
        for _ in range(3):
            model(images, calibs, None, sizes)
        torch.cuda.synchronize()
        ms = []
        for _ in range(steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            model(images, calibs, None, sizes)
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
    del model
    torch.cuda.empty_cache()
    return B * steps / (sum(ms) * 1e-3), statistics.median(ms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dab needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tc.set_precision("bf16x3")
    print(json.dumps({"card": card(), "precision": tc.get_precision()}), flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    res = {(w, d): [] for w in ("step", "eval") for d in BRANCHES}
    for r in range(args.rounds):
        for d in (BRANCHES if r % 2 == 0 else BRANCHES[::-1]):
            for what, fn in (("step", time_step), ("eval", time_eval)):
                ips, med = fn(d, args.steps, dev, flush)
                res[(what, d)].append(ips)
                print(json.dumps({"round": r, "what": what, "use_dab": d, "img_s": round(ips, 2), "median_ms": round(med, 2)}),
                      flush=True)
        print(json.dumps({"round": r, "sm_mhz": sm_mhz()}), flush=True)
    for (what, d), v in res.items():
        print(json.dumps({"what": {"step": "train B=8 1280x384 graph", "eval": "eval B=32 1280x384"}[what], "use_dab": d,
                          "img_s_per_round": [round(x, 2) for x in v], "median": round(statistics.median(v), 2)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
