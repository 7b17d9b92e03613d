"""GPU benchmark of the learned position embedding (`position_embedding: 'learned'`) against the default sine embedding, printed
as JSON lines:

  step     the graph-captured training step (forward, surrogate loss of monodetr_b200.bench_model, backward) at batch 8,
           1280 x 384, in images/s
  eval     the eval forward at batch 32, 1280 x 384, in images/s
  kernels  CUDA-event times of mdb_pos_learned_forward_f32 / mdb_pos_learned_backward_f32 at the four level shapes of 1280 x 384
           (48 x 160, 24 x 80, 12 x 40, 6 x 20), averaged over KERNEL_ITERS back-to-back launches replayed as one CUDA graph
The two branches alternate within one session, ROUNDS times (the order reversed every other round), each round timing STEPS
replays / forwards per branch; the SM clock is sampled after every round.

    python tools/bench_learned_pos.py [--steps 20] [--rounds 3]

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

from bench_dab import time_eval as _time_eval, time_step as _time_step  # noqa: E402
import bench_dab  # noqa: E402
from bench_gemm import card, sm_mhz  # noqa: E402
from monodetr_b200 import _lib, build_monodetr, tc  # noqa: E402
from monodetr_b200.monodetr import DEFAULT_MODEL_CFG  # noqa: E402

BRANCHES = ("sine", "learned")
LEVELS = ((48, 160), (24, 80), (12, 40), (6, 20))
KERNEL_ITERS = 200


def _model(pos, dev):
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, position_embedding=pos))
    return model.to(dev)


def time_kernels(dev):
    """Microseconds per launch of the forward and the backward at each level shape."""
    g = torch.Generator(device=dev).manual_seed(0)
    col, row = (torch.randn(50, 128, device=dev, generator=g) for _ in range(2))
    dcol, drow = torch.empty_like(col), torch.empty_like(row)
    out = []
    for H, W in LEVELS:
        dpos = torch.randn(H * W, 256, device=dev, generator=g)
        pos = torch.empty(H * W, 256, device=dev)
        res = {}
        for what, run in (("fwd", lambda: _lib.call("mdb_pos_learned_forward_f32", col, row, H, W, pos)),
                          ("bwd", lambda: _lib.call("mdb_pos_learned_backward_f32", dpos, H, W, dcol, drow))):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(10):
                    run()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            # the launches are captured and replayed as one graph: timed one after another from Python, a launch costs more
            # host time than these kernels take
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                for _ in range(KERNEL_ITERS):
                    run()
            graph.replay()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graph.replay()
            e1.record()
            torch.cuda.synchronize()
            res[what] = e0.elapsed_time(e1) * 1e3 / KERNEL_ITERS
        out.append({"H": H, "W": W, "fwd_us": round(res["fwd"], 2), "bwd_us": round(res["bwd"], 2),
                    "table_MB": round(H * W * 256 * 4 / 1e6, 3)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_learned_pos needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tc.set_precision("bf16x3")
    bench_dab._model = _model                      # bench_dab's timers with this benchmark's branch switch
    print(json.dumps({"card": card(), "precision": tc.get_precision()}), flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    res = {(w, d): [] for w in ("step", "eval") for d in BRANCHES}
    for r in range(args.rounds):
        for d in (BRANCHES if r % 2 == 0 else BRANCHES[::-1]):
            for what, fn in (("step", _time_step), ("eval", _time_eval)):
                ips, med = fn(d, args.steps, dev, flush)
                res[(what, d)].append(ips)
                print(json.dumps({"round": r, "what": what, "position_embedding": d, "img_s": round(ips, 2),
                                  "median_ms": round(med, 2)}), flush=True)
        print(json.dumps({"round": r, "sm_mhz": sm_mhz()}), flush=True)
    for lv in time_kernels(dev):
        print(json.dumps(dict(lv, what="kernels")), flush=True)
    for (what, d), v in res.items():
        print(json.dumps({"what": {"step": "train B=8 1280x384 graph", "eval": "eval B=32 1280x384"}[what], "position_embedding": d,
                          "img_s_per_round": [round(x, 2) for x in v], "median": round(statistics.median(v), 2)}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
