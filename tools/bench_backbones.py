"""GPU benchmark of the backbone variants (cfg `backbone` / `dilation`), printed as JSON lines:

  step   the graph-captured training step (forward, surrogate loss of monodetr_b200.bench_model, backward) at batch 8,
         1280 x 384, in images/s, for resnet50, resnet50 + DC5, resnet101, resnet101 + DC5 and resnet152.  The variants run
         in turn, ROUNDS times (the order reversed every other round), each round timing STEPS replays per variant.
  conv   the dilated 3x3 512 -> 512 of the DC5 stage at batch 8, 24 x 80 (forward, data gradient with a ReLU mask, weight
         gradient) against the undilated convolution of the same shape, alternating the two in one session.

    python tools/bench_backbones.py [--steps 20] [--rounds 2] [--skip-step]

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

from bench_gemm import card  # noqa: E402
from monodetr_b200 import build_monodetr, tc  # noqa: E402
from monodetr_b200.bench_model import surrogate_loss, synthetic_batch  # noqa: E402
from monodetr_b200.ddp import FlatGradBucket  # noqa: E402
from monodetr_b200.monodetr import DEFAULT_MODEL_CFG  # noqa: E402

VARIANTS = [("resnet50", False), ("resnet50", True), ("resnet101", False), ("resnet101", True), ("resnet152", False)]
B = 8


def time_step(backbone, dilation, steps, dev, flush):
    """Images/s of `steps` replays of the captured training step (256 MiB L2 flush before each, untimed)."""
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, backbone=backbone, dilation=dilation))
    model = model.to(dev).train()
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


def conv_cases(dev):
    """(name, dilation, callable) for the 512 -> 512 3x3 at batch 8, 24 x 80: forward, dgrad + mask, wgrad."""
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(B, 24, 80, 512, device=dev, generator=g)
    dy = torch.randn(B, 24, 80, 512, device=dev, generator=g)
    mask = torch.randn(B, 24, 80, 512, device=dev, generator=g)
    w = torch.randn(512, 512, 3, 3, device=dev, generator=g) / 48.0
    sw = tc.split_weights([w])[0]
    out = []
    for d in (1, 2):
        out += [(f"fwd d{d}", lambda d=d: tc.conv2d_forward(x, sw, None, None, 3, 3, 1, d, dilation=d)),
                (f"dgrad+mask d{d}", lambda d=d: tc.conv2d_dgrad(dy, sw, x.shape, None, mask, 3, 3, 1, d, dilation=d)),
                (f"wgrad d{d}", lambda d=d: tc.conv2d_wgrad(dy, x, None, 3, 3, 1, d, dilation=d))]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_backbones needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tc.set_precision("bf16x3")
    print(json.dumps({"card": card(), "precision": tc.get_precision()}), flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    # ---- the dilated convolution against the undilated one, alternating ------------------------------------------------
    cases = conv_cases(dev)
    for _, fn in cases:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {name: [] for name, _ in cases}
    n = 20
    for _ in range(7):
        for name, fn in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / n * 1e3)
    for name in times:
        print(json.dumps({"conv": "3x3 512->512 B=8 24x80 bf16x3 " + name, "median_us": round(statistics.median(times[name]), 2),
                          "min_us": round(min(times[name]), 2), "max_us": round(max(times[name]), 2)}), flush=True)

    # ---- training step per variant ------------------------------------------------------------------------------------
    if args.skip_step:
        return
    res = {v: [] for v in VARIANTS}
    for r in range(args.rounds):
        for v in (VARIANTS if r % 2 == 0 else VARIANTS[::-1]):
            ips, med = time_step(*v, args.steps, dev, flush)
            res[v].append(ips)
            print(json.dumps({"round": r, "backbone": v[0], "dilation": v[1], "img_s": round(ips, 2),
                              "median_step_ms": round(med, 2)}), flush=True)
    for v in VARIANTS:
        print(json.dumps({"step": "train B=8 1280x384 graph", "backbone": v[0], "dilation": v[1],
                          "img_s_per_round": [round(x, 2) for x in res[v]]}), flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
