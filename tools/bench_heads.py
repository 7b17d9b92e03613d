"""GPU benchmark of the head counts (cfg `nheads` 4 / 8 / 16: attention head widths 64 / 32 / 16), printed as JSON lines:

  attn   the fused attention kernels, forward and backward (delta + dQ + dK/dV), at the model's three call shapes -- the
         depth encoder's self-attention (1920 x 1920), the depth cross-attention (550 x 1920), the group self-attention
         (88 x (50 x 50)) -- at batch 8, width 256, dropout 0.1, for head widths 16 / 32 / 64.  CUDA events over 20 calls,
         7 rounds with the widths alternating; median, min and max per call.
  step   the graph-captured training step (forward, surrogate loss of monodetr_b200.bench_model, backward) at batch 8,
         1280 x 384, in images/s, for nheads 4 / 8 / 16.  The variants run in turn, ROUNDS times (the order reversed every
         other round), each round timing STEPS replays per variant.

    python tools/bench_heads.py [--steps 20] [--rounds 2] [--skip-step]

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

from bench_backbones import time_step  # noqa: E402
from bench_gemm import card  # noqa: E402
import bench_backbones  # noqa: E402
from monodetr_b200 import kernels as K, tc  # noqa: E402

WIDTHS = (16, 32, 64)
SHAPES = [("depth-encoder self 1920x1920", 8, 1920, 1920), ("depth cross 550x1920", 8, 550, 1920), ("group self 88x50x50", 88, 50, 50)]
NHEADS = (4, 8, 16)


def attn_cases(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    cases = []
    for name, B, Lq, Lk in SHAPES:
        q, dout = (torch.randn(B, Lq, 256, device=dev, generator=g) for _ in range(2))
        k, v = (torch.randn(B, Lk, 256, device=dev, generator=g) for _ in range(2))
        for hd in WIDTHS:
            H = 256 // hd
            o, lse, _ = K.attention_forward(q, k, v, None, drop_p=0.1, site=1, heads=H)
            fwd = lambda q=q, k=k, v=v, H=H: K.attention_forward(q, k, v, None, drop_p=0.1, site=1, heads=H)
            bwd = lambda q=q, k=k, v=v, o=o, lse=lse, dout=dout, H=H: K.attention_backward(q, k, v, None, o, lse, dout, drop_p=0.1,
                                                                                         site=1, heads=H)
            cases.append((name, hd, "fwd", fwd))
            cases.append((name, hd, "bwd", bwd))
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_heads needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tc.set_precision("bf16x3")
    print(json.dumps({"card": card(), "precision": tc.get_precision()}), flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    # ---- attention kernels, widths alternating --------------------------------------------------------------------------
    cases = attn_cases(dev)
    for *_, fn in cases:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {c[:3]: [] for c in cases}
    n = 20
    for _ in range(7):
        for name, hd, d, fn in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[(name, hd, d)].append(e0.elapsed_time(e1) / n * 1e3)
    for (name, hd, d), t in times.items():
        print(json.dumps({"attn": name, "B": 8, "head_dim": hd, "heads": 256 // hd, "dir": d, "dropout": 0.1,
                          "median_us": round(statistics.median(t), 1), "min_us": round(min(t), 1), "max_us": round(max(t), 1)}),
              flush=True)
    del cases
    torch.cuda.empty_cache()

    # ---- training step per head count -----------------------------------------------------------------------------------
    if args.skip_step:
        return
    base = bench_backbones.DEFAULT_MODEL_CFG
    res = {h: [] for h in NHEADS}
    try:
        for r in range(args.rounds):
            for h in (NHEADS if r % 2 == 0 else NHEADS[::-1]):
                bench_backbones.DEFAULT_MODEL_CFG = dict(base, nheads=h)       # time_step builds from this dict
                ips, med = time_step("resnet50", False, args.steps, dev, flush)
                res[h].append(ips)
                print(json.dumps({"round": r, "nheads": h, "img_s": round(ips, 2), "median_step_ms": round(med, 2)}), flush=True)
    finally:
        bench_backbones.DEFAULT_MODEL_CFG = base
    for h in NHEADS:
        print(json.dumps({"step": "train B=8 1280x384 graph", "nheads": h, "img_s_per_round": [round(x, 2) for x in res[h]]}),
              flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
