"""GPU benchmark of the ResNeXt / wide-ResNet backbones (cfg `backbone`), printed as JSON lines:

  conv   the grouped 3x3 of each resnext50_32x4d stage (32 groups; C = 128 / 256 / 512 / 1024 at 96 x 320 / 48 x 160 /
         24 x 80 / 12 x 40, batch 8: the stride-1 blocks of a 1280 x 384 batch) on the channel-banded kernels, against the
         same convolution as a dense block-diagonal weight on the dense kernels, alternating the two in one session: forward,
         data gradient with a ReLU mask, weight gradient (+ the grouped unpack).
  step   the graph-captured training step of tools/bench_backbones.py (batch 8, 1280 x 384) in images/s for resnet50,
         resnet101 and the five new backbones; ROUNDS rounds, the order reversed every other round.

    python tools/bench_grouped.py [--steps 20] [--rounds 2] [--skip-step]

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

from bench_backbones import B, time_step  # noqa: E402
from bench_gemm import card  # noqa: E402
from monodetr_b200 import tc  # noqa: E402

VARIANTS = [("resnet50", False), ("resnet101", False), ("resnext50_32x4d", False), ("resnext50_32x4d", True),
            ("resnext101_32x8d", False), ("resnext101_64x4d", False), ("wide_resnet50_2", False), ("wide_resnet101_2", False)]
STAGES = [("layer1", 128, 96, 320), ("layer2", 256, 48, 160), ("layer3", 512, 24, 80), ("layer4", 1024, 12, 40)]
GROUPS = 32


def stage_cases(dev, C, H, W):
    g = torch.Generator(device=dev).manual_seed(C)
    gc = C // GROUPS
    x = torch.randn(B, H, W, C, device=dev, generator=g)
    dy = torch.randn(B, H, W, C, device=dev, generator=g)
    mask = torch.randn(B, H, W, C, device=dev, generator=g)
    w = torch.randn(C, gc, 3, 3, device=dev, generator=g) / (9 * gc) ** 0.5
    dense = torch.zeros(C, C, 3, 3, device=dev)
    for q in range(GROUPS):
        dense[q * gc:(q + 1) * gc, q * gc:(q + 1) * gc] = w[q * gc:(q + 1) * gc]
    gw = tc.pack_grouped_multi([w], None, [GROUPS])[0]
    sw = tc.split_weights([dense])[0]
    return [("fwd banded", lambda: tc.conv2d_forward(x, gw, None, None, 3, 3, 1, 1, groups=GROUPS)),
            ("fwd dense", lambda: tc.conv2d_forward(x, sw, None, None, 3, 3, 1, 1)),
            ("dgrad+mask banded", lambda: tc.conv2d_dgrad(dy, gw, x.shape, None, mask, 3, 3, 1, 1, groups=GROUPS)),
            ("dgrad+mask dense", lambda: tc.conv2d_dgrad(dy, sw, x.shape, None, mask, 3, 3, 1, 1)),
            ("wgrad banded", lambda: tc.unpack_grouped_wgrads_multi([tc.conv2d_wgrad(dy, x, None, 3, 3, 1, 1, groups=GROUPS)],
                                                                    [GROUPS])),
            ("wgrad dense", lambda: tc.unpack_wgrad(tc.conv2d_wgrad(dy, x, None, 3, 3, 1, 1), 3, 3))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_grouped needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tc.set_precision("bf16x3")
    print(json.dumps({"card": card(), "precision": tc.get_precision()}), flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    for stage, C, H, W in STAGES:
        cases = stage_cases(dev, C, H, W)
        for _, fn in cases:
            for _ in range(3):
                fn()
        torch.cuda.synchronize()
        times = {name: [] for name, _ in cases}
        n = 10
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
            print(json.dumps({"conv": f"{stage} grouped 3x3 C={C} g={GROUPS} B={B} {H}x{W} bf16x3 {name}",
                              "median_us": round(statistics.median(times[name]), 2), "min_us": round(min(times[name]), 2),
                              "max_us": round(max(times[name]), 2)}), flush=True)
        del cases
        torch.cuda.empty_cache()

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
