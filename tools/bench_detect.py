"""What the Detector's CUDA graph buys: images/s of `Detector.detect_device` replaying its graph against the same Detector with
the graphs off (the eager chain: the same staging, pre-process, forward, extract and decode, launched one by one), on one GPU.

    python tools/bench_detect.py [--batches 1,8,32] [--iters 20] [--rounds 5] [--out FILE]

The model is configs/monodetr.yaml's (ResNet-50, seeded random weights, eval mode) at 1280 x 384; the frames are KITTI-sized
(1242 x 375, 1224 x 370, 1238 x 374, 1241 x 376, in turn) uint8 RGB tensors already on the device, as an ImageBank holds them.
Per batch size both paths are warmed up (the graph path captures), then `rounds` rounds alternate the two paths; a round times
`iters` calls back to back with the host clock, ending in a synchronise.  The JSON line gives the median, min and max images/s
over the rounds, whether the two paths returned the same bits, and the GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

KITTI_SIZES = ((1242, 375), (1224, 370), (1238, 374), (1241, 376))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_detect: a CUDA device is required")
    from monodetr_b200 import build_monodetr, tc
    from monodetr_b200.detect import Detector
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from oracle.preprocess import synthetic_images
    from synthetic_kitti import p2_of

    tc.set_precision(os.environ.get("MDB_PRECISION", "bf16x3"))
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG))
    model = model.cuda().eval()
    batches = [int(b) for b in args.batches.split(",")]
    n = max(batches)
    frames = [torch.from_numpy(im).cuda() for im in synthetic_images(7, [KITTI_SIZES[i % 4] for i in range(n)])]
    P2 = np.stack([p2_of(i % 2) for i in range(n)])
    result = {"gpu": gpu_info(), "resolution": [1280, 384], "iters": args.iters, "rounds": args.rounds, "batches": {}}
    for B in batches:
        graph = Detector(model, max_batch=B)
        eager = Detector(model, max_batch=B)
        eager.use_graphs = False
        f, p = frames[:B], P2[:B]
        outs = {}
        for name, det in (("graph", graph), ("eager", eager)):
            for _ in range(3):                                       # eager, capture + replay, replay
                outs[name] = det.detect_device(f, p)
        torch.cuda.synchronize()
        assert graph.live_graphs == 1 and eager.live_graphs == 0
        same = bool(torch.equal(outs["graph"][0], outs["eager"][0]) and torch.equal(outs["graph"][1], outs["eager"][1]))
        rates = {"graph": [], "eager": []}
        for _ in range(args.rounds):
            for name, det in (("graph", graph), ("eager", eager)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.iters):
                    det.detect_device(f, p)
                torch.cuda.synchronize()
                rates[name].append(B * args.iters / (time.perf_counter() - t0))
        result["batches"][str(B)] = {
            **{f"{k}_images_per_s": {"median": float(np.median(v)), "min": float(min(v)), "max": float(max(v))}
               for k, v in rates.items()},
            "speedup_median": float(np.median(rates["graph"]) / np.median(rates["eager"])),
            "same_bits": same}
        del graph, eager
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
