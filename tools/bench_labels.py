"""Time the device target encoder (monodetr_b200.labels.TargetEncoder: record packing, one pinned upload, one launch) at B = 8 and
16 on a synthetic KITTI-like label bank, and the same batches on the CPU through the numpy restatement (oracle/labels.py, a stand-in
for the reference's per-object Python loop, which is not available where this runs; labelled as a CPU time).

    python tools/bench_labels.py [--iters 200] [--warmup 20] [--images 3712]

Line counts per image follow KITTI train (mean about 7.6 lines incl. DontCare, a few images above 20); each batch draws random
images and augmentation records (flip 0.5, crop 0.5) with the shipped config's writelist ['Car'].  Prints one JSON line per batch
size with the card's name and power limit.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def kitti_like_bank(n_img, seed=0):
    from oracle import labels as ol
    g = np.random.default_rng(seed)
    counts = np.minimum(g.poisson(6.6, n_img) + (g.random(n_img) < 0.1) * g.integers(5, 20, n_img), 60)
    M = int(counts.sum())
    recs = np.zeros((M, ol.WIDTH))
    recs[:, ol.CLS] = g.choice([1, 1, 1, 1, 0, 2, -1, -1], M)
    recs[:, ol.TRUNC] = g.choice([0, 0, 0, 0.1, 0.3, 0.6], M)
    recs[:, ol.OCC] = g.integers(0, 3, M)
    z = g.uniform(3, 70, M)
    x = g.uniform(-0.4, 0.4, M) * z
    u = 721.5 * x / z + 609.6
    v = 721.5 * 1.65 / z + 172.9
    hw = 721.5 * 1.6 / z
    recs[:, ol.X1:ol.Y2 + 1] = np.stack([u - hw, v - 1.2 * hw, u + hw, v + 0.2 * hw], 1).astype(np.float32)
    recs[:, ol.H:ol.L + 1] = np.round(np.array([1.53, 1.63, 3.88]) * g.uniform(0.85, 1.15, (M, 3)), 2)
    recs[:, ol.PX:ol.PZ + 1] = np.stack([x, np.full(M, 1.65), z], 1).astype(np.float32)
    recs[:, ol.RY] = np.round(g.uniform(-np.pi, np.pi, M), 2)
    P2 = np.tile(np.array([[721.5377, 0, 609.5593, 44.85728], [0, 721.5377, 172.854, 0.2163791], [0, 0, 1, 0.002745884]],
                          np.float32), (n_img, 1, 1))
    return counts, recs, P2


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--images", type=int, default=3712)
    ap.add_argument("--cpu-iters", type=int, default=20)
    a = ap.parse_args()
    import torch
    from monodetr_b200 import labels as lb
    from oracle import labels as ol
    if not torch.cuda.is_available():
        raise SystemExit("bench_labels: no CUDA device")
    counts, recs, P2 = kitti_like_bank(a.images)
    bank = lb.LabelBank.from_arrays(counts, recs, P2)
    enc = lb.TargetEncoder(["Car"])
    sampler = lb.AugmentationSampler("train", aug_pd=False, aug_crop=True, random_crop=0.5, scale=0.05, shift=0.05,
                                     rs=np.random.RandomState(0))
    sizes = [(1242, 375), (1224, 370), (1238, 374), (1241, 376)]
    g = np.random.default_rng(1)
    card = gpu_info()
    for B in (8, 16):
        batches = []
        for _ in range(8):
            idx = g.integers(0, a.images, B).tolist()
            batches.append((idx, [sampler.sample(sizes[i % 4]) for i in range(B)]))
        for i in range(a.warmup):
            enc(bank, *batches[i % 8])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(a.iters):
            enc(bank, *batches[i % 8])
        e1.record()
        torch.cuda.synchronize()
        gpu_ms = e0.elapsed_time(e1) / a.iters
        t0 = time.perf_counter()
        for i in range(a.cpu_iters):
            idx, rb = batches[i % 8]
            ol.encode_batch(bank.host_offsets, bank.host_objects, P2, idx, [r.img_size for r in rb], [r.flip for r in rb],
                            [r.crop_scale for r in rb], [r.trans for r in rb], class_mask=2)
        cpu_ms = (time.perf_counter() - t0) * 1e3 / a.cpu_iters
        lines = float(np.mean([sum(min(int(counts[k]), 50) for k in idx) for idx, _ in batches]))
        print(json.dumps({"bench": "labels", "B": B, "lines_per_batch": lines, "encoder_ms_per_batch": round(gpu_ms, 4),
                          "cpu_numpy_restatement_ms_per_batch": round(cpu_ms, 3), "iters": a.iters, "gpu": card,
                          "note": "encoder time = host packing + pinned upload + launch, CUDA events; CPU arm = oracle/labels.py"}))


if __name__ == "__main__":
    main()
