"""Time the device KITTI evaluation (Car, Pedestrian, Cyclist together) on a KITTI-val-sized synthetic set.

    python tools/bench_kitti_eval.py [--images 3769] [--dets 50] [--iters 10] [--reference]

Reports, as one JSON line: host packing (monodetr_b200.kitti_eval.pack) in ms, and the device pipeline (upload, 6 launches,
download: kitti_eval.eval_counts) in ms, by CUDA events after one warm-up, plus the GPU name and power limit.  The reference
path (numba) is timed only with --reference, on a machine that has numba with a CUDA target and the reference checkout."""
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

from monodetr_b200 import kitti_eval as ke  # noqa: E402


def synthetic(n_img, max_dets, seed=0):
    """KITTI-like annotations: up to 12 labelled objects and up to `max_dets` detections per image, detections jittered from
    the labels, values rounded to 2 decimals as in the label and result files."""
    rng = np.random.default_rng(seed)
    names = np.array(["Car", "Car", "Car", "Pedestrian", "Cyclist", "Van", "DontCare"])

    def boxes(n, pick):
        x0, y0 = rng.uniform(0, 1100, n), rng.uniform(100, 250, n)
        return {"name": rng.choice(pick, n), "truncated": np.round(rng.uniform(0, 0.6, n), 2), "occluded": rng.integers(0, 4, n),
                "alpha": np.round(rng.uniform(-np.pi, np.pi, n), 2),
                "bbox": np.round(np.stack([x0, y0, x0 + rng.uniform(10, 300, n), y0 + rng.uniform(15, 200, n)], 1), 2),
                "dimensions": np.round(np.stack([rng.uniform(3, 5, n), rng.uniform(1.2, 2, n), rng.uniform(1.4, 2, n)], 1), 2),
                "location": np.round(np.stack([rng.uniform(-15, 15, n), rng.uniform(1, 2, n), rng.uniform(5, 60, n)], 1), 2),
                "rotation_y": np.round(rng.uniform(-np.pi, np.pi, n), 2), "score": np.round(rng.uniform(0, 1, n), 2)}
    gts, dts = [], []
    for _ in range(n_img):
        g, d = boxes(int(rng.integers(0, 13)), names), boxes(int(rng.integers(0, max_dets + 1)), names[:5])
        k = min(len(g["name"]), len(d["name"]))
        for key in ("bbox", "dimensions", "location", "rotation_y"):
            d[key][:k] = np.round(g[key][:k] + rng.normal(0, 0.05, g[key][:k].shape), 2)
        gts.append(g)
        dts.append(d)
    return gts, dts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--dets", type=int, default=50)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--reference", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_eval: needs a CUDA device")
    gt, dt = synthetic(a.images, a.dets)
    mo = ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]]
    t0 = time.perf_counter()
    for _ in range(a.iters):
        ke.pack(gt, dt)
    pack_ms = (time.perf_counter() - t0) * 1e3 / a.iters
    table = ke.eval_counts(gt, dt, [0, 1, 2], mo, True)                          # warm-up
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        ke.eval_counts(gt, dt, [0, 1, 2], mo, True)
    e1.record()
    torch.cuda.synchronize()
    out = {"images": a.images, "gt": sum(len(g["name"]) for g in gt), "detections": sum(len(d["name"]) for d in dt),
           "host_pack_ms": round(pack_ms, 2), "device_eval_ms_incl_pack": round(e0.elapsed_time(e1) / a.iters, 2),
           "max_thresholds": int(table[:, 0].max()), "gpu": torch.cuda.get_device_name()}
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out["power_limit"] = "unknown"
    if a.reference:
        os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "0")              # numba's real CUDA target, not its simulator
        sys.path.insert(0, os.path.join(ROOT, "tools"))
        from gen_golden_kitti_eval import reference
        ev, _ = reference()
        t0 = time.perf_counter()
        for c in range(3):
            ev.get_official_eval_result(gt, dt, c)
        out["reference_s"] = round(time.perf_counter() - t0, 2)
    else:
        out["reference_s"] = "not measured"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
