"""Time the device photometric distortion: ImageBatchPreprocessor with distort= (distortion + warp, 2 launches) against the warp
alone (1 launch), on batches of 8 and 16 KITTI-sized ragged images (1242x375, 1224x370, 1238x374, 1241x376, repeated) already
on the device, output 1280x384.

    python tools/bench_photometric.py [--iters 200] [--warmup 20]

Prints one JSON line: per batch size, the mean ms per call of each variant by CUDA events around `iters` back-to-back calls (host
packing, one metadata upload and the launches included), their difference, and the distortion kernel alone (pre.distort; its
per-call upload included) -- plus the device time of each kernel (torch.profiler, mean over `iters` calls), the GPU name and
power limit.  The per-call times include the host work of a call (record packing, pinned upload, allocation); the kernel times do
not."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from monodetr_b200.preprocess import ImageBatchPreprocessor, PhotometricDistort, get_affine_transform  # noqa: E402
from oracle.preprocess import synthetic_images  # noqa: E402

SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376)]


def _power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _time(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def _kernel_us(fn, iters):
    """Mean device time per call of each library kernel that `fn` launches, in microseconds (torch.profiler, CUDA activity)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for name in ("photometric_distort_kernel", "warp_affine_normalize_kernel"):
            if name in e.key:
                out[name] = round(e.device_time_total / iters, 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_photometric: a CUDA device is required")
    base = [torch.from_numpy(im).cuda() for im in synthetic_images(0, SIZES)]
    pre = ImageBatchPreprocessor(resolution=(1280, 384))
    np.random.seed(0)
    pd = PhotometricDistort()
    result = {"gpu": torch.cuda.get_device_name(0), "power_limit": _power_limit(), "iters": args.iters}
    for B in (8, 16):
        imgs = [base[i % len(base)] for i in range(B)]
        recs = [pd.sample() for _ in range(B)]
        tinv = np.stack([get_affine_transform(np.array(im.shape[1::-1]) / 2, np.array(im.shape[1::-1], np.float64), 0,
                                              np.array([1280, 384]), inv=1)[1] for im in imgs])
        flip = [bool(i % 2) for i in range(B)]
        warp = _time(lambda: pre(imgs, tinv, flip), args.iters, args.warmup)
        both = _time(lambda: pre(imgs, tinv, flip, distort=recs), args.iters, args.warmup)
        alone = _time(lambda: pre.distort(imgs, recs), args.iters, args.warmup)
        result[f"B{B}"] = {"warp_ms": round(warp, 4), "distort_warp_ms": round(both, 4), "added_ms": round(both - warp, 4),
                           "distort_only_ms": round(alone, 4),
                           "kernel_us": _kernel_us(lambda: pre(imgs, tinv, flip, distort=recs), args.iters)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()
