"""GPU benchmark of the sampling-point counts (cfg `enc_n_points` / `dec_n_points`), printed as JSON lines:

  msda   the deformable-attention core at P = 2 / 4 / 8 points per level, fused (mdb_msda_fused_*: the pre-processing inside the
         sampling kernels) against two-step (mdb_msda_prep_* + mdb_msda_forward/backward_f32), forward and backward, at the
         encoder's call (B = 8, Lq = 10200 pixel queries, 2-d reference points) and the decoder's (B = 8, Lq = 550 queries, 6-d
         boxes); 8 heads x 32 channels, 4 levels at 1280 x 384.  CUDA events over 20 calls, 7 rounds with the cases
         alternating; median, min and max per call.
  step   the graph-captured training step (forward, surrogate loss of monodetr_b200.bench_model, backward) at batch 8,
         1280 x 384, in images/s, for enc / dec points 2 / 2, 4 / 4 and 8 / 8, ROUNDS times in alternating order.

    python tools/bench_points.py [--steps 20] [--rounds 2] [--skip-step]

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
from monodetr_b200 import _lib, tc  # noqa: E402

POINTS = (2, 4, 8)
LEVELS = [(48, 160), (24, 80), (12, 40), (6, 20)]
CALLS = [("encoder", 10200, 2), ("decoder", 550, 6)]
B, M, D, L = 8, 8, 32, 4


def msda_cases(dev):
    g = torch.Generator(device=dev).manual_seed(0)
    shapes = torch.tensor(LEVELS, dtype=torch.long, device=dev)
    lsi = torch.cat((shapes.new_zeros(1), shapes.prod(1).cumsum(0)[:-1]))
    S = int(shapes.prod(1).sum())
    value = torch.randn(B, S, M, D, device=dev, generator=g)
    cases = []
    for call, Lq, rd in CALLS:
        dout = torch.randn(B, Lq, M * D, device=dev, generator=g)
        ref = torch.rand(B, Lq, L, rd, device=dev, generator=g)
        if rd == 6:
            ref[..., 2:] *= 0.3
        for P in POINTS:
            off = torch.randn(B, Lq, M * L * P * 2, device=dev, generator=g)
            logits = torch.randn(B, Lq, M * L * P, device=dev, generator=g)
            out = torch.empty(B, Lq, M * D, device=dev)
            loc, attn = torch.empty(B, Lq, M, L, P, 2, device=dev), torch.empty(B, Lq, M, L, P, device=dev)
            gv, goff, glog = torch.empty_like(value), torch.empty_like(off), torch.empty_like(logits)
            gl, ga = torch.empty_like(loc), torch.empty_like(attn)
            a = (value, shapes, lsi)

            def fused_fwd(off=off, logits=logits, ref=ref, Lq=Lq, P=P, rd=rd, out=out):
                _lib.call("mdb_msda_fused_forward_f32", *a, off, logits, ref, B, S, M, D, L, Lq, P, rd, out)

            def fused_bwd(off=off, logits=logits, ref=ref, dout=dout, Lq=Lq, P=P, rd=rd, goff=goff, glog=glog):
                _lib.call("mdb_msda_fused_backward_f32", *a, off, logits, ref, dout, B, S, M, D, L, Lq, P, rd, gv, goff, glog)

            def two_fwd(off=off, logits=logits, ref=ref, Lq=Lq, P=P, rd=rd, out=out, loc=loc, attn=attn):
                _lib.call("mdb_msda_prep_forward_f32", off, logits, ref, shapes, B, Lq, M, L, P, rd, loc, attn)
                _lib.call("mdb_msda_forward_f32", *a, loc, attn, B, S, M, D, L, Lq, P, out)

            def two_bwd(ref=ref, dout=dout, Lq=Lq, P=P, rd=rd, loc=loc, attn=attn, gl=gl, ga=ga, goff=goff, glog=glog):
                _lib.call("mdb_msda_backward_f32", *a, loc, attn, dout, B, S, M, D, L, Lq, P, gv, gl, ga)
                _lib.call("mdb_msda_prep_backward_f32", gl, ga, attn, ref, shapes, B, Lq, M, L, P, rd, goff, glog)

            two_fwd()
            cases += [(call, P, "fused", "fwd", fused_fwd), (call, P, "fused", "bwd", fused_bwd),
                      (call, P, "two-step", "fwd", two_fwd), (call, P, "two-step", "bwd", two_bwd)]
    return cases


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_points needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tc.set_precision("bf16x3")
    print(json.dumps({"card": card(), "precision": tc.get_precision()}), flush=True)

    # ---- deformable-attention core, cases alternating ---------------------------------------------------------------------
    cases = msda_cases(dev)
    for *_, fn in cases:
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {c[:4]: [] for c in cases}
    n = 20
    for _ in range(7):
        for call, P, path, d, fn in cases:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(n):
                fn()
            e1.record()
            torch.cuda.synchronize()
            times[(call, P, path, d)].append(e0.elapsed_time(e1) / n * 1e3)
    for (call, P, path, d), t in times.items():
        print(json.dumps({"msda": call, "P": P, "path": path, "dir": d, "median_us": round(statistics.median(t), 1),
                          "min_us": round(min(t), 1), "max_us": round(max(t), 1)}), flush=True)
    del cases
    torch.cuda.empty_cache()

    # ---- training step per point count ------------------------------------------------------------------------------------
    if args.skip_step:
        return
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    base = bench_backbones.DEFAULT_MODEL_CFG
    res = {p: [] for p in POINTS}
    try:
        for r in range(args.rounds):
            for p in (POINTS if r % 2 == 0 else POINTS[::-1]):
                bench_backbones.DEFAULT_MODEL_CFG = dict(base, enc_n_points=p, dec_n_points=p)    # time_step builds from this
                ips, med = time_step("resnet50", False, args.steps, dev, flush)
                res[p].append(ips)
                print(json.dumps({"round": r, "points": p, "img_s": round(ips, 2), "median_step_ms": round(med, 2)}), flush=True)
    finally:
        bench_backbones.DEFAULT_MODEL_CFG = base
    for p in POINTS:
        print(json.dumps({"step": "train B=8 1280x384 graph", "enc/dec points": p, "img_s_per_round": [round(x, 2) for x in res[p]]}),
              flush=True)
    print(json.dumps({"card_after": card()}), flush=True)


if __name__ == "__main__":
    main()
