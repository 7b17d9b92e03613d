"""Per-kernel time shares of one eager training step, measured with torch.profiler (CUDA activities).

usage: profile_step_kernels.py [--batch 8] [--out DIR]

Two warm-up steps, then one profiled step.  Kernel times are summed per kernel name; every template instance of
`tc_conv_gemm_kernel` keeps its own row (its name carries the template arguments <BN, STAGES, MODE, B_MN, PREC>).  Kernels
of the side stream overlap the main stream, so the shares are of the summed kernel time, which can exceed the wall time
of the step printed beside it.  With --out the table is also written to DIR/step_kernels.txt."""
import argparse
import os
import re
import sys
import time
from collections import defaultdict

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from monodetr_b200 import build_monodetr, tc  # noqa: E402
from monodetr_b200.bench_model import surrogate_loss, synthetic_batch  # noqa: E402
from monodetr_b200.monodetr import DEFAULT_MODEL_CFG  # noqa: E402


def short_name(name):
    name = re.sub(r"\(anonymous namespace\)::|<unnamed>::|void |at::native::", "", name)
    return re.sub(r"\((CUtensorMap|[A-Za-z_:]+ const\*|float|int).*\)$", "", name).strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--out", default=None)
    ap.add_argument("--top", type=int, default=40)
    args = ap.parse_args()

    tc.set_precision(os.environ.get("MDB_PRECISION", "bf16x3"))
    torch.manual_seed(0)
    model, _ = build_monodetr(DEFAULT_MODEL_CFG)
    model = model.cuda().train()
    images, calibs, sizes = (t.cuda() for t in synthetic_batch(args.batch, 1))

    def step():
        for p in model.parameters():
            p.grad = None
        surrogate_loss(model(images, calibs, None, sizes)).backward()

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        step()
        torch.cuda.synchronize()
        wall_ms = (time.perf_counter() - t0) * 1e3

    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = short_name(e.name)
        tot[k] += e.time_range.elapsed_us()
        cnt[k] += 1
    total = sum(tot.values())
    gemm = sum(v for k, v in tot.items() if k.startswith("tc_conv_gemm_kernel"))
    lines = [f"{torch.cuda.get_device_name()}, batch {args.batch}: step wall {wall_ms:.2f} ms (profiled), "
             f"kernel time {total / 1e3:.2f} ms over {sum(cnt.values())} device activities; "
             f"tc_conv_gemm_kernel {gemm / 1e3:.2f} ms = {100 * gemm / max(total, 1e-9):.1f} %"]
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1])[:args.top]:
        lines.append(f"{v / 1e3:9.3f} ms {100 * v / total:5.1f}%  n={cnt[k]:4d}  avg {v / cnt[k]:8.1f} us  {k[:120]}")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_kernels.txt"), "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
