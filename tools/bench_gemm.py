"""GPU micro-benchmark of the wgmma conv/linear family on the model's real shapes (B=8), both precision modes.

--tile-probe: the per-tile fixed cost of the GEMM instead (see tile_probe)."""
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from monodetr_b200 import tc  # noqa: E402

B = 8
SHAPES = [  # name, H, W, Cin, Cout, k, stride
    ("l1.conv1 1x1 64->64", 96, 320, 64, 64, 1, 1),
    ("l1.conv2 3x3 64->64", 96, 320, 64, 64, 3, 1),
    ("l1.conv3 1x1 64->256", 96, 320, 64, 256, 1, 1),
    ("l1.conv1 1x1 256->64", 96, 320, 256, 64, 1, 1),
    ("l2.conv2 3x3 128->128", 48, 160, 128, 128, 3, 1),
    ("l2.conv3 1x1 128->512", 48, 160, 128, 512, 1, 1),
    ("l3.conv2 3x3 256->256", 24, 80, 256, 256, 3, 1),
    ("l3.conv3 1x1 256->1024", 24, 80, 256, 1024, 1, 1),
    ("l3.conv1 1x1 1024->256", 24, 80, 1024, 256, 1, 1),
    ("l4.conv2 3x3 512->512", 12, 40, 512, 512, 3, 1),
    ("enc linear 256->256 (M=81600)", 1, 10200, 256, 256, 1, 1),
]


def timeit(fn, n=10):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3   # us


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0] + f"  ({q})"
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name()


def sm_mhz():
    """Current SM clock of device 0 in MHz (nvidia-smi), or None."""
    try:
        return float(subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                                    capture_output=True, text=True, timeout=30).stdout.split()[0])
    except (OSError, subprocess.SubprocessError, IndexError, ValueError):
        return None


def pick_tile3(W, H, Bn, n_pix=128):
    """(tw, th, tb) of an fprop / dgrad M tile: restates pick_tile3 of conv_gemm.cu."""
    best, res = -1, (n_pix, 1, 1)
    b = 1
    while b <= n_pix:
        w = n_pix // b
        while w >= 1:
            h = n_pix // b // w
            if not (b > 1 and b >= 2 * Bn):
                cov = -(-W // w) * w * -(-H // h) * h * -(-Bn // b) * b
                if best < 0 or cov < best:
                    best, res = cov, (w, h, b)
            w >>= 1
        b <<= 1
    return res


def pick_bn(N, m_tiles, kblocks, sms, mode):
    """Tile width of an fprop / dgrad launch with N output columns: restates pick_bn of conv_gemm.cu (BF16x3 only)."""
    base = 64 if N <= 64 else 128
    if mode != "bf16x3" or N % 256 or kblocks < 64:
        return base
    t = m_tiles * (N // 256)
    return 256 if 2 * -(-t // sms) <= -(-2 * t // sms) else base


def fwd_schedule(H, W, Cin, Cout, k, sms, mode="bf16x3"):
    """(tiles per CTA, k-blocks per tile, tile width) of a stride-1 fprop launch (B = 8) with Cin in, Cout out; a dgrad
    of the layer Cin -> Cout is the fprop Cout -> Cin.  Restates the tile walk of conv_forward_impl (no split-K at these
    shapes)."""
    if k == 1:
        W, H, Bn = B * H * W, 1, 1
    else:
        Bn = B
    tw, th, tb = pick_tile3(W, H, Bn)
    m_tiles = -(-W // tw) * -(-H // th) * -(-Bn // tb)
    kb = k * k * -(-Cin // 32)
    bn = pick_bn(Cout, m_tiles, kb, sms, mode)
    tiles = m_tiles * -(-Cout // bn)
    return -(-tiles // min(tiles, sms)), kb, bn


def wgrad_schedule(M, Cin, Cout, sms):
    """(tiles per CTA, k-blocks per tile) of a pointwise wgrad launch: restates the split rule of mdb_conv2d_wgrad_bias_f32."""
    total_red = (M + 31) // 32
    tiles = ((Cout + 127) // 128) * ((Cin + 127) // 128)
    big, small = min((2 * sms + tiles - 1) // tiles, total_red // 24), min(sms // tiles, total_red // 8)
    per = -(-total_red // max(big, small, 1))
    n = tiles * -(-total_red // per)
    return -(-n // min(n, sms)), per


def fit(rows):
    """Least squares t = fixed * tiles_per_cta + per_kb * tiles_per_cta * kb over rows of (tiles_per_cta, kb, t)."""
    X = np.array([[tpc, tpc * kb] for tpc, kb, _ in rows], dtype=np.float64)
    (fixed, per_kb), *_ = np.linalg.lstsq(X, np.array([t for *_, t in rows]), rcond=None)
    return fixed, per_kb


def tile_probe():
    """Per-tile fixed cost of tc_conv_gemm_kernel (BF16x3) at the encoder size M = 81 600, N = 256.  K (the reduction, 1-8
    k-blocks of 32) varies at a constant tile count, so the fit t = tiles_per_cta * (fixed + kb * per_kb) separates the
    cost of a tile's k-blocks from what a tile costs whatever its K (epilogue, tile switch; the launch is in it too).
    wgrad varies M instead, which changes both its split count and the k-blocks per split."""
    tc.set_precision("bf16x3")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M, N = 81600, 256
    tpc = -(-(-(-M // 128) * (N // 128)) // sms)
    print(f"== tile probe: {card()}; {sms} SMs, M = {M}, N = {N}, {tpc} tiles per CTA in fwd / dgrad")
    res = {"fwd": [], "fwd+res": [], "dgrad+mask": [], "wgrad": []}
    for K in (32, 64, 128, 256):
        x = torch.randn(M, K, device="cuda")
        w = tc.split_weights([torch.randn(N, K, 1, 1, device="cuda") / K ** 0.5])[0]
        wd = tc.split_weights([torch.randn(K, N, 1, 1, device="cuda") / N ** 0.5])[0]   # layer N -> K: its dgrad writes N
        r = torch.randn(M, N, device="cuda")
        dy = torch.randn(M, K, device="cuda")
        x4, r4, dy4 = x.view(1, 1, M, K), r.view(1, 1, M, N), dy.view(1, 1, M, K)
        kb = K // 32
        t_f = timeit(lambda: tc.conv2d_forward(x4, w), 50)
        t_fr = timeit(lambda: tc.conv2d_forward(x4, w, None, r4, relu=True), 50)
        t_d = timeit(lambda: tc.conv2d_dgrad(dy4, wd, (1, 1, M, N), r4, r4), 50)
        floor = lambda nbytes: nbytes / 3.35e6   # us at the data-sheet 3.35 TB/s
        out_b, in_b = M * N * 4, M * K * 4
        res["fwd"].append((tpc, kb, t_f))
        res["fwd+res"].append((tpc, kb, t_fr))
        res["dgrad+mask"].append((tpc, kb, t_d))
        print(f"K = {K:3d}: fwd {t_f:7.1f} us (HBM floor {floor(in_b + out_b):5.1f})  fwd+res+relu {t_fr:7.1f} "
              f"(floor {floor(in_b + 2 * out_b):5.1f})  dgrad+res+mask {t_d:7.1f} (floor {floor(in_b + 3 * out_b):5.1f})")
    for Mw in (10200, 20400, 40800, 81600):
        dy, x = torch.randn(1, 1, Mw, N, device="cuda"), torch.randn(1, 1, Mw, N, device="cuda")
        t_w = timeit(lambda: tc.conv2d_wgrad(dy, x), 50)
        wt, wkb = wgrad_schedule(Mw, N, N, sms)
        res["wgrad"].append((wt, wkb, t_w))
        print(f"wgrad {N}x{N} over M = {Mw:5d}: {t_w:7.1f} us ({wt} tiles per CTA, {wkb} k-blocks per tile)")
    mhz = sm_mhz()
    print(f"SM clock sampled after the timings: {mhz} MHz")
    for name, rows in res.items():
        fixed, per_kb = fit(rows)
        t_enc = rows[-1][2]
        clk = f" ({per_kb * mhz:5.0f} clk)" if mhz else ""
        print(f"{name:11s} fixed {fixed:6.2f} us/tile, {per_kb:6.3f} us/k-block{clk};  at the largest point fixed x tiles per CTA = "
              f"{fixed * rows[-1][0]:6.1f} us of {t_enc:6.1f} us ({100 * fixed * rows[-1][0] / t_enc:4.1f} %)")


if "--tile-probe" in sys.argv:
    tile_probe()
    sys.exit(0)

sms = torch.cuda.get_device_properties(0).multi_processor_count
print(f"== {card()}; {sms} SMs.  clk/kb = SM clocks per k-block of 32 (time x SM clock / (tiles per CTA x k-blocks per tile)); "
      "n = tile width (a 256-wide tile does twice a 128-wide one's work per k-block)")
for mode in tuple(os.environ["MDB_MODES"].split(",")) if os.environ.get("MDB_MODES") else (("tf32x3",) if os.environ.get("MDB_ONLY_X3") else ("bf16x3", "tf32x3", "tf32")):
    tc.set_precision(mode)
    print(f"== {mode}")
    mhz = None
    for name, H, W, Cin, Cout, k, s in SHAPES:
        x = torch.randn(B, H, W, Cin, device="cuda")
        w = torch.randn(Cout, Cin, k, k, device="cuda") / (Cin * k * k) ** 0.5
        wp = tc.split_weights([w])[0] if mode == "bf16x3" else tc.pack_weight(w)
        pad = k // 2
        y = tc.conv2d_forward(x, wp, None, None, k, k, s, pad)
        dy = torch.randn_like(y)
        res = torch.randn_like(y)
        flop = 2.0 * y.numel() * Cin * k * k
        byt = (x.numel() + y.numel()) * 4
        t_f = timeit(lambda: tc.conv2d_forward(x, wp, None, None, k, k, s, pad))
        t_fr = timeit(lambda: tc.conv2d_forward(x, wp, None, res, k, k, s, pad, relu=True))
        t_d = timeit(lambda: tc.conv2d_dgrad(dy, wp, x.shape, None, x, k, k, s, pad))
        t_w = timeit(lambda: tc.conv2d_wgrad(dy, x, None, k, k, s, pad))
        mhz = mhz or sm_mhz()   # sampled once per mode, right after the first shape's timings
        clk = lambda t, sched: f"{t * mhz / (sched[0] * sched[1]):5.0f}" if mhz else "  n/a"
        sf, sd = fwd_schedule(H, W, Cin, Cout, k, sms, mode), fwd_schedule(H, W, Cout, Cin, k, sms, mode)
        print(f"{name:34s} fwd {t_f:7.1f} us ({flop / t_f / 1e6:6.1f} TF/s, {byt / t_f / 1e3:6.0f} GB/s, "
              f"{clk(t_f, sf)} clk/kb, n {sf[2]:3d})  fwd+res {t_fr:7.1f}  "
              f"dgrad+mask {t_d:7.1f} ({flop / t_d / 1e6:6.1f} TF/s, {clk(t_d, sd)} clk/kb, n {sd[2]:3d})  "
              f"wgrad {t_w:7.1f} ({flop / t_w / 1e6:6.1f} TF/s)")
    print(f"   SM clock sampled: {mhz} MHz")
