"""Constructed inputs on which the warp's fp64 arithmetic decides the 8-bit result: the floor of a sample coordinate and the
truncation of the interpolated value, where rounding each product before its sum (Pillow, the fixed kernel) and fusing it into an
FMA (what nvcc makes of a plain fp64 `a * b + c`) give different 8-bit values.  Each case is a small image, an affine `data`, the
output size and the output pixel / channel where the two forms disagree, checked against live Pillow here.

    python tools/gen_golden_preprocess_edges.py      -> tests/golden/preprocess_edges.npz

Cases:
  floor_x   sheared maps (a1 != 0) on a horizontal ramp: fused and separate `xin - 0.5` fall on two sides of an integer
            (the first is the 16x16 ramp img[:, x] = 10x, data (1/30, 0.1, 0.1, 0, 1, 0), 140x12, pixel (130, 10): Pillow 49,
            fused 50)
  floor_y   the same for `yin` (a3 != 0) on a vertical ramp
  trunc     scalings by small-denominator factors (a1 = a3 = 0, so both forms give the same coordinates) with the four
            neighbours chosen so that one form's interpolated value is an integer and the other's is just below it
"""
import math
import os
import sys

import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import preprocess as op  # noqa: E402
import warp_fp64_model as wm  # noqa: E402

RAMP = (10, 7, 15)                    # per-channel slope of the ramp images: 16 steps stay inside 0..255


def ramp(W, H, axis):
    t = np.arange(W if axis == 0 else H)
    chans = np.stack([(s * t) % 256 for s in RAMP], -1).astype(np.uint8)
    return np.broadcast_to(chans[None, :, :] if axis == 0 else chans[:, None, :], (H, W, 3)).copy()


def pillow(img, data, out_wh):
    return np.array(Image.fromarray(img).transform(tuple(out_wh), Image.AFFINE, data=tuple(float(v) for v in data),
                                                   resample=Image.BILINEAR))


def disagreement(img, data, x, y):
    """(channel, separate value, fused value) of the first channel where the two forms differ at (x, y), or None."""
    s, f = wm.sample(img, data, x, y, False), wm.sample(img, data, x, y, True)
    for c in range(3):
        if s[c] != f[c]:
            return c, s[c], f[c]
    return None


def floor_cases(axis, rng, want, tries=400):
    """Sheared maps on a ramp along `axis`; output pixels whose coordinate sits within 1e-9 of an integer after - 0.5 are
    checked exactly in both forms."""
    out, W, H, Wo, Ho = [], 16, 16, 64, 48
    img = ramp(W, H, axis)
    for _ in range(tries):
        q = [int(v) for v in rng.integers(2, 41, 4)]
        if axis == 0:
            data = (1 / q[0], int(rng.integers(1, 6)) / q[1], int(rng.integers(-5, 6)) / 10, 0.0, W / Wo * 3 / 4, 0.0)
        else:
            data = (W / Wo * 3 / 4, 0.0, 0.0, int(rng.integers(1, 6)) / q[1], 1 / q[0], int(rng.integers(-5, 6)) / 10)
        xs, ys = np.meshgrid(np.arange(Wo) + 0.5, np.arange(Ho) + 0.5)
        a = data[0:3] if axis == 0 else data[3:6]
        t = a[0] * xs + a[1] * ys + a[2] - 0.5
        for y, x in zip(*np.nonzero(np.abs(t - np.rint(t)) < 1e-9)):
            d = disagreement(img, data, int(x), int(y))
            if d is not None:
                out.append((img, data, (Wo, Ho), (int(x), int(y), d[0])))
                break
        if len(out) == want:
            return out
    raise RuntimeError(f"floor search (axis {axis}): {len(out)} of {want} cases")


def trunc_cases(rng, want_each, n=400_000):
    """Scalings by 1/s (s small): per output pixel the (dx, dy) pair is fixed, so draw random neighbour quadruples, keep the
    ones whose separate value is within 1e-9 of an integer and check them exactly; `want_each` cases of each sign of
    fused - separate, at most one of each sign per scaling."""
    W, H = 12, 10
    hits = {+1: [], -1: []}
    for sx, sy in ((6, 35), (3, 3), (2, 3), (3, 2), (12, 5), (6, 7), (5, 12), (35, 6)):
        data = (1 / sx, 0.0, 0.0, 0.0, 1 / sy, 0.0)
        Wo, Ho = min(W * sx, 256), min(H * sy, 256)
        seen, signs = set(), set()
        for y in range(Ho):
            for x in range(Wo):
                xin, yin = wm.coords(data, x, y, False)
                assert (xin, yin) == wm.coords(data, x, y, True)          # a1 = a3 = 0: the same coordinates
                xin, yin = xin - 0.5, yin - 0.5
                xf, yf = math.floor(xin), math.floor(yin)
                dx, dy = xin - xf, yin - yf
                if not (0 <= xf < W - 1 and 0 <= yf < H - 1) or dx == 0 or dy == 0 or (dx, dy) in seen:
                    continue
                seen.add((dx, dy))
                q = rng.integers(0, 256, (n, 4)).astype(np.float64)
                v1 = q[:, 0] + (q[:, 1] - q[:, 0]) * dx
                v2 = q[:, 2] + (q[:, 3] - q[:, 2]) * dx
                v = v1 + (v2 - v1) * dy
                exact = (v1 == np.rint(v1)) & (v2 == np.rint(v2)) & (v == np.rint(v))     # no rounding anywhere: no case
                for i in np.nonzero((np.abs(v - np.rint(v)) < 1e-9) & ~exact)[0][:200]:
                    p = [float(t) for t in q[i]]
                    s = int(wm.lerp(wm.lerp(p[0], p[1], dx, False), wm.lerp(p[2], p[3], dx, False), dy, False))
                    f = int(wm.lerp(wm.lerp(p[0], p[1], dx, True), wm.lerp(p[2], p[3], dx, True), dy, True))
                    sign = int(np.sign(f - s))
                    if s != f and sign not in signs and len(hits[sign]) < want_each:
                        signs.add(sign)
                        c = int(rng.integers(0, 3))
                        img = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
                        img[yf, xf, c], img[yf, xf + 1, c], img[yf + 1, xf, c], img[yf + 1, xf + 1, c] = p
                        assert disagreement(img, data, x, y)[0] == c
                        hits[sign].append((img, data, (Wo, Ho), (x, y, c)))
                        break
                if all(len(h) == want_each for h in hits.values()):
                    return hits[+1] + hits[-1]
    raise RuntimeError(f"truncation search: {len(hits[+1])} / {len(hits[-1])} of {want_each} cases")


def main():
    rng = np.random.default_rng(20261018)
    cases = [("floor_x", ramp(16, 16, 0), (1 / 30, 0.1, 0.1, 0.0, 1.0, 0.0), (140, 12), (130, 10, 0))]
    cases += [("floor_x", *c) for c in floor_cases(0, rng, 3)]
    cases += [("floor_y", *c) for c in floor_cases(1, rng, 3)]
    cases += [("trunc", *c) for c in trunc_cases(rng, 3)]
    out = {"n": np.array(len(cases))}
    for k, (kind, img, data, out_wh, (x, y, c)) in enumerate(cases):
        pil = pillow(img, data, out_wh)
        assert np.array_equal(pil, op.warp_affine_bilinear(img, data, out_wh)), k
        sep, fused = wm.sample(img, data, x, y, False), wm.sample(img, data, x, y, True)
        assert pil[y, x, c] == sep[c] != fused[c], (k, kind, pil[y, x, c], sep, fused)
        out.update({f"{k}.kind": np.array(kind), f"{k}.img": img, f"{k}.data": np.array(data, np.float64),
                    f"{k}.out_wh": np.array(out_wh), f"{k}.pixel": np.array([x, y, c]),
                    f"{k}.pillow": np.array(int(pil[y, x, c])), f"{k}.fused": np.array(fused[c])})
        print(k, kind, [float(v) for v in data], out_wh, (x, y, c), "pillow", int(pil[y, x, c]), "fused", fused[c])
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "preprocess_edges.npz"), **out)


if __name__ == "__main__":
    main()
