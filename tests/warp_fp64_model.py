"""Exact model of the device warp's fp64 arithmetic at one output pixel (csrc/preprocess.cu, warp_affine_normalize_kernel), in
two forms -- TEST INFRASTRUCTURE ONLY.

  separate   every product rounded before its sum, in Pillow's order (Geometry.c, affine_transform + BILINEAR, as built for
             x86-64 without FMA): xin = (a0*xc + a1*yc) + a2, then - 0.5; v = a + (b - a) * d.  The kernel computes this.
  fused      what nvcc makes of the same source written with plain `*` and `+` (its sm_90a SASS contracts into DFMA):
             xin = fma(a0, xc, a1*yc) + a2, yin = fma(a3, xc, a4*yc) + a5, v = fma(b - a, d, a) for all three bilinear steps.

A float64 FMA is computed exactly with Fraction and rounded once (CPython's int / int true division is correctly rounded).
Python's own float arithmetic rounds every operation, so the separate form is plain Python.
"""
import math
from fractions import Fraction


def fma(a, b, c):
    """float64 fma(a, b, c), correctly rounded."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def coords(data, x, y, fused):
    """(xin, yin) of output pixel (x, y) before the bounds test."""
    a0, a1, a2, a3, a4, a5 = (float(v) for v in data)
    xc, yc = x + 0.5, y + 0.5
    if fused:
        return fma(a0, xc, a1 * yc) + a2, fma(a3, xc, a4 * yc) + a5
    return a0 * xc + a1 * yc + a2, a3 * xc + a4 * yc + a5


def lerp(a, b, d, fused):
    return fma(b - a, d, a) if fused else a + (b - a) * d


def sample(img, data, x, y, fused):
    """The 8-bit (r, g, b) that output pixel (x, y) gets from (H, W, 3) uint8 `img` under the affine `data`."""
    H, W, _ = img.shape
    xin, yin = coords(data, x, y, fused)
    if xin < 0.0 or xin >= W or yin < 0.0 or yin >= H:
        return (0, 0, 0)
    xin, yin = xin - 0.5, yin - 0.5
    xf, yf = math.floor(xin), math.floor(yin)
    dx, dy = xin - xf, yin - yf
    x0, x1 = min(max(xf, 0), W - 1), min(max(xf + 1, 0), W - 1)
    y0 = min(max(yf, 0), H - 1)
    has_y1 = 0 <= yf + 1 < H
    out = []
    for c in range(3):
        v1 = lerp(float(img[y0, x0, c]), float(img[y0, x1, c]), dx, fused)
        v2 = lerp(float(img[yf + 1, x0, c]), float(img[yf + 1, x1, c]), dx, fused) if has_y1 else v1
        out.append(int(lerp(v1, v2, dy, fused)))
    return tuple(out)
