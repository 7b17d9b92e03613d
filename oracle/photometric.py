"""CPU restatement (numpy) of the reference's photometric distortion -- TEST INFRASTRUCTURE ONLY.

  PhotometricDistort.__call__   lib/datasets/kitti/pd.py:376-397, as called at lib/datasets/kitti/kitti_dataset.py:136-138:
                                `pd(np.array(img).astype(np.float32)).astype(np.uint8)`

Per pixel, in float32 (every scalar is a Python float applied to a float32 array, i.e. rounded to float32 first):
  1. brightness: x + delta
  2. contrast_last == 0 (pd[:-1]): x * alpha, BGR->HSV, S * sat, H + hue (wrapped), HSV->BGR
     contrast_last == 1 (pd[1:]):  BGR->HSV, S * sat, H + hue (wrapped), HSV->BGR, x * alpha
  3. channel permutation (RandomLightingNoise): out[c] = in[PERMS[perm][c]]
  4. astype(uint8): truncation toward zero, then modulo 256 (290.3 -> 34, -5.7 -> 251)

The two colour conversions are cv2.cvtColor on float32 (opencv color_hsv.simd.hpp) as it runs with AVX2 + FMA3 dispatch: the RGB
image is read as BGR, so channel 0 is "B".  Each row is converted by a vector loop over SIMD_WIDTH pixels and a scalar loop over
the remaining W % SIMD_WIDTH pixels at the end of the row; the two loops round differently in BGR->HSV:
  vector:  d = 60 / (diff + FLT_EPSILON) (float32), H = fma(num, d, off), off = 0 / 120 / 240, 360 folded into the FMA when V == R
           and num < 0
  scalar:  d = (float)(60.0 / (diff + FLT_EPSILON)) (double), H = fma(num, d, off), then H < 0 -> H + 360
(SIMD_WIDTH = 8 and both rules were found by comparing with cv2 4.13 on every width 1..40 and 1224..1242.)
HSV->BGR is the same in both: hs = H * (6/360)f, sector = trunc(hs) mod 6, f = hs - trunc(hs),
tab = {v, v * (1 - s), v * fma(-s, f, 1), v * fma(-s, 1 - f, 1)}.
FMA is emulated exactly (round-to-odd in float64, then one rounding to float32).

Pinned against the unmodified pd.py + cv2 by tests/golden/photometric.npz (tools/gen_golden_photometric.py) and, where the
reference tree is present, live (tests/test_oracle_photometric.py).
"""
from typing import NamedTuple

import numpy as np

PERMS = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))       # pd.py:143-145
SECTOR = ((1, 3, 0), (1, 0, 2), (3, 0, 1), (0, 2, 1), (0, 1, 3), (2, 1, 0))       # cv2 HSV2RGB sector table (b, g, r)
SIMD_WIDTH = 8
FLT_EPS = np.float32(np.finfo(np.float32).eps)
F32 = np.float32


class Params(NamedTuple):
    """One image's draws.  A step whose coin said no carries its neutral value (0 / 1 / 1 / 0 / perm 0), which gives the same bits
    as skipping it."""
    brightness: float = 0.0
    contrast: float = 1.0
    saturation: float = 1.0
    hue: float = 0.0
    contrast_last: int = 0
    perm: int = 0


def sample(rs=np.random):
    """The draws of pd.py:389-397 from `rs` (the global numpy.random by default), in the reference's order."""
    p = {}
    if rs.randint(2):                                                      # RandomBrightness
        p["brightness"] = rs.uniform(-32, 32)
    first = rs.randint(2)                                                  # pd[:-1] (contrast first) or pd[1:]
    p["contrast_last"] = 0 if first else 1
    if first and rs.randint(2):                                            # RandomContrast (first)
        p["contrast"] = rs.uniform(0.5, 1.5)
    if rs.randint(2):                                                      # RandomSaturation
        p["saturation"] = rs.uniform(0.5, 1.5)
    if rs.randint(2):                                                      # RandomHue
        p["hue"] = rs.uniform(-18.0, 18.0)
    if not first and rs.randint(2):                                        # RandomContrast (last)
        p["contrast"] = rs.uniform(0.5, 1.5)
    if rs.randint(2):                                                      # RandomLightingNoise
        p["perm"] = rs.randint(6)
    return Params(**p)


def fma32(a, b, c):
    """float32 fma(a, b, c), correctly rounded: the product of two float32 is exact in float64, the sum is rounded to odd, then
    rounded once to float32."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = np.broadcast_to(np.asarray(c, np.float64), p.shape)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                                          # TwoSum: s + e == p + c exactly
    odd = (s.view(np.int64) & 1) == 1
    fix = (e != 0) & ~odd
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def bgr2hsv(x, simd_width=SIMD_WIDTH):
    b, g, r = x[..., 0], x[..., 1], x[..., 2]
    v = np.maximum(np.maximum(r, g), b)
    vmin = np.minimum(np.minimum(r, g), b)
    diff = v - vmin
    s = diff / (np.abs(v) + FLT_EPS)
    r_max, g_max = r == v, g == v
    num = np.where(r_max, g - b, np.where(g_max, b - r, r - g))
    off = np.where(r_max, F32(0), np.where(g_max, F32(120), F32(240))).astype(np.float32)
    dd = diff + FLT_EPS
    # vector loop
    off_v = np.where(r_max & (num < 0), F32(360), off)
    h = fma32(num, F32(60) / dd, off_v)
    # scalar tail of each row
    W = x.shape[1]
    t0 = W - W % simd_width
    if t0 < W:
        ds = (60.0 / dd[:, t0:].astype(np.float64)).astype(np.float32)
        ht = fma32(num[:, t0:], ds, off[:, t0:])
        h[:, t0:] = np.where(ht < 0, ht + F32(360), ht)
    return h, s, v


def hsv2bgr(h, s, v):
    hs = h * F32(6.0 / 360.0)
    pre = np.trunc(hs)
    f = hs - pre
    sector = (pre - np.trunc(pre * F32(1.0 / 6.0)) * F32(6)).astype(np.int64)
    sector = np.where(sector < 0, sector + 6, sector)
    tab = np.stack([v, v * (F32(1) - s), v * fma32(-s, f, F32(1)), v * fma32(-s, F32(1) - f, F32(1))], -1)
    idx = np.asarray(SECTOR)[sector]                                       # (..., 3): tab index of b, g, r
    return np.take_along_axis(tab, idx, -1)


def distort_float(img_u8, p: Params, simd_width=SIMD_WIDTH):
    """(H, W, 3) uint8 -> the float32 image pd() returns (before the uint8 cast)."""
    x = img_u8.astype(np.float32)
    x = x + F32(p.brightness)
    if not p.contrast_last:
        x = x * F32(p.contrast)
    h, s, v = bgr2hsv(x, simd_width)
    s = s * F32(p.saturation)
    h = h + F32(p.hue)
    h = np.where(h > F32(360), h - F32(360), h)
    h = np.where(h < F32(0), h + F32(360), h)
    x = hsv2bgr(h, s, v)
    if p.contrast_last:
        x = x * F32(p.contrast)
    return x[..., list(PERMS[p.perm])]


def distort_float_rows(img_u8, p: Params, simd_width=SIMD_WIDTH, workers=8):
    """distort_float over blocks of rows on a thread pool (numpy releases the GIL in its loops): the same bits, since each row
    is converted on its own.  For the all-colour images, where one call is 2**24 pixels."""
    from concurrent.futures import ThreadPoolExecutor
    blocks = np.array_split(np.arange(img_u8.shape[0]), workers)
    with ThreadPoolExecutor(workers) as ex:
        parts = ex.map(lambda r: distort_float(img_u8[r[0]:r[-1] + 1], p, simd_width), [r for r in blocks if len(r)])
        return np.concatenate(list(parts))


def every_colour(W):
    """All 2**24 8-bit colours, in order, in one (ceil(2**24 / W), W, 3) image; a last partial row is filled with colour 0.
    W % SIMD_WIDTH == 0 sends every pixel through cv2's vector loop, W < SIMD_WIDTH through its scalar loop."""
    n = 1 << 24
    H = -(-n // W)
    c = np.zeros(H * W, np.uint32)
    c[:n] = np.arange(n, dtype=np.uint32)
    return np.stack([c >> 16, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(H, W, 3)


# Records at the ends of the sampled ranges (brightness +-32, contrast and saturation 0.5 / 1.5, hue +-18), both contrast orders,
# every channel permutation, and the neutral record.
EDGE_RECORDS = (Params(32.0, 1.5, 1.5, 18.0, 0, 0), Params(-32.0, 0.5, 0.5, -18.0, 1, 1), Params(32.0, 0.5, 1.5, -18.0, 0, 2),
                Params(-32.0, 1.5, 0.5, 18.0, 1, 3), Params(0.0, 1.5, 1.5, 18.0, 1, 4), Params(32.0, 1.5, 0.5, -18.0, 1, 5),
                Params(-32.0, 0.5, 1.5, 18.0, 0, 5), Params())


def to_u8(x):
    """numpy's float32 -> uint8 cast as it behaves on x86: truncate toward zero, keep the low 8 bits."""
    return np.trunc(x).astype(np.int64).astype(np.uint8)


def distort(img_u8, p: Params, simd_width=SIMD_WIDTH):
    return to_u8(distort_float(img_u8, p, simd_width))


def replay_getitem(gold, k, sample, get_affine_transform):
    """The image-side draws of KITTI_Dataset.__getitem__ (kitti_dataset.py:130-154) for the fixture's end-to-end case k:
    np.random.seed, the distortion's draws through `sample()`, then the flip and crop draws.  Returns (record, flip, trans_inv)."""
    np.random.seed(int(gold["e2e.seeds"][k]))
    rec = sample()
    img_size = np.array([int(v) for v in gold["e2e.size"]])
    center = np.array(img_size) / 2
    crop_size = img_size
    scale, shift = float(gold["e2e.scale"]), float(gold["e2e.shift"])
    flip = bool(np.random.random() < float(gold["e2e.random_flip"]))
    if np.random.random() < float(gold["e2e.random_crop"]):
        crop_scale = np.clip(np.random.randn() * scale + 1, 1 - scale, 1 + scale)
        crop_size = img_size * crop_scale
        center[0] += img_size[0] * np.clip(np.random.randn() * shift, -2 * shift, 2 * shift)
        center[1] += img_size[1] * np.clip(np.random.randn() * shift, -2 * shift, 2 * shift)
    trans_inv = get_affine_transform(center, crop_size, 0, np.array([int(v) for v in gold["e2e.res"]]), inv=1)[1]
    return rec, flip, trans_inv


def state_matches(gold, prefix):
    """np.random.get_state() equals the one stored under `prefix` in the fixture."""
    _, keys, pos, has_gauss, gauss = np.random.get_state()
    g = gold[prefix + "state_gauss"]
    return (np.array_equal(keys, gold[prefix + "state_keys"]) and pos == int(gold[prefix + "state_pos"])
            and has_gauss == int(g[0]) and gauss == g[1])
