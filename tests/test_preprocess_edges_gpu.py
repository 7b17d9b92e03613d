"""Device input pipeline at its decision edges, bit for bit: the warp (csrc/preprocess.cu, warp_affine_normalize_kernel) against
live Pillow and oracle/preprocess.py, the photometric distortion against oracle/photometric.py on every 8-bit colour.

The warp's 8-bit value is decided by a floor of each sample coordinate and a truncation of the interpolated value; random smooth
images and random crops almost never land on either.  The cases here do: the constructed inputs of
tests/golden/preprocess_edges.npz (tools/gen_golden_preprocess_edges.py), where rounding every product before its sum (Pillow)
and fusing it into an FMA give different bytes, sample points exactly on and one ulp off the image border, degenerate sources,
the grid's x tail, flips, mirrors, pitched sources and the reference's own transforms."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import photometric as ph
from oracle import preprocess as op

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "preprocess_edges.npz"))
KITTI_SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376)]
# normalize() of every 8-bit value, per channel: (3, 256), increasing
TABLE = op.normalize(np.repeat(np.arange(256, dtype=np.uint8)[None, :, None], 3, -1))[:, 0, :]


def _pillow(img, data, out_wh):
    return np.array(Image.fromarray(np.ascontiguousarray(img)).transform(
        tuple(int(v) for v in out_wh), Image.AFFINE, data=tuple(float(v) for v in np.asarray(data).reshape(-1)),
        resample=Image.BILINEAR))


def _u8(out):
    """(3, H, W) normalised device output -> the (3, H, W) 8-bit values it was normalised from (-1 where it is none)."""
    got = np.full(out.shape, -1, np.int64)
    for c in range(3):
        i = np.clip(np.searchsorted(TABLE[c], out[c]), 0, 255)
        got[c] = np.where(TABLE[c][i] == out[c], i, -1)
    return got


def _warp(imgs, datas, out_wh, flips=None):
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    srcs = [im if torch.is_tensor(im) else torch.from_numpy(np.ascontiguousarray(im)) for im in imgs]
    pre = ImageBatchPreprocessor(resolution=tuple(int(v) for v in out_wh))
    return pre(srcs, np.asarray(datas, np.float64).reshape(-1, 2, 3), flips).cpu().numpy()


def _mismatch(out, img, data, out_wh, flip=False):
    """None when the device output equals normalize(Pillow) bit for bit and the oracle equals Pillow; else a short report."""
    src = np.ascontiguousarray(img[:, ::-1] if flip else img)
    want = _pillow(src, data, out_wh)
    if not np.array_equal(op.warp_affine_bilinear(src, np.asarray(data).reshape(-1), tuple(out_wh)), want):
        return "the oracle differs from Pillow"
    got, want = _u8(out), want.transpose(2, 0, 1).astype(np.int64)
    bad = np.argwhere(got != want)
    if len(bad):
        return f"{len(bad)} bytes differ, first (c, y, x, device, Pillow): " + \
            str([(int(c), int(y), int(x), int(got[c, y, x]), int(want[c, y, x])) for c, y, x in bad[:4]])
    if not np.array_equal(out, op.normalize(want.transpose(1, 2, 0).astype(np.uint8))):
        return "the normalisation differs"
    return None


def _check_all(cases):
    """cases: (label, img, data, out_wh, flip); one launch per case; every mismatch reported together."""
    bad = []
    for label, img, data, out_wh, flip in cases:
        out = _warp([img], [data], out_wh, None if flip is None else [flip])[0]
        m = _mismatch(out, img, data, out_wh, bool(flip))
        if m:
            bad.append((label, m))
    assert not bad, bad


def _case(k):
    g = lambda name: GOLD[f"{k}.{name}"]  # noqa: E731
    return str(g("kind")), g("img"), g("data"), tuple(int(v) for v in g("out_wh")), tuple(int(v) for v in g("pixel"))


def test_fused_and_separate_arithmetic_disagree_here():
    """Each case's pixel is one where an FMA-contracted coordinate map or interpolation gives another byte than Pillow's
    separately rounded one (tests/test_preprocess_edges_host_logic.py proves it on the host): on the floor of a sheared
    coordinate, and on the 8-bit truncation.  Case 0 is the 16x16 ramp where Pillow gives 49 and the fused form 50."""
    n = int(GOLD["n"])
    assert {_case(k)[0] for k in range(n)} == {"floor_x", "floor_y", "trunc"}
    bad = []
    for k in range(n):
        kind, img, data, out_wh, (x, y, c) = _case(k)
        out = _warp([img], [data], out_wh)[0]
        got = int(_u8(out)[c, y, x])
        if got != int(GOLD[f"{k}.pillow"]):
            bad.append(f"case {k} ({kind}) pixel ({x}, {y}) channel {c}: device {got}, Pillow {int(GOLD[f'{k}.pillow'])}, "
                       f"fused arithmetic {int(GOLD[f'{k}.fused'])}")
        m = _mismatch(out, img, data, out_wh)
        if m:
            bad.append(f"case {k} ({kind}): {m}")
    assert not bad, "\n".join(bad)


def test_sample_points_on_the_border():
    """xin / yin exactly 0, one ulp below 0, one ulp below W / H and exactly W / H (zero fill); a0 = a1 = 0 makes xin = a2
    exactly.  Translations by -0.5 / +0.5 put the first / last pixel centre exactly on 0 / W through the full map.  Upsampling by
    4 samples xf == -1 and yf == -1 (clamped neighbours) and yf + 1 == H (no second row)."""
    g = np.random.default_rng(1)
    W, H = 7, 5
    img = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
    cases = []
    for name, X in (("0", 0.0), ("-ulp", np.nextafter(0.0, -1.0)), ("W-ulp", np.nextafter(float(W), 0.0)), ("W", float(W))):
        cases.append((f"xin={name}", img, (0.0, 0.0, X, 0.0, 1.0, 0.0), (3, H), None))
    for name, Y in (("0", 0.0), ("-ulp", np.nextafter(0.0, -1.0)), ("H-ulp", np.nextafter(float(H), 0.0)), ("H", float(H))):
        cases.append((f"yin={name}", img, (1.0, 0.0, 0.0, 0.0, 0.0, Y), (W, 3), None))
    cases += [("translate -0.5", img, (1.0, 0.0, -0.5, 0.0, 1.0, -0.5), (W, H), None),
              ("translate +0.5", img, (1.0, 0.0, 0.5, 0.0, 1.0, 0.5), (W, H), None),
              ("up x4", img, (0.25, 0.0, 0.0, 0.0, 0.25, 0.0), (4 * W, 4 * H), None)]
    _check_all(cases)
    out = _warp([img], [(0.0, 0.0, float(W), 0.0, 1.0, 0.0)], (3, H))[0]            # xin == W: zero fill
    assert np.array_equal(out, np.broadcast_to(TABLE[:, :1, None], out.shape))


def test_degenerate_sources_flips_and_scales():
    """1x1, 1xN and Nx1 sources; flips of odd and even widths; output widths 1, 255, 256, 257 (the grid's x tail); upsampling
    by 2 and 3, downsampling by 2; integer translations (dx == 0 exactly); mirrors through a negative a0."""
    g = np.random.default_rng(2)
    rnd = lambda W, H: g.integers(0, 256, (H, W, 3), dtype=np.uint8)  # noqa: E731
    cases = []
    for W, H in ((1, 1), (9, 1), (1, 9), (7, 6), (8, 6)):
        img = rnd(W, H)
        for flip in (False, True):
            cases.append((f"{W}x{H} flip={flip}", img, (W / 5, 0.0, 0.0, 0.0, H / 4, 0.0), (5, 4), flip))
            cases.append((f"{W}x{H} shear flip={flip}", img, (W / 6, 0.05, -0.3, -0.04, H / 5, 0.2), (6, 5), flip))
    img = rnd(40, 9)
    for Wo in (1, 255, 256, 257):
        cases.append((f"out width {Wo}", img, (40 / Wo, 0.0, 0.0, 0.0, 9 / 3, 0.0), (Wo, 3), Wo == 257))
    cases += [("up x2", img, (0.5, 0.0, 0.0, 0.0, 0.5, 0.0), (80, 18), None),
              ("up x3", img, (1 / 3, 0.0, 0.0, 0.0, 1 / 3, 0.0), (120, 27), None),
              ("down x2", img, (2.0, 0.0, 0.0, 0.0, 2.0, 0.0), (20, 5), None),
              ("translate (3, -2)", img, (1.0, 0.0, 3.0, 0.0, 1.0, -2.0), (40, 9), None),
              ("translate (-5, 1)", img, (1.0, 0.0, -5.0, 0.0, 1.0, 1.0), (40, 9), True),
              ("mirror", img, (-1.0, 0.0, 40.0, 0.0, 1.0, 0.0), (40, 9), None),
              ("mirror, scaled and sheared", img, (-0.75, 0.1, 41.3, 0.02, 0.9, -0.4), (56, 11), None)]
    _check_all(cases)


def test_everything_outside_is_normalized_zero():
    img = np.random.default_rng(3).integers(1, 256, (9, 40, 3), dtype=np.uint8)
    out = _warp([img, img], [(1.0, 0.0, -1000.0, 0.0, 1.0, 0.0), (1.0, 0.0, 0.0, 0.0, -1.0, -0.25)], (257, 5))
    assert np.array_equal(out, np.broadcast_to(TABLE[None, :, :1, None], out.shape))


def test_pitched_sources_on_the_device_and_the_host():
    """(H, W, 3) views into wider images (row pitch 3 * 53 > 3 * W): used in place on the device, uploaded from pageable and
    pinned host memory; and a ragged batch of them in one launch."""
    g = np.random.default_rng(4)
    big = g.integers(0, 256, (21, 53, 3), dtype=np.uint8)
    host = torch.from_numpy(big)
    views = [host.cuda()[:, 5:36], host[:, 5:36], host.pin_memory()[:, 17:52], host.cuda()[2:20, 0:53:1][:, 1:50]]
    assert views[0].stride(0) == 3 * 53 and views[1].stride(0) == 3 * 53
    datas = [(31 / 64, 0.02, 0.1, 0.0, 21 / 24, -0.1), (31 / 64, 0.0, 0.0, 0.0, 21 / 24, 0.0), (35 / 64, 0.0, 0.3, 0.01, 0.8, 0.0),
             (49 / 64, 0.0, 0.0, 0.0, 0.75, 0.0)]
    flips = [False, True, True, False]
    out = _warp(views, datas, (64, 24), flips)
    for i, v in enumerate(views):
        m = _mismatch(out[i], v.cpu().numpy(), datas[i], (64, 24), flips[i])
        assert m is None, (i, m)


def test_normalize_every_value():
    """Identity map (dx == dy == 0) of an image holding all 256 values in each channel: the device's fp32 normalisation of each
    is numpy's."""
    v = np.arange(256)
    img = np.stack([v, (v + 85) % 256, (255 - v)], -1).astype(np.uint8)[None]
    out = _warp([img], [(1.0, 0.0, 0.0, 0.0, 1.0, 0.0)], (256, 1))[0]
    assert np.array_equal(out, op.normalize(img))
    for c in range(3):
        assert np.array_equal(np.sort(out[c, 0]), TABLE[c])


def test_reference_transforms_on_the_kitti_sizes():
    """kitti_dataset.py's transforms on all four KITTI sizes -> 1280x384: the val centre crop, the clipped crop scales 0.6 and
    1.4 with random shifts, each with and without the flip; CUDA and CPU sources."""
    from monodetr_b200.preprocess import get_affine_transform
    imgs = op.synthetic_images(31, KITTI_SIZES)
    rng = np.random.default_rng(32)
    res = np.array([1280, 384])
    srcs, datas, flips, refs = [], [], [], []
    for i, (W, H) in enumerate(KITTI_SIZES):
        size = np.array([W, H], np.float64)
        for j, scale in enumerate((None, 0.6, 1.4)):
            center = size / 2
            if scale is not None:
                center = center + size * np.clip(rng.standard_normal(2) * 0.1, -0.2, 0.2)
            datas.append(get_affine_transform(center, size * (scale or 1.0), 0, res, inv=1)[1])
            flips.append(bool((i + j) % 2))
            srcs.append(torch.from_numpy(imgs[i]).cuda() if j % 2 else torch.from_numpy(imgs[i]))
            refs.append(imgs[i])
    out = _warp(srcs, datas, (1280, 384), flips)
    for k in range(len(srcs)):
        m = _mismatch(out[k], refs[k], datas[k], (1280, 384), flips[k])
        assert m is None, (k, m)


@pytest.fixture(scope="module")
def every_colour():
    """All 2**24 colours as a 4096x4096 image (W % 8 == 0: cv2's vector loop only) and a width-7 image (its scalar loop only)."""
    return [ph.every_colour(4096), ph.every_colour(7)]


def test_photometric_every_colour_through_both_loops(every_colour):
    """Every 8-bit colour under records at the ends of the sampled ranges, both contrast orders, all six permutations: grey
    pixels (diff == 0), ties of V with R and G, the hue wrap at 0 and 360, every sector boundary, values outside [0, 256)."""
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    pre = ImageBatchPreprocessor()
    dev = [torch.from_numpy(im).cuda() for im in every_colour]
    n_wrap, bad = 0, []
    for r, rec in enumerate(ph.EDGE_RECORDS):
        outs = pre.distort(dev, [rec, rec])
        for im, o in zip(every_colour, outs):
            want = ph.distort_float_rows(im, rec)
            n_wrap += int(((want < 0) | (want >= 256)).sum())
            got, want = o.cpu().numpy(), ph.to_u8(want)
            if not np.array_equal(got, want):
                i = np.argwhere((got != want).any(-1))[0]
                bad.append((r, im.shape[1], int((got != want).any(-1).sum()), tuple(im[i[0], i[1]]), tuple(got[i[0], i[1]]),
                            tuple(want[i[0], i[1]])))
    assert not bad, bad                                   # (record, width, pixels, first colour, device, oracle)
    assert n_wrap > 0


def test_reproducible_mode_gives_the_same_bits(every_colour):
    import monodetr_b200
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    imgs = [GOLD[f"{k}.img"] for k in range(int(GOLD["n"]))]
    datas = [GOLD[f"{k}.data"] for k in range(int(GOLD["n"]))]
    flips = [bool(k % 2) for k in range(len(imgs))]
    recs = [ph.EDGE_RECORDS[k % len(ph.EDGE_RECORDS)] for k in range(len(imgs))]
    srcs = [torch.from_numpy(im).cuda() for im in imgs]
    tail = [torch.from_numpy(every_colour[1]).cuda()]
    pre = ImageBatchPreprocessor(resolution=(140, 48))
    a = (pre(srcs, np.stack(datas).reshape(-1, 2, 3), flips, distort=recs), pre.distort(tail, ph.EDGE_RECORDS[3:4])[0])
    prev = monodetr_b200.set_deterministic(True)
    try:
        b = (pre(srcs, np.stack(datas).reshape(-1, 2, 3), flips, distort=recs), pre.distort(tail, ph.EDGE_RECORDS[3:4])[0])
    finally:
        monodetr_b200.set_deterministic(prev)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    for k, im in enumerate(imgs):                         # and those bits are the reference's
        assert _mismatch(a[0][k].cpu().numpy(), ph.distort(im, recs[k]), datas[k], (140, 48), flips[k]) is None, k
