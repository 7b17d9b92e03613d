"""Host half of tests/test_preprocess_edges_gpu.py: the constructed warp cases really separate FMA-contracted arithmetic from
Pillow's (so the device test would catch a contracted kernel), the photometric oracle equals live cv2 on every 8-bit colour,
and the sm_90a SASS of the warp kernel contains no DFMA."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
from PIL import Image

import warp_fp64_model as wm
from oracle import photometric as ph
from oracle import preprocess as op

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "preprocess_edges.npz"))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _case(k):
    g = lambda name: GOLD[f"{k}.{name}"]  # noqa: E731
    return str(g("kind")), g("img"), g("data"), tuple(int(v) for v in g("out_wh")), tuple(int(v) for v in g("pixel"))


def test_fused_form_disagrees_with_pillow_and_separate_form_agrees():
    signs = set()
    for k in range(int(GOLD["n"])):
        kind, img, data, out_wh, (x, y, c) = _case(k)
        pil = np.array(Image.fromarray(img).transform(out_wh, Image.AFFINE, data=tuple(float(v) for v in data),
                                                      resample=Image.BILINEAR))
        assert np.array_equal(op.warp_affine_bilinear(img, data, out_wh), pil), k
        sep, fused = wm.sample(img, data, x, y, False), wm.sample(img, data, x, y, True)
        assert sep == tuple(pil[y, x]) and sep[c] == int(GOLD[f"{k}.pillow"]), k
        assert fused[c] != sep[c] and fused[c] == int(GOLD[f"{k}.fused"]), k
        (xs, ys), (xq, yq) = wm.coords(data, x, y, False), wm.coords(data, x, y, True)
        if kind == "trunc":                       # same coordinates: the interpolation alone decides
            assert (xs, ys) == (xq, yq), k
            signs.add(fused[c] > sep[c])
        else:                                     # the floor of the sheared coordinate moves by one source pixel
            s, q = (xs, xq) if kind == "floor_x" else (ys, yq)
            assert np.floor(s - 0.5) != np.floor(q - 0.5), k
    assert signs == {False, True}
    x, y, c = (int(v) for v in GOLD["0.pixel"])
    assert (int(GOLD["0.pillow"]), int(GOLD["0.fused"])) == (49, 50) and (x, y) == (130, 10)
    assert np.array_equal(GOLD["0.img"][0, :, 0], 10 * np.arange(16)) and tuple(GOLD["0.data"]) == (1 / 30, 0.1, 0.1, 0, 1, 0)


def test_separate_form_is_the_oracle_on_random_pixels():
    """The scalar model's separate form is the numpy oracle pixel for pixel (a sheared, flipped, partly outside map)."""
    g = np.random.default_rng(0)
    img = g.integers(0, 256, (11, 13, 3), dtype=np.uint8)
    data = (0.37, -0.11, 2.3, 0.07, 0.61, -1.2)
    want = op.warp_affine_bilinear(img, data, (40, 22))
    for y in range(22):
        for x in range(40):
            assert wm.sample(img, data, x, y, False) == tuple(want[y, x]), (x, y)


# ---- photometric: the oracle against live cv2 ---------------------------------------------------------------------------------

def _cv2_dispatches_8_wide_hsv(cv2):
    """cv2 converts float BGR<->HSV in AVX2 (8-lane) code when AVX2 is a dispatched or baseline feature and the CPU has it; the
    oracle's vector / scalar split (ph.SIMD_WIDTH) is that build's."""
    feats = cv2.getCPUFeaturesLine().split()
    return cv2.useOptimized() and any(f.lstrip("*") == "AVX2" for f in feats) and cv2.checkHardwareSupport(13)   # CV_CPU_AVX2


def _cv2_distort(cv2, img, p):
    """The distortion with cv2.cvtColor for both colour conversions and numpy float32 for the rest (oracle/photometric.py's steps)."""
    x = img.astype(np.float32) + np.float32(p.brightness)
    if not p.contrast_last:
        x = x * np.float32(p.contrast)
    hsv = cv2.cvtColor(x, cv2.COLOR_BGR2HSV)
    hsv[..., 1] *= np.float32(p.saturation)
    hsv[..., 0] += np.float32(p.hue)
    hsv[..., 0][hsv[..., 0] > 360.0] -= 360.0
    hsv[..., 0][hsv[..., 0] < 0.0] += 360.0
    x = cv2.cvtColor(hsv, cv2.COLOR_HSV2BGR)
    if p.contrast_last:
        x = x * np.float32(p.contrast)
    return x[..., list(ph.PERMS[p.perm])]


@pytest.mark.parametrize("width", [4096, 7])
def test_oracle_matches_live_cv2_on_every_colour(width):
    cv2 = pytest.importorskip("cv2")
    if not _cv2_dispatches_8_wide_hsv(cv2):
        pytest.skip("this cv2 does not convert float HSV 8 pixels at a time")
    img = ph.every_colour(width)
    for rec in (ph.EDGE_RECORDS[0], ph.EDGE_RECORDS[3], ph.EDGE_RECORDS[-1]):
        want = np.ascontiguousarray(_cv2_distort(cv2, img, rec))
        got = ph.distort_float_rows(img, rec)
        assert np.array_equal(got.view(np.int32), want.view(np.int32)), (width, rec, int((got != want).any(-1).sum()))


# ---- the warp kernel's SASS ---------------------------------------------------------------------------------------------------

def test_warp_kernel_sass_has_no_dfma(tmp_path):
    """nvcc contracts `a * b + c` in fp64 into DFMA unless told otherwise; Pillow rounds the product first."""
    cuobjdump = os.path.join(os.path.dirname(NVCC), "cuobjdump")
    if not (shutil.which(NVCC) and shutil.which(cuobjdump)):
        pytest.skip("no nvcc / cuobjdump")
    cubin = str(tmp_path / "preprocess.cubin")
    subprocess.run([NVCC, "-cubin", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--expt-relaxed-constexpr",
                    "-o", cubin, os.path.join(ROOT, "monodetr_b200", "csrc", "preprocess.cu")], check=True, capture_output=True)
    sass = subprocess.run([cuobjdump, "-sass", cubin], check=True, capture_output=True, text=True).stdout
    funcs = {m.group(1): body for m in re.finditer(r"Function : (\S+)\n(.*?)(?=\n\s*Function :|\Z)", sass, re.S) for body in
             [m.group(2)]}
    warp = [body for name, body in funcs.items() if "warp_affine_normalize_kernel" in name]
    assert len(warp) == 1, list(funcs)
    assert "DMUL" in warp[0] and "F2I.F64.FLOOR" in warp[0]          # the fp64 arithmetic is there, and unfused
    assert "DFMA" not in warp[0], [ln.strip() for ln in warp[0].splitlines() if "DFMA" in ln]
