"""CPU restatement (numpy) of the image half of the reference dataset's __getitem__ -- TEST INFRASTRUCTURE ONLY.

  warp_affine_bilinear   PIL Image.transform(size, Image.AFFINE, data, resample=Image.BILINEAR) as called at
                         lib/datasets/kitti/kitti_dataset.py:153-156 (Pillow's Geometry.c: pixel-centre mapping, zero fill outside,
                         clamped neighbours, fp64 interpolation truncated to 8 bits)
  normalize              kitti_dataset.py:159-161   float32 / 255, (x - mean) / std, HWC -> CHW
  flip                   kitti_dataset.py:140-142   Image.FLIP_LEFT_RIGHT

Pinned against Pillow itself and the reference's get_affine_transform (cv2) by tests/golden/preprocess.npz
(tools/gen_golden_preprocess.py) -- tests/test_oracle_preprocess.py; and against live Pillow on inputs constructed to sit on a
coordinate floor or an 8-bit truncation edge (tests/golden/preprocess_edges.npz) -- tests/test_preprocess_edges_host_logic.py.
numpy rounds every product before its sum, as Pillow's C code does.
"""
import numpy as np

MEAN = np.array([0.485, 0.456, 0.406], dtype=np.float32)
STD = np.array([0.229, 0.224, 0.225], dtype=np.float32)


def warp_affine_bilinear(img, data, out_wh):
    """img (H, W, 3) uint8, data = (a, b, c, d, e, f), out_wh = (W_out, H_out) -> (H_out, W_out, 3) uint8."""
    H, W, _ = img.shape
    Wo, Ho = out_wh
    a, b, c, d, e, f = (float(v) for v in data)
    xs, ys = np.meshgrid(np.arange(Wo, dtype=np.float64) + 0.5, np.arange(Ho, dtype=np.float64) + 0.5)
    xin = a * xs + b * ys + c
    yin = d * xs + e * ys + f
    inside = ~((xin < 0.0) | (xin >= W) | (yin < 0.0) | (yin >= H))
    xin, yin = xin - 0.5, yin - 0.5
    xf, yf = np.floor(xin), np.floor(yin)
    dx, dy = (xin - xf)[..., None], (yin - yf)[..., None]
    xf, yf = xf.astype(np.int64), yf.astype(np.int64)
    x0, x1 = np.clip(xf, 0, W - 1), np.clip(xf + 1, 0, W - 1)
    y0 = np.clip(yf, 0, H - 1)
    has_y1 = ((yf + 1 >= 0) & (yf + 1 < H))[..., None]
    y1 = np.clip(yf + 1, 0, H - 1)
    im = img.astype(np.float64)
    v1 = im[y0, x0] + (im[y0, x1] - im[y0, x0]) * dx
    v2 = np.where(has_y1, im[y1, x0] + (im[y1, x1] - im[y1, x0]) * dx, v1)
    out = (v1 + (v2 - v1) * dy).astype(np.uint8)                # C cast: truncation
    out[~inside] = 0
    return out


def normalize(img_u8, mean=MEAN, std=STD):
    x = img_u8.astype(np.float32) / 255.0
    return ((x - mean) / std).transpose(2, 0, 1)


def preprocess(img, data, out_wh, flip=False):
    if flip:
        img = img[:, ::-1]
    return normalize(warp_affine_bilinear(img, data, out_wh))


def synthetic_images(seed, sizes):
    """Smooth-ish random RGB images (low-frequency field + noise) of the given (W, H) sizes."""
    g = np.random.default_rng(seed)
    out = []
    for (W, H) in sizes:
        yy, xx = np.mgrid[0:H, 0:W]
        base = 128 + 90 * np.sin(xx[..., None] / (7.0 + np.arange(3)) + yy[..., None] / (5.0 + np.arange(3)))
        out.append(np.clip(base + g.normal(0, 25, (H, W, 3)), 0, 255).astype(np.uint8))
    return out
