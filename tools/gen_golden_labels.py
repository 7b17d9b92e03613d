"""Generate tests/golden/labels.npz from the UNMODIFIED reference dataset (CPU only).

    python tools/gen_golden_labels.py

Needs the reference checkout (MONODETR_REFERENCE, default /root/reference), cv2, yaml and numba (the dataset module imports the
KITTI evaluation; its CUDA kernel is never run here, NUMBA_ENABLE_CUDASIM=1 is set if absent).  No reference file is edited or
copied.  A synthetic KITTI folder is written to a temporary directory: N_IMG images of KITTI sizes (oracle.preprocess
.synthetic_images), two sets of calibration and label files whose lines cover every class the encoder tells apart (the three
classes, Van, Truck, Tram, Person_sitting, Misc, DontCare), depths below 2 and above 65, 3-d centres projected outside the
frame, boxes that do not contain the projected centre (negative l / r / t / b), truncated and occluded objects (mask 0 and
'UnKnown' levels), and one file with more than 50 lines.  Then `KITTI_Dataset(split, cfg).__getitem__(i)` runs after
np.random.seed for every image under each configuration variant (VARIANTS below; the shipped configs/monodetr.yaml is the base).

Contents:
  label.{i} / calib.{i}: the file texts; sizes (N, 2) [W, H]; img_ids (N,); img_seed.
  parsed.*: the reference's Object3d fields of every line (cls, f64 (trunc, occ, alpha, h, w, l, ry), box2d f32, pos f32, level)
            and Calibration.P2 per image, counts per image.
  {v}.cfg (json), {v}.split, {v}.resolution, {v}.seeds; {v}.<target key> (N, 50, ...) as __getitem__ returns them;
  {v}.P2 (N, 3, 4); {v}.info_* ; the draws replayed through the reference's own calls with the same seed: {v}.flip, {v}.crop_scale,
  {v}.center, {v}.trans / {v}.trans_inv (cv2), and {v}.state_* = np.random.get_state() after __getitem__.
  e2e.u8 (n, H, W, 3): the warped image of variant e2e, recovered exactly from the normalised output (the 256-entry inverse of
  the normalisation, asserted injective).

Every decision the encoder takes on a kept object (depth range, centre inside the frame, l / r / t / b sign) is asserted to lie more
than 1e-6 from its threshold and every heading angle more than 1e-5 rad from a bin edge, so a 1-ulp difference in an fp64 dot
product (OpenBLAS may contract to FMA) or in float32 arctan2 cannot move the reference's result across one.
"""
import copy
import importlib
import json
import os
import sys
import tempfile
import types

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")

import numpy as np  # noqa: E402
from PIL import Image  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
REF = os.environ.get("MONODETR_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "labels.npz")
from oracle import labels as ol  # noqa: E402
from oracle.preprocess import normalize, synthetic_images  # noqa: E402

IMG_SEED = 70
SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1242, 375), (1224, 370)]
E2E_RES = (320, 96)
E2E_N = 4
ALL3 = ["Pedestrian", "Car", "Cyclist"]
BIG_CROP = {"random_crop": 0.9, "scale": 0.4, "shift": 0.1}
VARIANTS = [
    ("shipped", "train", {}),
    ("all3", "train", {"writelist": ALL3}),
    ("clip2d", "train", {"writelist": ALL3, "clip_2d": True}),
    ("inverse", "train", {"writelist": ALL3, "depth_scale": "inverse", **BIG_CROP}),
    ("none", "train", {"writelist": ALL3, "depth_scale": "none", **BIG_CROP}),
    ("meanshape", "train", {"writelist": ALL3, "meanshape": True}),
    ("val", "val", {"writelist": ALL3}),
    ("e2e", "train", {}),
]

CALIBS = [
    """P0: 7.215377e+02 0.000000e+00 6.095593e+02 0.000000e+00 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P1: 7.215377e+02 0.000000e+00 6.095593e+02 -3.875744e+02 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P2: 7.215377e+02 0.000000e+00 6.095593e+02 4.485728e+01 0.000000e+00 7.215377e+02 1.728540e+02 2.163791e-01 0.000000e+00 0.000000e+00 1.000000e+00 2.745884e-03
P3: 7.215377e+02 0.000000e+00 6.095593e+02 -3.395242e+02 0.000000e+00 7.215377e+02 1.728540e+02 2.199936e+00 0.000000e+00 0.000000e+00 1.000000e+00 2.729905e-03
R0_rect: 9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 4.351614e-03 9.999631e-01
Tr_velo_to_cam: 7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 -7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01
Tr_imu_to_velo: 9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 9.998898e-01 -1.482298e-02 3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01
""",
    """P0: 7.070493e+02 0.000000e+00 6.040814e+02 0.000000e+00 0.000000e+00 7.070493e+02 1.805066e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P1: 7.070493e+02 0.000000e+00 6.040814e+02 -3.797842e+02 0.000000e+00 7.070493e+02 1.805066e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P2: 7.070493e+02 0.000000e+00 6.040814e+02 4.575831e+01 0.000000e+00 7.070493e+02 1.805066e+02 -3.454157e-01 0.000000e+00 0.000000e+00 1.000000e+00 4.981016e-03
P3: 7.070493e+02 0.000000e+00 6.040814e+02 -3.341081e+02 0.000000e+00 7.070493e+02 1.805066e+02 2.330660e+00 0.000000e+00 0.000000e+00 1.000000e+00 3.201153e-03
R0_rect: 9.999454e-01 7.259129e-03 -7.519551e-03 -7.292213e-03 9.999638e-01 -4.381729e-03 7.487471e-03 4.436324e-03 9.999621e-01
Tr_velo_to_cam: 7.967514e-03 -9.999679e-01 -8.462264e-04 -1.377769e-02 -2.771053e-03 8.241710e-04 -9.999958e-01 -5.542117e-02 9.999644e-01 7.969825e-03 -2.764397e-03 -2.918589e-01
Tr_imu_to_velo: 9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 9.998898e-01 -1.482298e-02 3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01
""",
]

# hand-written lines: (cls trunc occ alpha x1 y1 x2 y2 h w l x y z ry)
EDGE_LINES = [
    "Car 0.00 0 -1.58 587.01 173.33 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59",
    "Pedestrian 0.00 0 0.21 712.40 143.00 810.73 307.92 1.89 0.48 1.20 1.84 1.47 8.41 0.01",
    "Cyclist 0.00 1 -2.13 300.10 160.30 360.80 240.90 1.72 0.61 1.78 -6.30 1.62 14.20 -2.54",
    "Van 0.00 0 -1.55 580.05 160.70 620.44 198.58 2.27 1.80 4.93 -0.51 1.79 31.34 -1.57",
    "Truck 0.00 0 1.20 420.00 120.00 540.00 230.00 3.20 2.60 9.80 -8.10 1.90 32.00 0.95",
    "Tram 0.00 0 -1.40 640.00 100.00 780.00 220.00 3.50 2.60 16.00 3.80 1.60 35.00 -1.30",
    "Person_sitting 0.00 0 2.80 820.00 170.00 860.00 240.00 1.20 0.60 0.80 5.10 1.55 16.00 3.10",
    "Misc 0.00 0 -1.90 540.00 170.00 580.00 200.00 1.40 1.00 2.00 -2.10 1.70 40.00 -1.95",
    "DontCare -1 -1 -10 503.89 169.71 590.61 190.13 -1 -1 -1 -1000 -1000 -1000 -10",
    "Car 0.00 0 0.50 100.00 170.00 300.00 300.00 1.50 1.60 3.90 -1.20 1.60 1.50 0.50",          # z < 2
    "Car 0.00 0 -1.60 600.00 172.00 612.00 181.00 1.50 1.60 3.90 0.50 1.60 70.00 -1.59",       # z > 65
    "Car 0.00 0 1.00 0.00 160.00 60.00 260.00 1.50 1.60 3.90 -30.00 1.60 10.00 -0.20",        # centre left of the frame
    "Car 0.00 0 -0.80 1180.00 150.00 1241.00 300.00 1.50 1.60 3.90 25.00 1.60 9.00 0.40",     # centre right of the frame
    "Car 0.00 0 -1.57 700.00 170.00 800.00 220.00 1.50 1.60 3.90 0.00 1.60 20.00 -1.57",      # box right of the centre: l < 0
    "Car 0.00 0 -1.57 560.00 120.00 660.00 150.00 1.50 1.60 3.90 0.00 1.60 22.00 -1.57",      # box above the centre: b < 0
    "Car 0.60 0 -1.20 650.00 170.00 720.00 220.00 1.50 1.60 3.90 2.00 1.60 25.00 -1.12",      # truncation > 0.5: UnKnown
    "Car 0.00 3 -1.20 500.00 170.00 570.00 220.00 1.50 1.60 3.90 -2.00 1.60 25.00 -1.28",     # occlusion 3: UnKnown
    "Car 0.00 0 -1.58 600.00 175.00 618.00 190.00 1.50 1.60 3.90 0.00 1.60 55.00 -1.58",      # height < 25: UnKnown
    "Car -1 3 -1.40 620.00 165.00 700.00 215.00 1.50 1.60 3.90 1.50 1.60 24.00 -1.34",        # level DontCare, occluded: mask 0
    "Car 0.40 2 -1.70 520.00 165.00 600.00 215.00 1.50 1.60 3.90 -1.50 1.60 24.00 -1.76",     # Hard, mask 1
]


def kitti_object(g, P2, W, H):
    """One random KITTI-like label line whose box is the clipped projection of its 3-d box, or None if it leaves the image."""
    cls = g.choice(["Car", "Car", "Car", "Car", "Pedestrian", "Cyclist", "Van", "DontCare", "Misc"])
    if cls == "DontCare":
        x1, y1 = g.uniform(0, W - 80), g.uniform(150, 200)
        return f"DontCare -1 -1 -10 {x1:.2f} {y1:.2f} {x1 + g.uniform(10, 80):.2f} {y1 + g.uniform(5, 40):.2f} -1 -1 -1 -1000 -1000 -1000 -10"
    dims = {"Car": (1.53, 1.63, 3.88), "Van": (2.2, 1.9, 5.0), "Pedestrian": (1.76, 0.66, 0.84), "Cyclist": (1.74, 0.6, 1.76),
            "Misc": (1.9, 1.5, 3.6)}[cls]
    h, w, l = (d * g.uniform(0.85, 1.15) for d in dims)
    z = g.uniform(3.0, 62.0)
    x = g.uniform(-0.45, 0.45) * z + g.uniform(-3, 3)
    y = 1.65 + g.uniform(-0.25, 0.25)
    ry = g.uniform(-np.pi, np.pi)
    c, s = np.cos(ry), np.sin(ry)
    xs = np.array([l, l, -l, -l, l, l, -l, -l]) / 2
    ys = np.array([0, 0, 0, 0, -h, -h, -h, -h])
    zs = np.array([w, -w, -w, w, w, -w, -w, w]) / 2
    pts = np.stack([c * xs + s * zs + x, ys + y, -s * xs + c * zs + z, np.ones(8)])
    if (pts[2] < 0.5).any():
        return None
    uvw = P2.astype(np.float64) @ pts
    u, v = uvw[0] / uvw[2], uvw[1] / uvw[2]
    x1, y1, x2, y2 = max(u.min(), 0), max(v.min(), 0), min(u.max(), W - 1), min(v.max(), H - 1)
    if x2 - x1 < 2 or y2 - y1 < 2:
        return None
    full = (u.max() - u.min()) * (v.max() - v.min())
    trunc = min(max(1 - (x2 - x1) * (y2 - y1) / full, 0.0), 1.0)
    occ = int(g.integers(0, 3))
    alpha = ry - np.arctan2(x, z)
    return (f"{cls} {trunc:.2f} {occ} {alpha:.2f} {x1:.2f} {y1:.2f} {x2:.2f} {y2:.2f} {h:.2f} {w:.2f} {l:.2f} {x:.2f} {y:.2f} "
            f"{z:.2f} {ry:.2f}")


def label_files(g):
    """Per image a list of lines: image 0 the hand-written cases, image 3 more than 50 lines, the rest random."""
    files = []
    for i, (W, H) in enumerate(SIZES):
        P2 = np.array(CALIBS[i % 2].splitlines()[2].split()[1:], np.float32).reshape(3, 4)
        n = {0: 0, 3: 55}.get(i, int(g.integers(8, 20)))
        lines = list(EDGE_LINES) if i == 0 else []
        while len(lines) < n:
            ln = kitti_object(g, P2, W, H)
            if ln is not None:
                lines.append(ln)
        files.append(lines)
    return files


def state_arrays():
    _, keys, pos, has_gauss, gauss = np.random.get_state()
    return keys, pos, np.array([has_gauss, gauss], np.float64)


def replay_draws(ds, seed, img_size, PhotometricDistort, get_affine_transform):
    """kitti_dataset.py:130-154 through the reference's own calls (the distortion on a dummy image)."""
    np.random.seed(seed)
    center = np.array(img_size) / 2
    crop_size, crop_scale, flip = img_size, 1, False
    if ds.data_augmentation:
        if ds.aug_pd:
            PhotometricDistort()(np.zeros((1, 1, 3), np.float32))
        flip = np.random.random() < ds.random_flip
        if ds.aug_crop and np.random.random() < ds.random_crop:
            crop_scale = np.clip(np.random.randn() * ds.scale + 1, 1 - ds.scale, 1 + ds.scale)
            crop_size = img_size * crop_scale
            center[0] += img_size[0] * np.clip(np.random.randn() * ds.shift, -2 * ds.shift, 2 * ds.shift)
            center[1] += img_size[1] * np.clip(np.random.randn() * ds.shift, -2 * ds.shift, 2 * ds.shift)
    trans, trans_inv = get_affine_transform(center, crop_size, 0, ds.resolution, inv=1)
    return bool(flip), float(crop_scale), center, trans, trans_inv


def main():
    import yaml
    if REF not in sys.path:
        sys.path.insert(0, REF)
    try:
        import skimage.io  # noqa: F401
    except ImportError:                                   # kitti_common.py imports skimage.io; nothing here calls it
        sk = types.ModuleType("skimage")
        sk.io = types.ModuleType("skimage.io")
        sys.modules["skimage"], sys.modules["skimage.io"] = sk, sk.io
    kd = importlib.import_module("lib.datasets.kitti.kitti_dataset")
    ku = importlib.import_module("lib.datasets.kitti.kitti_utils")
    from lib.datasets.kitti.pd import PhotometricDistort
    with open(os.path.join(REF, "configs", "monodetr.yaml")) as f:
        base_cfg = yaml.load(f, Loader=yaml.Loader)["dataset"]
    out = {"sizes": np.array(SIZES), "img_ids": np.arange(len(SIZES)), "img_seed": np.array(IMG_SEED)}
    files = label_files(np.random.default_rng(5))
    imgs = synthetic_images(IMG_SEED, SIZES)
    table = normalize(np.tile(np.arange(256, dtype=np.uint8)[None, :, None], (1, 1, 3)))[:, 0, :]     # (3, 256)
    assert all(np.unique(table[c]).size == 256 for c in range(3)) and (np.diff(table, axis=1) > 0).all()
    n_margin, covered = 0, set()
    with tempfile.TemporaryDirectory() as d:
        for sub in ("ImageSets", "training/image_2", "training/calib", "training/label_2"):
            os.makedirs(os.path.join(d, sub))
        ids = "".join("%06d\n" % i for i in range(len(SIZES)))
        for split in ("train", "val"):
            open(os.path.join(d, "ImageSets", split + ".txt"), "w").write(ids)
        parsed = {"cls": [], "f64": [], "box2d": [], "pos": [], "level": [], "count": [], "P2": []}
        for i, (im, lines) in enumerate(zip(imgs, files)):
            Image.fromarray(im).save(os.path.join(d, "training", "image_2", "%06d.png" % i))
            text = "".join(ln + "\n" for ln in lines)
            open(os.path.join(d, "training", "label_2", "%06d.txt" % i), "w").write(text)
            open(os.path.join(d, "training", "calib", "%06d.txt" % i), "w").write(CALIBS[i % 2])
            out[f"label.{i}"], out[f"calib.{i}"] = np.array(text), np.array(CALIBS[i % 2])
            objs = ku.get_objects_from_label(os.path.join(d, "training", "label_2", "%06d.txt" % i))
            for o in objs:
                parsed["cls"].append(o.cls_type)
                parsed["f64"].append([o.trucation, o.occlusion, o.alpha, o.h, o.w, o.l, o.ry])
                parsed["box2d"].append(o.box2d)
                parsed["pos"].append(o.pos)
                parsed["level"].append(o.level_str)
            parsed["count"].append(len(objs))
            parsed["P2"].append(ku.Calibration(os.path.join(d, "training", "calib", "%06d.txt" % i)).P2)
        for k, v in parsed.items():
            out[f"parsed.{k}"] = np.array(v)
        assert out["parsed.box2d"].dtype == np.float32 and out["parsed.pos"].dtype == np.float32
        for name, split, over in VARIANTS:
            cfg = dict(copy.deepcopy(base_cfg), root_dir=d, **copy.deepcopy(over))
            ds = kd.KITTI_Dataset(split, cfg)
            n = E2E_N if name == "e2e" else len(SIZES)
            if name == "e2e":
                ds.resolution = np.array(E2E_RES)
            out[f"{name}.cfg"], out[f"{name}.split"] = np.array(json.dumps(over)), np.array(split)
            out[f"{name}.resolution"] = np.array(ds.resolution)
            assert sorted(ds.writelist) == sorted(over.get("writelist", ["Car"]))
            seeds = [1000 * (VARIANTS.index((name, split, over)) + 1) + 7 * i for i in range(n)]
            rows = {k: [] for k in ol.KEYS + ("P2", "flip", "crop_scale", "center", "trans", "trans_inv", "state_keys",
                                               "state_pos", "state_gauss", "info_img_id", "info_img_size", "info_ratio", "u8")}
            for i, seed in enumerate(seeds):
                np.random.seed(seed)
                inputs, P2, targets, info = ds[i]
                keys, pos, gauss = state_arrays()
                flip, crop_scale, center, trans, trans_inv = replay_draws(ds, seed, np.array(SIZES[i]), PhotometricDistort,
                                                                          ku.get_affine_transform)
                assert np.array_equal(targets["img_size"], SIZES[i])
                for k in ol.KEYS:
                    rows[k].append(targets[k])
                for k, v in (("P2", P2), ("flip", flip), ("crop_scale", crop_scale), ("center", center), ("trans", trans),
                             ("trans_inv", trans_inv), ("state_keys", keys), ("state_pos", pos), ("state_gauss", gauss),
                             ("info_img_id", info["img_id"]), ("info_img_size", info["img_size"]),
                             ("info_ratio", info["bbox_downsample_ratio"])):
                    rows[k].append(v)
                if name == "e2e":
                    u8 = np.stack([np.searchsorted(table[c], inputs[c]) for c in range(3)], -1).astype(np.uint8)
                    assert np.array_equal(normalize(u8), inputs)
                    rows["u8"].append(u8)
                covered.add((name, flip, crop_scale != 1))
                # margins of every decision the encoder takes, on the oracle's intermediate values
                offsets, recs, P2s = ol.gold_bank(out)
                margins = []
                ol.encode_image(recs[offsets[i]:offsets[i + 1]], P2s[i], SIZES[i], flip, crop_scale, trans, margins=margins,
                                **ol.gold_config(out, name))
                for what, m in margins:
                    assert abs(m) > (1e-5 if what == "bin" else 1e-6), (name, i, what, m)
                n_margin += len(margins)
            for k, v in rows.items():
                if v:
                    out[f"{name}.{k}"] = np.array(v)
            out[f"{name}.seeds"] = np.array(seeds)
            print(name, "flips", out[f"{name}.flip"].astype(int).tolist(), "crop_scale",
                  np.round(out[f"{name}.crop_scale"], 4).tolist(), "kept", int(out[f"{name}.mask_2d"].sum()),
                  "labelled", int((out[f"{name}.size_2d"][..., 0] != 0).sum()))
    both = {(f, c) for (_, f, c) in covered}
    assert both == {(False, False), (False, True), (True, False), (True, True)}, both       # flip x crop all met
    print("decisions checked for margin:", n_margin)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
