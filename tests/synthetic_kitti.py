"""A small seeded KITTI folder for the loader tests, `tools/gen_golden_loader.py` and `tools/bench_loader.py`:

    root/ImageSets/{train,val,trainval,test}.txt
    root/training/{image_2/%06d.png, label_2/%06d.txt, calib/%06d.txt}
    root/testing/{image_2/%06d.png, calib/%06d.txt}

Images are KITTI's real sizes (oracle.preprocess.synthetic_images: a smooth field plus noise), labels hold Car, Pedestrian,
Cyclist and DontCare lines whose 2-d boxes are the clipped projections of their 3-d boxes, and the images alternate between two
calibrations.  Training ids are not contiguous (id != position in the split), train and val are disjoint.  The same arguments
always write the same bytes.
"""
import os

import numpy as np

KITTI_SIZES = ((1242, 375), (1224, 370), (1238, 374), (1241, 376))
CALIB_TEMPLATE = ("P0: {p0}\nP1: {p1}\nP2: {p2}\nP3: {p3}\nR0_rect: 9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 "
                  "9.999421e-01 -4.278459e-03 7.402527e-03 4.351614e-03 9.999631e-01\nTr_velo_to_cam: 7.533745e-03 -9.999714e-01 "
                  "-6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 -7.631618e-02 9.998621e-01 7.523790e-03 "
                  "1.480755e-02 -2.717806e-01\nTr_imu_to_velo: 9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 "
                  "9.998898e-01 -1.482298e-02 3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01\n")
# (f, cu, cv, P2 tx, ty, tz) of two KITTI drives
CAMERAS = ((7.215377e+02, 6.095593e+02, 1.728540e+02, 4.485728e+01, 2.163791e-01, 2.745884e-03),
           (7.070493e+02, 6.040814e+02, 1.805066e+02, 4.575831e+01, -3.454157e-01, 4.981016e-03))
DIMS = {"Car": (1.53, 1.63, 3.88), "Pedestrian": (1.76, 0.66, 0.84), "Cyclist": (1.74, 0.6, 1.76)}


def calib_text(cam):
    f, cu, cv, tx, ty, tz = CAMERAS[cam]

    def row(a, b, c):
        return " ".join("%e" % v for v in (f, 0, cu, a, 0, f, cv, b, 0, 0, 1, c))
    return CALIB_TEMPLATE.format(p0=row(0, 0, 0), p1=row(-3.875744e+02, 0, 0), p2=row(tx, ty, tz), p3=row(-3.395242e+02, 2.2, 2.7e-3))


def p2_of(cam):
    return np.array(calib_text(cam).splitlines()[2].split()[1:], np.float32).reshape(3, 4)


def label_line(g, P2, W, H):
    """One KITTI-like label line, or None when the object leaves the image."""
    cls = g.choice(["Car", "Car", "Car", "Pedestrian", "Cyclist", "DontCare"])
    if cls == "DontCare":
        x1, y1 = g.uniform(0, W - 80), g.uniform(150, 200)
        return f"DontCare -1 -1 -10 {x1:.2f} {y1:.2f} {x1 + g.uniform(10, 80):.2f} {y1 + g.uniform(5, 40):.2f} -1 -1 -1 -1000 -1000 -1000 -10"
    h, w, l = (d * g.uniform(0.85, 1.15) for d in DIMS[cls])
    z = g.uniform(4.0, 60.0)
    x = g.uniform(-0.4, 0.4) * z + g.uniform(-2, 2)
    y = 1.65 + g.uniform(-0.2, 0.2)
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
    trunc = min(max(1 - (x2 - x1) * (y2 - y1) / ((u.max() - u.min()) * (v.max() - v.min())), 0.0), 1.0)
    alpha = ry - np.arctan2(x, z)
    return (f"{cls} {trunc:.2f} {int(g.integers(0, 3))} {alpha:.2f} {x1:.2f} {y1:.2f} {x2:.2f} {y2:.2f} {h:.2f} {w:.2f} {l:.2f} "
            f"{x:.2f} {y:.2f} {z:.2f} {ry:.2f}")


def write_tree(root, n_train=14, n_val=6, n_test=6, seed=0, objects=(3, 12)):
    """Write the folder under `root`; returns {split: [ids]}."""
    from PIL import Image
    from oracle.preprocess import synthetic_images
    g = np.random.default_rng(seed)
    n = n_train + n_val
    ids = sorted(g.choice(3 * n, n, replace=False).tolist())
    order = g.permutation(n)
    splits = {"train": sorted(ids[i] for i in order[:n_train]), "val": sorted(ids[i] for i in order[n_train:]),
              "test": list(range(n_test))}
    splits["trainval"] = ids
    for sub in ("ImageSets", "training/image_2", "training/label_2", "training/calib", "testing/image_2", "testing/calib"):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
    for split, lst in splits.items():
        with open(os.path.join(root, "ImageSets", split + ".txt"), "w") as f:
            f.write("".join("%06d\n" % i for i in lst))
    for data, lst in (("training", ids), ("testing", splits["test"])):
        sizes = [KITTI_SIZES[int(g.integers(len(KITTI_SIZES)))] for _ in lst]
        for k, (img_id, im) in enumerate(zip(lst, synthetic_images(seed * 1000 + len(lst) + (data == "testing"), sizes))):
            d = os.path.join(root, data)
            Image.fromarray(im).save(os.path.join(d, "image_2", "%06d.png" % img_id))
            cam = img_id % 2
            with open(os.path.join(d, "calib", "%06d.txt" % img_id), "w") as f:
                f.write(calib_text(cam))
            if data == "training":
                W, H = sizes[k]
                lines, want = [], int(g.integers(*objects))
                while len(lines) < want:
                    ln = label_line(g, p2_of(cam), W, H)
                    if ln is not None:
                        lines.append(ln)
                with open(os.path.join(d, "label_2", "%06d.txt" % img_id), "w") as f:
                    f.write("".join(ln + "\n" for ln in lines))
    return splits


def set_random_seed(seed):
    """lib/helpers/utils_helper.py:18-26's generator seeding (the cudnn flags aside)."""
    import random

    import torch
    random.seed(seed)
    np.random.seed(seed ** 2)
    torch.manual_seed(seed ** 3)
    if torch.cuda.is_available():
        torch.cuda.manual_seed_all(seed ** 4)
