"""Generate tests/golden/photometric.npz from the UNMODIFIED reference photometric distortion (CPU only).

    python tools/gen_golden_photometric.py

Needs the reference checkout (MONODETR_REFERENCE, default /root/reference), cv2 and numba (the reference dataset module imports
its KITTI evaluation; its one CUDA kernel is never run here, NUMBA_ENABLE_CUDASIM=1 is set if absent).  No reference file is
edited or copied: lib/datasets/kitti/pd.py is loaded in place and its module-level `random` (numpy.random) is wrapped by a proxy
that forwards every call and logs the draw, so that each case's record is read off the reference's own draws.

The bits of the reference depend on cv2's CPU dispatch (cvtColor on float32); this fixture was produced with cv2 4.13 running its
AVX2 + FMA3 (AVX-512 capable host) code and numpy 2.3 on x86-64.

Contents:
  sizes (N, 2) [W, H], seeds (N,): case i distorts oracle.preprocess.synthetic_images(IMG_SEED + i, [sizes[i]])[0] after
  np.random.seed(seeds[i]); {i}.record = (brightness, contrast, saturation, hue, contrast_last, perm) read off the draws (a
  skipped step holds its neutral value), {i}.u8 = pd(img.astype(float32)).astype(uint8), {i}.state_* = np.random.get_state()
  after the call.  The widths cover every residue mod 8 (cv2's row tail); the seeds are picked so that the cases cover both
  branch orders, each optional step on and off, and all six channel permutations.
  e2e.*: KITTI_Dataset('train', cfg).__getitem__(0) with the shipped configs/monodetr.yaml (aug_pd, random_flip, aug_crop) on a
  one-image KITTI folder written to a temporary directory, after np.random.seed(e2e.seeds[k]); the output resolution is set to
  E2E_RES on the dataset object to keep the fixture small.  Stored as the warped uint8 image, recovered from the normalised float
  output through the normalisation's 256-entry inverse (asserted injective and exact), with the flip / crop draws replayed from
  the same seed through the reference's own calls and the state after.
"""
import importlib.util
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
OUT = os.path.join(ROOT, "tests", "golden", "photometric.npz")
from oracle.preprocess import normalize, synthetic_images  # noqa: E402

IMG_SEED = 40
WIDTHS = [1, 3, 5, 8, 9, 10, 11, 12, 13, 14, 15, 16, 17, 21, 30, 46, 63, 100, 7, 2]
E2E_SIZE = (1242, 375)
E2E_RES = (640, 192)
E2E_SEEDS = (3, 10)


class _LoggingRandom:
    """numpy.random as pd.py sees it, with a log of (name, result)."""

    def __init__(self):
        self.log = []

    def randint(self, *a):
        v = np.random.randint(*a)
        self.log.append(("randint", v))
        return v

    def uniform(self, *a):
        v = np.random.uniform(*a)
        self.log.append(("uniform", v))
        return v


def load_pd():
    spec = importlib.util.spec_from_file_location("ref_pd", os.path.join(REF, "lib", "datasets", "kitti", "pd.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def record_from_log(log):
    """The six record fields from the draw log of one PhotometricDistort.__call__ (pd.py:389-397, 114-195)."""
    it = iter(log)
    nxt = lambda: next(it)[1]                                                     # noqa: E731
    rec = [0.0, 1.0, 1.0, 0.0, 0, 0]
    if nxt():
        rec[0] = nxt()
    first = nxt()
    rec[4] = 0 if first else 1
    if first and nxt():
        rec[1] = nxt()
    if nxt():
        rec[2] = nxt()
    if nxt():
        rec[3] = nxt()
    if not first and nxt():
        rec[1] = nxt()
    if nxt():
        rec[5] = nxt()
    assert next(it, None) is None
    return rec


def features(rec):
    return {("order", rec[4]), ("bright", rec[0] != 0), ("contrast", rec[1] != 1, rec[4]), ("sat", rec[2] != 1),
            ("hue", rec[3] != 0), ("perm", rec[5])}


def state_arrays(prefix, out):
    name, keys, pos, has_gauss, gauss = np.random.get_state()
    out[prefix + "state_keys"], out[prefix + "state_pos"] = keys, np.array(pos)
    out[prefix + "state_gauss"] = np.array([has_gauss, gauss], np.float64)


def gen_cases(out):
    pdm = load_pd()
    logger = _LoggingRandom()
    pdm.random = logger
    pd = pdm.PhotometricDistort()
    covered, seeds, sizes, n_wrap = set(), [], [], 0
    for i, W in enumerate(WIDTHS):
        H = 6 if W > 20 else 9
        img = synthetic_images(IMG_SEED + i, [(W, H)])[0]
        seed = 1000 * i
        while True:                                       # the first seed that covers something new (or any, once all is)
            np.random.seed(seed)
            logger.log = []
            pd(np.zeros((1, 1, 3), np.float32))
            f = features(record_from_log(logger.log))
            if not f <= covered or len(covered) >= 18:
                break
            seed += 1
        covered |= f
        np.random.seed(seed)
        logger.log = []
        res = pd(img.astype(np.float32))
        out[f"{i}.record"] = np.array(record_from_log(logger.log), np.float64)
        out[f"{i}.u8"] = res.astype(np.uint8)
        n_wrap += int(((res < 0) | (res >= 256)).sum())
        state_arrays(f"{i}.", out)
        seeds.append(seed)
        sizes.append((W, H))
    out["sizes"], out["seeds"], out["img_seed"] = np.array(sizes), np.array(seeds), np.array(IMG_SEED)
    print("covered", sorted(covered, key=str), "values outside [0, 256):", n_wrap)
    assert len(covered) == 18 and n_wrap > 0


CALIB = """P0: 7.215377e+02 0.000000e+00 6.095593e+02 0.000000e+00 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P1: 7.215377e+02 0.000000e+00 6.095593e+02 -3.875744e+02 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P2: 7.215377e+02 0.000000e+00 6.095593e+02 4.485728e+01 0.000000e+00 7.215377e+02 1.728540e+02 2.163791e-01 0.000000e+00 0.000000e+00 1.000000e+00 2.745884e-03
P3: 7.215377e+02 0.000000e+00 6.095593e+02 -3.395242e+02 0.000000e+00 7.215377e+02 1.728540e+02 2.199936e+00 0.000000e+00 0.000000e+00 1.000000e+00 2.729905e-03
R0_rect: 9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 4.351614e-03 9.999631e-01
Tr_velo_to_cam: 7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 -7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01
Tr_imu_to_velo: 9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 9.998898e-01 -1.482298e-02 3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01
"""
LABEL = "Car 0.00 0 -1.58 587.01 173.33 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59\n"


def gen_e2e(out):
    import yaml
    if REF not in sys.path:
        sys.path.insert(0, REF)
    try:
        import skimage.io  # noqa: F401
    except ImportError:                                   # kitti_common.py imports skimage.io; nothing here calls it
        sk = types.ModuleType("skimage")
        sk.io = types.ModuleType("skimage.io")
        sys.modules["skimage"], sys.modules["skimage.io"] = sk, sk.io
    from lib.datasets.kitti.kitti_dataset import KITTI_Dataset
    from lib.datasets.kitti.pd import PhotometricDistort
    with open(os.path.join(REF, "configs", "monodetr.yaml")) as f:
        cfg = yaml.load(f, Loader=yaml.Loader)["dataset"]
    src = synthetic_images(IMG_SEED - 1, [E2E_SIZE])[0]
    out["e2e.size"], out["e2e.img_seed"], out["e2e.res"] = np.array(E2E_SIZE), np.array(IMG_SEED - 1), np.array(E2E_RES)
    for key in ("random_flip", "random_crop", "scale", "shift"):
        out[f"e2e.{key}"] = np.array(float(cfg[key]))
    assert cfg["aug_pd"] and cfg["aug_crop"]
    with tempfile.TemporaryDirectory() as d:
        for sub in ("ImageSets", "training/image_2", "training/calib", "training/label_2"):
            os.makedirs(os.path.join(d, sub))
        open(os.path.join(d, "ImageSets", "train.txt"), "w").write("000000\n")
        Image.fromarray(src).save(os.path.join(d, "training", "image_2", "000000.png"))
        open(os.path.join(d, "training", "calib", "000000.txt"), "w").write(CALIB)
        open(os.path.join(d, "training", "label_2", "000000.txt"), "w").write(LABEL)
        cfg = dict(cfg, root_dir=d)
        ds = KITTI_Dataset("train", cfg)
        ds.resolution = np.array(E2E_RES)
        table = normalize(np.tile(np.arange(256, dtype=np.uint8)[None, :, None], (1, 1, 3)))[:, 0, :]     # (3, 256)
        assert all(np.unique(table[c]).size == 256 for c in range(3)) and (np.diff(table, axis=1) > 0).all()
        for k, seed in enumerate(E2E_SEEDS):
            np.random.seed(seed)
            img = ds[0][0]
            state_arrays(f"e2e.{k}.", out)
            u8 = np.stack([np.searchsorted(table[c], img[c]) for c in range(3)], -1).astype(np.uint8)
            assert np.array_equal(normalize(u8), img)
            out[f"e2e.{k}.u8"] = u8
            # the same draws again through the reference's own calls: PhotometricDistort on a dummy image, then
            # kitti_dataset.py:141-151
            np.random.seed(seed)
            PhotometricDistort()(np.zeros((1, 1, 3), np.float32))
            flip = np.random.random() < cfg["random_flip"]
            crop = np.random.random() < cfg["random_crop"]
            draws = np.random.randn(3) if crop else np.zeros(3)
            out[f"e2e.{k}.flip"], out[f"e2e.{k}.crop"], out[f"e2e.{k}.randn"] = np.array(flip), np.array(crop), draws
            print("e2e", k, "seed", seed, "flip", flip, "crop", crop)
    out["e2e.seeds"] = np.array(E2E_SEEDS)


def main():
    out = {}
    gen_cases(out)
    gen_e2e(out)
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
