"""Generate tests/golden/loader.npz from the UNMODIFIED reference loader (CPU only).

    python tools/gen_golden_loader.py

Needs the reference checkout (MONODETR_REFERENCE, default /root/reference), cv2, yaml, torchvision and numba (NUMBA_ENABLE_CUDASIM=1
is set if absent).  No reference file is edited or copied.  tests/synthetic_kitti.py writes its seeded KITTI folder to a temporary
directory; the shipped configs/monodetr.yaml dataset section (aug_pd, aug_crop, flip 0.5, crop 0.5) is used with batch size 4.
Each run seeds the generators as set_random_seed(444) does, calls the reference's build_dataloader and iterates:
  train_w0 / train_w2   the train loader with workers=0 / 2, two epochs, the generator reseeded before each epoch as
                        Trainer.train does (np.random.seed(np.random.get_state()[1][0] + epoch))
  val                   the test loader with test_split 'val', one epoch
  test                  the test loader with test_split 'test', one epoch

Per (run, epoch) `{run}.e{epoch}.*`, batches concatenated along the first axis, `bounds` their prefix sums:
  ids; sha (sha256 hex of each image's float32 `inputs`); sample_pos / sample_val (64 seeded positions per image and their values);
  calibs; t.<key> every target tensor (train / val); info_img_id, info_img_size, info_ratio; draws (n, 16) float64:
  [flip, crop_scale, center (2), trans_inv (6), brightness, contrast, saturation, hue, contrast_last, perm].
The draws are captured by wrapping KITTI_Dataset.__getitem__ inside this process: the numpy state before the call is replayed
through oracle.photometric.sample and the reference's own flip / crop calls and get_affine_transform, and the replay must end in
the state the call left (asserted), so it made exactly the reference's draws.  They travel back from loader workers in `info`.
Also: cfg (json), tree.sha.<split> (sha256 of each decoded image, in split order).
"""
import copy
import hashlib
import importlib
import json
import os
import sys
import tempfile
import types

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.environ.get("MONODETR_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "loader.npz")
import synthetic_kitti as sk  # noqa: E402
from oracle import photometric as oph  # noqa: E402

SEED = 444
BATCH = 4
N_SAMPLE = 64
TARGET_KEYS = ("calibs", "indices", "img_size", "labels", "boxes", "boxes_3d", "depth", "size_2d", "size_3d", "src_size_3d",
               "heading_bin", "heading_res", "mask_2d")


def _import_reference():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    try:
        import skimage.io  # noqa: F401
    except ImportError:                                   # kitti_common.py imports skimage.io; nothing here calls it
        skm = types.ModuleType("skimage")
        skm.io = types.ModuleType("skimage.io")
        sys.modules["skimage"], sys.modules["skimage.io"] = skm, skm.io
    kd = importlib.import_module("lib.datasets.kitti.kitti_dataset")
    dh = importlib.import_module("lib.helpers.dataloader_helper")
    return kd, dh


def _capture_draws(kd):
    """Wrap KITTI_Dataset.__getitem__ so that info['_draws'] carries the item's draws (see the module docstring)."""
    orig = kd.KITTI_Dataset.__getitem__

    def getitem(self, item):
        start = np.random.get_state()
        out = orig(self, item)
        end = np.random.get_state()
        img_size = np.array(self.get_image(int(self.idx_list[item])).size)
        np.random.set_state(start)
        center = np.array(img_size) / 2
        crop_size, crop_scale, flip, pd = img_size, 1, False, oph.Params(np.nan, np.nan, np.nan, np.nan, -1, -1)
        if self.data_augmentation:
            if self.aug_pd:
                pd = oph.sample()
            flip = np.random.random() < self.random_flip
            if self.aug_crop and np.random.random() < self.random_crop:
                crop_scale = np.clip(np.random.randn() * self.scale + 1, 1 - self.scale, 1 + self.scale)
                crop_size = img_size * crop_scale
                center[0] += img_size[0] * np.clip(np.random.randn() * self.shift, -2 * self.shift, 2 * self.shift)
                center[1] += img_size[1] * np.clip(np.random.randn() * self.shift, -2 * self.shift, 2 * self.shift)
        _, trans_inv = kd.get_affine_transform(center, crop_size, 0, self.resolution, inv=1)
        replayed = np.random.get_state()
        assert np.array_equal(replayed[1], end[1]) and replayed[2:] == end[2:], "the replay made other draws than __getitem__"
        info = dict(out[3], _draws=np.concatenate([[float(flip), float(crop_scale)], center, trans_inv.reshape(6),
                                                   np.array(pd, np.float64)]))
        return out[0], out[1], out[2], info

    kd.KITTI_Dataset.__getitem__ = getitem


def _record(loader, out, prefix, run_index, epoch_reseed=None):
    rows = {k: [] for k in ("ids", "sha", "sample_pos", "sample_val", "calibs", "info_img_id", "info_img_size", "info_ratio",
                            "draws") + tuple("t." + k for k in TARGET_KEYS)}
    sizes = []
    g = np.random.default_rng(run_index)                          # positions only: does not touch the loader's generators
    for inputs, calibs, targets, info in loader:
        x = inputs.numpy()
        assert x.dtype == np.float32 and x.flags.c_contiguous
        sizes.append(len(x))
        for b in range(len(x)):
            rows["sha"].append(hashlib.sha256(x[b].tobytes()).hexdigest())
            pos = g.integers(0, x[b].size, N_SAMPLE)
            rows["sample_pos"].append(pos)
            rows["sample_val"].append(x[b].reshape(-1)[pos])
        rows["ids"].append(info["img_id"].numpy())
        rows["calibs"].append(calibs.numpy())
        rows["info_img_id"].append(info["img_id"].numpy())
        rows["info_img_size"].append(info["img_size"].numpy())
        rows["info_ratio"].append(info["bbox_downsample_ratio"].numpy())
        rows["draws"].append(info["_draws"].numpy())
        if isinstance(targets, dict):
            for k in TARGET_KEYS:
                rows["t." + k].append(targets[k].numpy())
        else:                                                     # test split: the reference returns the image as targets
            assert np.array_equal(targets.numpy(), x)
    for k, v in rows.items():
        if v:
            out[f"{prefix}.{k}"] = np.array(v) if k in ("sha", "sample_pos", "sample_val") else np.concatenate(v)
    out[f"{prefix}.bounds"] = np.concatenate([[0], np.cumsum(sizes)])
    print(prefix, "batches", sizes, "ids", out[f"{prefix}.ids"].tolist())


def main():
    import torch
    import yaml
    from PIL import Image
    kd, dh = _import_reference()
    _capture_draws(kd)
    with open(os.path.join(REF, "configs", "monodetr.yaml")) as f:
        base = yaml.load(f, Loader=yaml.Loader)["dataset"]
    out = {}
    with tempfile.TemporaryDirectory() as d:
        splits = sk.write_tree(d)
        for split in ("train", "val", "test"):
            data = "testing" if split == "test" else "training"
            out[f"tree.sha.{split}"] = np.array([hashlib.sha256(np.array(Image.open(
                os.path.join(d, data, "image_2", "%06d.png" % i))).tobytes()).hexdigest() for i in splits[split]])
        cfg = dict(copy.deepcopy(base), root_dir=d, batch_size=BATCH)
        saved = dict(cfg)
        saved.pop("root_dir")
        out["cfg"] = np.array(json.dumps(saved))
        runs = [("train_w0", 0, "val", 2), ("train_w2", 2, "val", 2), ("val", 0, "val", 1), ("test", 0, "test", 1)]
        for r, (name, workers, test_split, epochs) in enumerate(runs):
            sk.set_random_seed(SEED)
            train_loader, test_loader = dh.build_dataloader(dict(cfg, test_split=test_split), workers=workers)
            loader = train_loader if name.startswith("train") else test_loader
            for epoch in range(epochs):
                if loader is train_loader:
                    np.random.seed(np.random.get_state()[1][0] + epoch)
                _record(loader, out, f"{name}.e{epoch}", 10 * r + epoch)
            assert torch.initial_seed() == SEED ** 3
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
