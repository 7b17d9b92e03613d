"""KITTI training targets on the device: the label half of the reference dataset's __getitem__
(lib/datasets/kitti/kitti_dataset.py:173-330) for a whole batch in one kernel (csrc/labels.cu).

  LabelBank.from_kitti(root_dir, split)        every label and calib file of a split parsed ONCE (kitti_utils.py:13-51, 118-155)
                                               and kept on the device in CSR form; LabelBank.from_arrays(...) for synthetic data
  AugmentationSampler(...).sample(img_size)    the random draws of kitti_dataset.py:130-154 on the host (same numpy.random calls,
                                               same order): one AugRecord per image (flip, crop, trans / trans_inv, photometric)
  TargetEncoder(...)(bank, bank_indices, records)   the padded targets (B, max_objs, ...) in the reference's collated dtypes
  KittiBatchBuilder(cfg, split, bank)(images_u8, bank_indices, records)
                                               what the reference's DataLoader yields for the batch: (inputs, P2, targets, info);
                                               the images go through ImageBatchPreprocessor with the SAME records

The label files never change between epochs, so a training step uploads only one 72-byte record per image.  The targets agree with
the reference's within the tolerances stated in oracle/labels.py (tests/golden/labels.npz).
"""
import math
import os
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import _lib
from .preprocess import ImageBatchPreprocessor, PhotometricDistort, PhotometricParams, get_affine_transform

# record columns (include/monodetr_b200.h MDB_LABEL_*)
RECORD_WIDTH = 16
CLS, TRUNC, OCC, ALPHA, X1, Y1, X2, Y2, H, W, L, PX, PY, PZ, RY = range(15)
CLASS_NAMES = ("Pedestrian", "Car", "Cyclist")          # kitti_dataset.py:31 cls2id; the class code of any other type is -1
MAX_OBJS = 50                                            # kitti_dataset.py:29
DEPTH_SCALES = {"normal": 0, "inverse": 1, "none": 2}
CLS_MEAN_SIZE = np.array([[1.76255119, 0.66068622, 0.84422524],         # kitti_dataset.py:75-77
                          [1.52563191462, 1.62856739989, 3.88311640418],
                          [1.73698127, 0.59706367, 1.76282397]])
TARGET_KEYS = ("calibs", "indices", "labels", "boxes", "boxes_3d", "depth", "size_2d", "size_3d", "src_size_3d", "heading_bin",
               "heading_res", "mask_2d")
_IMAGE_DTYPE = np.dtype([("trans", "<f8", (6,)), ("crop_scale", "<f8"), ("bank_index", "<i4"), ("img_w", "<i4"), ("img_h", "<i4"),
                         ("flip", "<i4")])                                          # mdb_label_image, 72 bytes
_CONFIG_DTYPE = np.dtype([("mean_size", "<f8", (9,)), ("class_mask", "<i4"), ("clip_2d", "<i4"), ("depth_scale", "<i4"),
                          ("res_w", "<i4"), ("res_h", "<i4"), ("max_objs", "<i4")])  # mdb_label_config, 96 bytes


def _require_cuda(device):
    if device.type != "cuda":
        raise RuntimeError("monodetr_b200.labels: a CUDA device is required (there is no CPU path)")


# ---- parsing (host, once per split) -------------------------------------------------------------------------------------------
def parse_label_file(path):
    """kitti_utils.get_objects_from_label: (class names, (n, RECORD_WIDTH) fp64 records).  Fields are split on single spaces and
    converted as the reference does (box2d and pos rounded to float32); a malformed line raises ValueError naming file and line."""
    names, rows = [], []
    with open(path) as f:
        for lineno, line in enumerate(f, 1):
            fields = line.strip().split(" ")
            try:
                if len(fields) not in (15, 16):
                    raise ValueError(f"{len(fields)} fields, expected 15 or 16")
                v = [float(x) for x in fields[1:15]]
            except ValueError as e:
                raise ValueError(f"{path}:{lineno}: malformed label line ({e})") from None
            rec = np.zeros(RECORD_WIDTH)
            rec[CLS] = CLASS_NAMES.index(fields[0]) if fields[0] in CLASS_NAMES else -1
            rec[[TRUNC, OCC, ALPHA]] = v[0:3]
            rec[X1:Y2 + 1] = np.array(v[3:7], np.float32)
            rec[[H, W, L]] = v[7:10]
            rec[PX:PZ + 1] = np.array(v[10:13], np.float32)
            rec[RY] = v[13]
            names.append(fields[0])
            rows.append(rec)
    return names, np.array(rows, np.float64).reshape(-1, RECORD_WIDTH)


def parse_calib_file(path):
    """kitti_utils.get_calib_from_file's P2: the third line's 12 numbers, float32 (3, 4)."""
    with open(path) as f:
        lines = f.readlines()
    try:
        return np.array(lines[2].strip().split(" ")[1:], dtype=np.float32).reshape(3, 4)
    except (IndexError, ValueError) as e:
        raise ValueError(f"{path}:3: malformed P2 line ({e})") from None


class LabelBank:
    """The label lines and P2 of a set of images, on the device: `offsets` (n+1) int64, `objects` (offsets[-1], RECORD_WIDTH) fp64,
    `P2` (n, 3, 4) float32.  `img_ids[k]` is the KITTI id of bank image k; `names` the class names of the lines (from_kitti only).
    Every line is kept, in file order: target slot i of an image is its line i, as in the reference."""

    def __init__(self, offsets, objects, P2, img_ids, names=None, device="cuda"):
        offsets = np.asarray(offsets, np.int64)
        objects = np.asarray(objects, np.float64).reshape(-1, RECORD_WIDTH)
        P2 = np.asarray(P2, np.float32).reshape(-1, 3, 4)
        n = len(P2)
        if n < 1 or offsets.shape != (n + 1,) or offsets[0] != 0 or (np.diff(offsets) < 0).any() or offsets[-1] != len(objects):
            raise ValueError("LabelBank: offsets must be n+1 non-decreasing prefix sums from 0 to the number of records")
        if len(img_ids) != n:
            raise ValueError("LabelBank: one img_id per image")
        if not np.isfinite(objects).all() or not np.isfinite(P2).all():
            raise ValueError("LabelBank: non-finite record or P2 value")
        self.host_offsets, self.host_objects, self.host_P2 = offsets, objects, P2
        self.img_ids = [int(i) for i in img_ids]
        self.names = names
        self.device = torch.device(device)
        self.offsets = torch.from_numpy(offsets).to(self.device)
        self.objects = torch.from_numpy(objects).to(self.device)
        self.P2 = torch.from_numpy(P2).to(self.device)

    def __len__(self):
        return len(self.img_ids)

    @classmethod
    def from_arrays(cls, counts, objects, P2, img_ids=None, device="cuda"):
        """counts (n,) lines per image, objects (sum(counts), RECORD_WIDTH) records in image order (box2d / pos columns are rounded
        to float32), P2 (n, 3, 4)."""
        counts = np.asarray(counts, np.int64)
        objects = np.array(objects, np.float64).reshape(-1, RECORD_WIDTH)
        for c in (slice(X1, Y2 + 1), slice(PX, PZ + 1)):
            objects[:, c] = objects[:, c].astype(np.float32)
        offsets = np.concatenate([[0], np.cumsum(counts)])
        return cls(offsets, objects, P2, range(len(counts)) if img_ids is None else img_ids, device=device)

    @classmethod
    def from_kitti(cls, root_dir, split, device="cuda"):
        """All images of ImageSets/<split>.txt (kitti_dataset.py:49-56), parsed once."""
        if split == "test":
            raise NotImplementedError("LabelBank: the test split has no labels")
        if split not in ("train", "val", "trainval"):
            raise ValueError(f"LabelBank: unknown split {split!r}")
        with open(os.path.join(root_dir, "ImageSets", split + ".txt")) as f:
            ids = [int(x.strip()) for x in f.readlines()]
        data = os.path.join(root_dir, "training")
        names, objs, P2, counts = [], [], [], []
        for i in ids:
            n, o = parse_label_file(os.path.join(data, "label_2", "%06d.txt" % i))
            names += n
            objs.append(o)
            counts.append(len(n))
            P2.append(parse_calib_file(os.path.join(data, "calib", "%06d.txt" % i)))
        offsets = np.concatenate([[0], np.cumsum(counts)])
        return cls(offsets, np.concatenate(objs) if objs else np.zeros((0, RECORD_WIDTH)), np.array(P2), ids, names, device)


# ---- augmentation draws (host) ------------------------------------------------------------------------------------------------
class AugRecord(NamedTuple):
    """One image's draws: what both halves of __getitem__ need.  crop_scale is 1 when no crop was drawn; distort is None when
    `aug_pd` is off."""
    img_size: tuple
    flip: bool
    crop_scale: float
    center: np.ndarray
    trans: np.ndarray
    trans_inv: np.ndarray
    distort: Optional[PhotometricParams] = None


class AugmentationSampler:
    """kitti_dataset.py:130-154: the same numpy.random calls in the same order, on `rs` (the global numpy.random by default):
    PhotometricDistort.sample() if aug_pd, random() < random_flip, and with aug_crop random() < random_crop then three randn().
    No draw at all outside the train / trainval splits."""

    def __init__(self, split="train", aug_pd=False, aug_crop=False, random_flip=0.5, random_crop=0.5, scale=0.4, shift=0.1,
                 resolution=(1280, 384), rs=None):
        self.augment = split in ("train", "trainval")               # kitti_dataset.py:59
        self.aug_pd, self.aug_crop = bool(aug_pd), bool(aug_crop)
        self.random_flip, self.random_crop, self.scale, self.shift = random_flip, random_crop, scale, shift
        self.resolution = np.array([int(resolution[0]), int(resolution[1])])
        self.rs = np.random if rs is None else rs
        self.pd = PhotometricDistort()

    @classmethod
    def from_config(cls, cfg, split, resolution=(1280, 384), rs=None):
        """The dataset section of the config, with kitti_dataset.py:61-68's defaults."""
        return cls(split, cfg.get("aug_pd", False), cfg.get("aug_crop", False), cfg.get("random_flip", 0.5),
                   cfg.get("random_crop", 0.5), cfg.get("scale", 0.4), cfg.get("shift", 0.1), resolution, rs)

    def sample(self, img_size):
        img_size = np.array([int(img_size[0]), int(img_size[1])])
        center = np.array(img_size) / 2
        crop_size, crop_scale, flip, distort = img_size, 1, False, None
        if self.augment:
            if self.aug_pd:
                distort = self.pd.sample(self.rs)
            if self.rs.random() < self.random_flip:
                flip = True
            if self.aug_crop and self.rs.random() < self.random_crop:
                crop_scale = np.clip(self.rs.randn() * self.scale + 1, 1 - self.scale, 1 + self.scale)
                crop_size = img_size * crop_scale
                center[0] += img_size[0] * np.clip(self.rs.randn() * self.shift, -2 * self.shift, 2 * self.shift)
                center[1] += img_size[1] * np.clip(self.rs.randn() * self.shift, -2 * self.shift, 2 * self.shift)
        trans, trans_inv = get_affine_transform(center, crop_size, 0, self.resolution, inv=1)
        return AugRecord((int(img_size[0]), int(img_size[1])), flip, float(crop_scale), center, trans, trans_inv, distort)


# ---- the encoder (device) -----------------------------------------------------------------------------------------------------
def class_mask(writelist):
    """Writelist -> bit mask over CLASS_NAMES.  A name outside them would reach the reference's cls2id and fail there."""
    bad = [c for c in writelist if c not in CLASS_NAMES]
    if bad:
        raise NotImplementedError(f"writelist classes {bad} have no class id (the reference fails with KeyError on them)")
    return sum(1 << CLASS_NAMES.index(c) for c in set(writelist))


def pack_images(bank, bank_indices, records):
    """B AugRecords -> B mdb_label_image records; ValueError on anything the kernel would read out of range."""
    B = len(bank_indices)
    if B < 1 or B > 65535:
        raise ValueError(f"labels: batch of {B} images (1..65535)")
    if len(records) != B:
        raise ValueError(f"labels: {len(records)} records for {B} images")
    out = np.zeros(B, _IMAGE_DTYPE)
    for b, (k, r) in enumerate(zip(bank_indices, records)):
        if int(k) != k or not 0 <= int(k) < len(bank):
            raise ValueError(f"labels: bank index {k!r} of image {b} outside 0..{len(bank) - 1}")
        trans = np.asarray(r.trans, np.float64)
        cs = float(r.crop_scale)
        if trans.shape != (2, 3) or not np.isfinite(trans).all():
            raise ValueError(f"labels: image {b}: trans must be a finite 2x3 matrix")
        if not math.isfinite(cs) or cs <= 0:
            raise ValueError(f"labels: image {b}: crop_scale must be finite and positive, got {r.crop_scale!r}")
        w, h = (int(v) for v in r.img_size)
        if w <= 0 or h <= 0:
            raise ValueError(f"labels: image {b}: img_size {r.img_size!r}")
        out[b] = (trans.reshape(6), cs, int(k), w, h, int(bool(r.flip)))
    return out


class TargetEncoder:
    """kitti_dataset.py:173-330 for a batch: options as the dataset's config (writelist, clip_2d, depth_scale, meanshape) plus the
    network input resolution and the number of target slots."""

    def __init__(self, writelist=("Car",), clip_2d=False, depth_scale="normal", meanshape=False, resolution=(1280, 384),
                 max_objs=MAX_OBJS, device="cuda"):
        if depth_scale not in DEPTH_SCALES:
            raise ValueError(f"depth_scale must be one of {sorted(DEPTH_SCALES)}, got {depth_scale!r}")
        if not 1 <= int(max_objs) <= 1024:
            raise ValueError("max_objs must be in 1..1024")
        self.cfg = np.zeros((), _CONFIG_DTYPE)
        self.cfg["mean_size"] = (CLS_MEAN_SIZE if meanshape else np.zeros((3, 3))).reshape(9)
        self.cfg["class_mask"] = class_mask(writelist)
        self.cfg["clip_2d"], self.cfg["depth_scale"] = int(bool(clip_2d)), DEPTH_SCALES[depth_scale]
        self.cfg["res_w"], self.cfg["res_h"], self.cfg["max_objs"] = int(resolution[0]), int(resolution[1]), int(max_objs)
        self.max_objs = int(max_objs)
        self.device = torch.device(device)

    def __call__(self, bank, bank_indices, records):
        """Targets of images bank_indices[b] with draws records[b] (AugRecords): dict of device tensors, every key of the
        reference's targets but `img_size`.  One pinned upload, one launch."""
        _require_cuda(self.device)
        recs = pack_images(bank, bank_indices, records)
        B, S = len(recs), self.max_objs
        meta = torch.from_numpy(recs.view(np.uint8)).pin_memory().to(self.device, non_blocking=True)
        dev = self.device
        t = {"calibs": torch.empty(B, S, 3, 4, device=dev), "indices": torch.empty(B, S, dtype=torch.int64, device=dev),
             "labels": torch.empty(B, S, dtype=torch.int8, device=dev), "boxes": torch.empty(B, S, 4, device=dev),
             "boxes_3d": torch.empty(B, S, 6, device=dev), "depth": torch.empty(B, S, 1, device=dev),
             "size_2d": torch.empty(B, S, 2, device=dev), "size_3d": torch.empty(B, S, 3, device=dev),
             "src_size_3d": torch.empty(B, S, 3, device=dev), "heading_bin": torch.empty(B, S, 1, dtype=torch.int64, device=dev),
             "heading_res": torch.empty(B, S, 1, device=dev), "mask_2d": torch.empty(B, S, dtype=torch.bool, device=dev)}
        with torch.cuda.device(dev):
            _lib.call("mdb_kitti_encode_targets", bank.offsets, bank.objects, bank.P2, len(bank), meta, B, self.cfg.ctypes.data,
                      *[t[k] for k in TARGET_KEYS])
        return t


# ---- batch assembly -----------------------------------------------------------------------------------------------------------
class KittiBatchBuilder:
    """One batch of KITTI_Dataset(split, cfg) + DataLoader's default collate, built on the device from decoded images, bank
    indices and the sampler's records: both halves of every image use the same AugRecord.

        builder = KittiBatchBuilder(cfg["dataset"], "train", LabelBank.from_kitti(root, "train"))
        records = [builder.sampler.sample((im.shape[1], im.shape[0])) for im in images]
        inputs, P2, targets, info = builder(images, bank_indices, records)

    `targets` goes into SetCriterion as it is.  Options the device path does not implement raise NotImplementedError."""

    def __init__(self, cfg, split, bank, resolution=(1280, 384), device="cuda", rs=None):
        if split == "test":
            raise NotImplementedError("KittiBatchBuilder: the test split has no labels")
        for opt, what in (("aug_calib", "the P2 refit of Calibration.flip"), ("class_merging", "class merging (Van, Truck)"),
                          ("use_dontcare", "DontCare targets")):
            if cfg.get(opt, False):
                raise NotImplementedError(f"KittiBatchBuilder: {opt} ({what}) is not implemented")
        self.bank = bank
        self.resolution = (int(resolution[0]), int(resolution[1]))
        self.device = torch.device(device)
        self.sampler = AugmentationSampler.from_config(cfg, split, self.resolution, rs)
        self.preprocessor = ImageBatchPreprocessor(self.resolution, device=device)
        self.encoder = TargetEncoder(cfg.get("writelist", ["Car"]), cfg.get("clip_2d", False), cfg.get("depth_scale", "normal"),
                                     cfg.get("meanshape", False), self.resolution, MAX_OBJS, device)

    def __call__(self, images, bank_indices, records):
        """images: list of (H, W, 3) uint8 tensors; bank_indices: B ints; records: B AugRecords of these images.  Returns
        (inputs (B, 3, H, W), P2 (B, 3, 4), targets, info) as the reference's loader yields them; inputs, P2 and targets on the
        device, info on the host."""
        B = len(images)
        if len(bank_indices) != B or len(records) != B:
            raise ValueError(f"KittiBatchBuilder: {B} images, {len(bank_indices)} bank indices, {len(records)} records")
        sizes = np.array([[im.shape[1], im.shape[0]] for im in images], np.int64)
        for b, r in enumerate(records):
            if tuple(r.img_size) != tuple(sizes[b]):
                raise ValueError(f"KittiBatchBuilder: record {b} was drawn for an image of size {r.img_size}, not {tuple(sizes[b])}")
        pd = [r.distort for r in records]
        if any(p is None for p in pd) and not all(p is None for p in pd):
            raise ValueError("KittiBatchBuilder: photometric records for some images only")
        targets = self.encoder(self.bank, bank_indices, records)
        inputs = self.preprocessor(images, np.stack([r.trans_inv for r in records]), [r.flip for r in records],
                                   distort=None if pd[0] is None else pd)
        targets["img_size"] = torch.from_numpy(sizes).to(self.device)
        P2 = torch.from_numpy(self.bank.host_P2[np.asarray(bank_indices, np.int64)]).to(self.device)
        feat = np.array(self.resolution, np.int64) // 32                              # kitti_dataset.py:127, downsample 32
        info = {"img_id": torch.tensor([self.bank.img_ids[int(k)] for k in bank_indices], dtype=torch.int64),
                "img_size": torch.from_numpy(sizes), "bbox_downsample_ratio": torch.from_numpy(sizes / feat)}
        return inputs, P2, targets, info
