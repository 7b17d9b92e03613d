"""Input pipeline on the device (SURVEY.md 8 f4): the image half of the reference dataset's __getitem__
(lib/datasets/kitti/kitti_dataset.py:121-163) for a whole batch in one kernel (csrc/preprocess.cu).

  get_affine_transform(center, scale, rot, output_size, shift, inv)   lib/datasets/kitti/kitti_utils.py:347-381 (host: 6 numbers
                                                                      per image; cv2.getAffineTransform restated as a 3-point solve)
  ImageBatchPreprocessor(resolution, mean, std)(images_u8, trans_inv, flip)  -> (B, 3, H, W) fp32 normalised, on the device
  PhotometricDistort().sample()                                       lib/datasets/kitti/pd.py:376-397 (`aug_pd`): the host draws
  ImageBatchPreprocessor(...)(images_u8, trans_inv, flip, distort=[records])  the distortion on the device first (a second launch,
                                                                      csrc/preprocess.cu), bit-identical to pd.py + cv2 + numpy

`images_u8`: list of (H_i, W_i, 3) uint8 tensors (ragged, as decoded; CPU tensors are uploaded through pinned memory, CUDA tensors
are used in place).  The result is bit-identical to PIL's AFFINE/BILINEAR transform followed by the reference's numpy
normalisation (tests/test_preprocess_gpu.py, tests/golden/preprocess.npz).
"""
from typing import NamedTuple

import numpy as np
import torch

from . import _lib

KITTI_MEAN = (0.485, 0.456, 0.406)        # kitti_dataset.py:73-74
KITTI_STD = (0.229, 0.224, 0.225)


def _get_dir(src_point, rot_rad):
    sn, cs = np.sin(rot_rad), np.cos(rot_rad)
    return np.array([src_point[0] * cs - src_point[1] * sn, src_point[0] * sn + src_point[1] * cs], dtype=np.float64)


def _third(a, b):
    d = a - b
    return b + np.array([-d[1], d[0]], dtype=np.float32)


def _solve_affine(src, dst):
    """The 2x3 matrix M with M @ [x, y, 1] = dst for three point pairs, bit for bit what cv2.getAffineTransform returns: its
    6x6 system solved as cv2.solve(DECOMP_LU) does -- Gaussian elimination with partial pivoting (first largest |pivot|),
    rows updated with a * (-1 / pivot), back substitution dividing by the pivot -- in fp64 without contraction.  A LAPACK
    solve differs in the last bits, which moves the occasional PIL sample point across a truncation edge."""
    A = [[0.0] * 6 for _ in range(6)]
    b = [0.0] * 6
    for i in range(3):
        x, y = float(src[i, 0]), float(src[i, 1])
        A[2 * i][0:3] = [x, y, 1.0]
        A[2 * i + 1][3:6] = [x, y, 1.0]
        b[2 * i], b[2 * i + 1] = float(dst[i, 0]), float(dst[i, 1])
    for i in range(6):
        k = i
        for j in range(i + 1, 6):
            if abs(A[j][i]) > abs(A[k][i]):
                k = j
        if abs(A[k][i]) < np.finfo(np.float64).eps * 10:
            raise np.linalg.LinAlgError("get_affine_transform: the three points are collinear")
        A[i], A[k] = A[k], A[i]
        b[i], b[k] = b[k], b[i]
        d = -1.0 / A[i][i]
        for j in range(i + 1, 6):
            alpha = A[j][i] * d
            for c in range(i + 1, 6):
                A[j][c] += alpha * A[i][c]
            b[j] += alpha * b[i]
    for i in range(5, -1, -1):
        s = b[i]
        for c in range(i + 1, 6):
            s -= A[i][c] * b[c]
        b[i] = s / A[i][i]
    return np.array(b, np.float64).reshape(2, 3)


def get_affine_transform(center, scale, rot, output_size, shift=np.array([0, 0], dtype=np.float32), inv=0):
    """kitti_utils.py:347-381, same arguments and return values (trans, or (trans, trans_inv) with inv=1)."""
    if not isinstance(scale, np.ndarray) and not isinstance(scale, list):
        scale = np.array([scale, scale], dtype=np.float32)
    src_w, dst_w, dst_h = scale[0], output_size[0], output_size[1]
    src_dir = _get_dir([0, src_w * -0.5], np.pi * rot / 180)
    dst_dir = np.array([0, dst_w * -0.5], np.float32)
    src = np.zeros((3, 2), dtype=np.float32)
    dst = np.zeros((3, 2), dtype=np.float32)
    src[0, :] = center + scale * shift
    src[1, :] = center + src_dir + scale * shift
    dst[0, :] = [dst_w * 0.5, dst_h * 0.5]
    dst[1, :] = np.array([dst_w * 0.5, dst_h * 0.5], np.float32) + dst_dir
    src[2:, :] = _third(src[0, :], src[1, :])
    dst[2:, :] = _third(dst[0, :], dst[1, :])
    trans = _solve_affine(src, dst)
    if inv:
        return trans, _solve_affine(dst, src)
    return trans


class PhotometricParams(NamedTuple):
    """One image's draws of the reference's PhotometricDistort (the C record mdb_photometric_params).  A step whose coin said no
    carries its neutral value, which gives the same bits as skipping it."""
    brightness: float = 0.0         # RandomBrightness delta
    contrast: float = 1.0           # RandomContrast alpha
    saturation: float = 1.0         # RandomSaturation factor
    hue: float = 0.0                # RandomHue delta (degrees)
    contrast_last: int = 0          # 0: contrast before the HSV steps (pd[:-1]); 1: after them (pd[1:])
    perm: int = 0                   # RandomLightingNoise: index into pd.py's perms (0 = identity)


class PhotometricDistort:
    """lib/datasets/kitti/pd.py:376-397 split in two: `sample()` makes the reference's random draws on the host, and
    ImageBatchPreprocessor(..., distort=[records]) applies them to the whole batch on the device.  In the dataset,
    `pd_params = self.pd.sample()` replaces the three lines of kitti_dataset.py:136-138."""

    def __init__(self, brightness_delta=32, contrast=(0.5, 1.5), saturation=(0.5, 1.5), hue_delta=18.0):
        self.brightness_delta = brightness_delta        # pd.py:185-188, 170-175, 114-119, 128-131 defaults
        self.contrast = contrast
        self.saturation = saturation
        self.hue_delta = hue_delta

    def sample(self, rs=np.random):
        """The same `randint` / `uniform` calls as PhotometricDistort.__call__, in the same order and on the same generator (the
        global numpy.random unless `rs` is given), including the ones whose step is then skipped; so the flip and crop draws that
        follow in __getitem__ see the stream they see in the reference."""
        p = {}
        if rs.randint(2):
            p["brightness"] = rs.uniform(-self.brightness_delta, self.brightness_delta)
        contrast_first = rs.randint(2)
        p["contrast_last"] = 0 if contrast_first else 1
        if contrast_first and rs.randint(2):
            p["contrast"] = rs.uniform(*self.contrast)
        if rs.randint(2):
            p["saturation"] = rs.uniform(*self.saturation)
        if rs.randint(2):
            p["hue"] = rs.uniform(-self.hue_delta, self.hue_delta)
        if not contrast_first and rs.randint(2):
            p["contrast"] = rs.uniform(*self.contrast)
        if rs.randint(2):
            p["perm"] = rs.randint(6)
        return PhotometricParams(**p)


_RECORD_DTYPE = np.dtype([("brightness", "<f4"), ("contrast", "<f4"), ("saturation", "<f4"), ("hue", "<f4"),
                          ("contrast_last", "<i4"), ("perm", "<i4")])         # 24 bytes, include/monodetr_b200.h


def pack_photometric(records, B):
    """(B, 6) records -> the bytes of B mdb_photometric_params (4 float32, 2 int32 each); ValueError on a malformed record."""
    if len(records) != B:
        raise ValueError(f"distort: {len(records)} records for {B} images")
    out = np.zeros(B, dtype=_RECORD_DTYPE)
    for i, r in enumerate(records):
        try:
            if len(r) != len(PhotometricParams._fields):
                raise ValueError(f"{len(r)} fields")
            r = PhotometricParams(*r)
            vals = np.array(r[:4], np.float64)
        except (TypeError, ValueError) as e:
            raise ValueError(f"distort[{i}]: not a record of 6 numbers ({e})") from None
        if not np.isfinite(vals).all() or np.any(np.abs(vals) > np.finfo(np.float32).max):
            raise ValueError(f"distort[{i}]: non-finite or out-of-range value {r}")
        if r.contrast_last not in (0, 1) or int(r.contrast_last) != r.contrast_last:
            raise ValueError(f"distort[{i}]: contrast_last must be 0 or 1, got {r.contrast_last!r}")
        if r.perm not in range(6) or int(r.perm) != r.perm:
            raise ValueError(f"distort[{i}]: perm must be in 0..5, got {r.perm!r}")
        out[i] = (*vals.astype(np.float32), int(r.contrast_last), int(r.perm))
    return out


def _require_cuda(device):
    if device.type != "cuda":
        raise RuntimeError("ImageBatchPreprocessor: a CUDA device is required (there is no CPU path)")


class ImageBatchPreprocessor:
    def __init__(self, resolution=(1280, 384), mean=KITTI_MEAN, std=KITTI_STD, device="cuda"):
        self.resolution = (int(resolution[0]), int(resolution[1]))        # (W, H) as the reference's `resolution`
        self.mean = np.asarray(mean, np.float32)
        self.std = np.asarray(std, np.float32)
        self.device = torch.device(device)

    def __call__(self, images, trans_inv, flip=None, distort=None):
        """images: list of (H, W, 3) uint8 tensors; trans_inv: (B, 2, 3) array (PIL `data`); flip: optional (B,) bools;
        distort: optional list of B PhotometricParams (PhotometricDistort.sample()), applied to each source image before the flip
        and the warp, as the reference's `aug_pd`.  The images themselves are never modified."""
        B = len(images)
        _require_cuda(self.device)
        records = None if distort is None else pack_photometric(distort, B)
        dev_imgs = self._device_images(images)
        # ONE pinned upload for all per-image metadata: pointers | pitches | matrices (fp64) | (W, H) int32 pairs | flip flags
        # [| distorted-image pointers | their pitches | distortion records]
        n_base = B * 9 + (B + 7) // 8
        buf = np.zeros(n_base + (0 if records is None else 5 * B), np.int64)
        for i, im in enumerate(dev_imgs):
            buf[i], buf[B + i] = im.data_ptr(), im.stride(0)
        buf[2 * B:8 * B].view(np.float64)[:] = np.asarray(trans_inv, np.float64).reshape(B * 6)
        wh = buf[8 * B:9 * B].view(np.int32)
        wh[0::2], wh[1::2] = [im.shape[1] for im in dev_imgs], [im.shape[0] for im in dev_imgs]
        if flip is not None:
            buf[9 * B:n_base].view(np.uint8)[:B] = np.asarray(flip).astype(np.uint8)
        scratch = None
        if records is not None:
            # one flat buffer holds every distorted image, rows packed (pitch 3 * W)
            sizes = [im.shape[0] * im.shape[1] * 3 for im in dev_imgs]
            scratch = torch.empty(max(sum(sizes), 1), dtype=torch.uint8, device=self.device)
            offs = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(np.int64)
            buf[n_base:n_base + B] = scratch.data_ptr() + offs
            buf[n_base + B:n_base + 2 * B] = [3 * im.shape[1] for im in dev_imgs]
            buf[n_base + 2 * B:n_base + 5 * B].view(_RECORD_DTYPE)[:] = records
        meta = torch.from_numpy(buf).pin_memory().to(self.device, non_blocking=True)
        base = meta.data_ptr()
        ptrs, pitch, trd, whd, fld = base, base + 8 * B, base + 16 * B, base + 64 * B, base + 72 * B
        W, H = self.resolution
        out = torch.empty(B, 3, H, W, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            if records is not None:
                dptrs, dpitch, recd = base + 8 * n_base, base + 8 * (n_base + B), base + 8 * (n_base + 2 * B)
                _lib.call("mdb_photometric_distort_u8", ptrs, whd, pitch, recd, dptrs, dpitch, B)
                ptrs, pitch = dptrs, dpitch                     # the warp samples the distorted images
            _lib.call("mdb_warp_affine_normalize_u8", ptrs, whd, pitch, trd, fld, B, W, H, self.mean.ctypes.data, self.std.ctypes.data,
                      out)
        return out

    def distort(self, images, distort):
        """The distortion alone: list of (H, W, 3) uint8 tensors + B records -> list of distorted (H, W, 3) uint8 CUDA tensors,
        bit-identical to the reference's `pd(img.astype(np.float32)).astype(np.uint8)` (kitti_dataset.py:136-138)."""
        B = len(images)
        _require_cuda(self.device)
        records = pack_photometric(distort, B)
        dev_imgs = self._device_images(images)
        outs = [torch.empty(tuple(im.shape), dtype=torch.uint8, device=self.device) for im in dev_imgs]
        buf = np.zeros(8 * B, np.int64)                 # src pointers | src pitches | (W, H) | dst pointers | dst pitches | records
        for i, (im, o) in enumerate(zip(dev_imgs, outs)):
            buf[i], buf[B + i], buf[3 * B + i], buf[4 * B + i] = im.data_ptr(), im.stride(0), o.data_ptr(), o.stride(0)
        wh = buf[2 * B:3 * B].view(np.int32)
        wh[0::2], wh[1::2] = [im.shape[1] for im in dev_imgs], [im.shape[0] for im in dev_imgs]
        buf[5 * B:8 * B].view(_RECORD_DTYPE)[:] = records
        meta = torch.from_numpy(buf).pin_memory().to(self.device, non_blocking=True)
        base = meta.data_ptr()
        with torch.cuda.device(self.device):
            _lib.call("mdb_photometric_distort_u8", base, base + 16 * B, base + 8 * B, base + 40 * B, base + 24 * B, base + 32 * B, B)
        return outs

    def _device_images(self, images):
        dev_imgs = []
        for im in images:
            if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise ValueError("images must be (H, W, 3) uint8 tensors")
            if not im.is_cuda:
                im = (im if im.is_pinned() else im.contiguous().pin_memory()).to(self.device, non_blocking=True)
            if im.stride(2) != 1 or im.stride(1) != 3:
                im = im.contiguous()
            dev_imgs.append(im)
        return dev_imgs
