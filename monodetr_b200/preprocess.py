"""Input pipeline on the device (SURVEY.md 8 f4): the image half of the reference dataset's __getitem__
(lib/datasets/kitti/kitti_dataset.py:121-163) for a whole batch in one kernel (csrc/preprocess.cu).

  get_affine_transform(center, scale, rot, output_size, shift, inv)   lib/datasets/kitti/kitti_utils.py:347-381 (host: 6 numbers
                                                                      per image; cv2.getAffineTransform restated as a 3-point solve)
  ImageBatchPreprocessor(resolution, mean, std)(images_u8, trans_inv, flip)  -> (B, 3, H, W) fp32 normalised, on the device

`images_u8`: list of (H_i, W_i, 3) uint8 tensors (ragged, as decoded; CPU tensors are uploaded through pinned memory, CUDA tensors
are used in place).  The result is bit-identical to PIL's AFFINE/BILINEAR transform followed by the reference's numpy
normalisation (tests/test_preprocess_gpu.py, tests/golden/preprocess.npz).
"""
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
    """The 2x3 matrix M with M @ [x, y, 1] = dst for three point pairs (what cv2.getAffineTransform returns, float64)."""
    A = np.zeros((6, 6), np.float64)
    b = np.zeros(6, np.float64)
    for i in range(3):
        A[2 * i, 0:3] = [src[i, 0], src[i, 1], 1.0]
        A[2 * i + 1, 3:6] = [src[i, 0], src[i, 1], 1.0]
        b[2 * i], b[2 * i + 1] = dst[i, 0], dst[i, 1]
    return np.linalg.solve(A, b).reshape(2, 3)


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


class ImageBatchPreprocessor:
    def __init__(self, resolution=(1280, 384), mean=KITTI_MEAN, std=KITTI_STD, device="cuda"):
        self.resolution = (int(resolution[0]), int(resolution[1]))        # (W, H) as the reference's `resolution`
        self.mean = np.asarray(mean, np.float32)
        self.std = np.asarray(std, np.float32)
        self.device = torch.device(device)

    def __call__(self, images, trans_inv, flip=None):
        """images: list of (H, W, 3) uint8 tensors; trans_inv: (B, 2, 3) array (PIL `data`); flip: optional (B,) bools."""
        B = len(images)
        if self.device.type != "cuda":
            raise RuntimeError("ImageBatchPreprocessor: a CUDA device is required (there is no CPU path)")
        dev_imgs = []
        for im in images:
            if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3:
                raise ValueError("images must be (H, W, 3) uint8 tensors")
            if not im.is_cuda:
                im = (im if im.is_pinned() else im.contiguous().pin_memory()).to(self.device, non_blocking=True)
            if im.stride(2) != 1 or im.stride(1) != 3:
                im = im.contiguous()
            dev_imgs.append(im)
        # ONE pinned upload for all per-image metadata: pointers | pitches | matrices (fp64) | (W, H) int32 pairs | flip flags
        buf = np.zeros(B * 9 + (B + 7) // 8, np.int64)
        for i, im in enumerate(dev_imgs):
            buf[i], buf[B + i] = im.data_ptr(), im.stride(0)
        buf[2 * B:8 * B].view(np.float64)[:] = np.asarray(trans_inv, np.float64).reshape(B * 6)
        wh = buf[8 * B:9 * B].view(np.int32)
        wh[0::2], wh[1::2] = [im.shape[1] for im in dev_imgs], [im.shape[0] for im in dev_imgs]
        if flip is not None:
            buf[9 * B:].view(np.uint8)[:B] = np.asarray(flip).astype(np.uint8)
        meta = torch.from_numpy(buf).pin_memory().to(self.device, non_blocking=True)
        base = meta.data_ptr()
        ptrs, pitch, trd, whd, fld = base, base + 8 * B, base + 16 * B, base + 64 * B, base + 72 * B
        W, H = self.resolution
        out = torch.empty(B, 3, H, W, dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.call("mdb_warp_affine_normalize_u8", ptrs, whd, pitch, trd, fld, B, W, H, self.mean.ctypes.data, self.std.ctypes.data,
                      out)
        return out
