"""Inference post-process on the device (SURVEY.md 8 f3) behind the reference's two functions.

  extract_dets_from_outputs(outputs, K=50, topk=50)                      lib/helpers/decode_helper.py:57-110
  decode_detections(dets, info, calibs, cls_mean_size, threshold)         lib/helpers/decode_helper.py:8-54

The reference's tester (lib/helpers/tester_helper.py:85-100) copies the (B, topk, 37) detections to the host and decodes them
with a Python loop per detection.  Here both steps are one kernel each on the model's stream (csrc/decode.cu);
`decode_detections` keeps the reference's signature and result (dict img_id -> list of 14-value rows) and performs ONE
device->host copy of the decoded rows; `decode_detections_device` returns device tensors and never synchronises.
There is no CPU path: host tensors raise.
"""
import numpy as np
import torch

from . import _lib

DET_COLS = 37
OUT_COLS = 14


def _f32(t, device):
    if not isinstance(t, torch.Tensor):
        t = torch.as_tensor(np.asarray(t, dtype=np.float32))
    return t.to(device=device, dtype=torch.float32).contiguous()


def extract_dets_from_outputs(outputs, K=50, topk=50):
    """outputs: MonoDETR.forward's dict (monodetr.py:270-283).  Returns (B, topk, 37) on the device, rows ordered by
    descending score: label, score, xs2d, ys2d, w, h, depth, heading[24], size_3d[3], xs3d, ys3d, sigma.
    `K` is accepted and unused, as in the reference."""
    logits = outputs["pred_logits"]
    if not logits.is_cuda:
        raise RuntimeError("extract_dets_from_outputs: CUDA tensors required (not implemented on the CPU)")
    dev = logits.device
    logits = logits.detach().float().contiguous()
    boxes, dim3, depth, angle = (_f32(outputs[k].detach(), dev) for k in ("pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle"))
    B, Q, C = logits.shape
    if boxes.shape != (B, Q, 6) or dim3.shape != (B, Q, 3) or depth.shape != (B, Q, 2) or angle.shape != (B, Q, 24):
        raise ValueError("extract_dets_from_outputs: head outputs with unexpected shapes")
    dets = torch.empty(B, topk, DET_COLS, device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.call("mdb_extract_dets_f32", logits, boxes, dim3, depth, angle, B, Q, C, topk, dets)
    return dets


def _calib_matrix(calibs, device):
    """list of Calibration objects (kitti_utils.py:136-155, `.P2`), or an array / tensor (B, 3, 4)."""
    if isinstance(calibs, (list, tuple)):
        calibs = np.stack([np.asarray(getattr(c, "P2", c), dtype=np.float32) for c in calibs])
    return _f32(calibs, device)


def decode_detections_device(dets, img_size, calibs, cls_mean_size, threshold):
    """dets (B, topk, 37) CUDA.  Returns (rows (B, topk, 14), count (B,) int32) on the device: the count[b] leading rows of
    image b are [cls, alpha, x0, y0, x1, y1, h, w, l, X, Y, Z, ry, score]; the others are zero."""
    if not dets.is_cuda:
        raise RuntimeError("decode_detections_device: CUDA tensors required (not implemented on the CPU)")
    dev = dets.device
    dets = dets.float().contiguous()
    B, topk, cols = dets.shape
    if cols != DET_COLS:
        raise ValueError("decode_detections_device: dets must have 37 columns")
    img_size, P2, mean = _f32(img_size, dev), _calib_matrix(calibs, dev), _f32(cls_mean_size, dev)
    if img_size.shape != (B, 2) or P2.shape != (B, 3, 4) or mean.dim() != 2 or mean.shape[1] != 3:
        raise ValueError("decode_detections_device: img_size (B,2), calibs (B,3,4), cls_mean_size (C,3) expected")
    rows = torch.empty(B, topk, OUT_COLS, device=dev, dtype=torch.float32)
    count = torch.empty(B, device=dev, dtype=torch.int32)
    with torch.cuda.device(dev):
        _lib.call("mdb_decode_dets_f32", dets, img_size, P2, mean, B, topk, mean.shape[0], float(threshold), rows, count)
    return rows, count


def decode_detections(dets, info, calibs, cls_mean_size, threshold):
    """The reference's signature and result: {img_id: [[cls_id, alpha, x0, y0, x1, y1, h, w, l, X, Y, Z, ry, score], ...]}.
    `dets` is the CUDA tensor from `extract_dets_from_outputs` (no .cpu() in between); info['img_size'] (B, 2),
    info['img_id'] (B,)."""
    rows, count = decode_detections_device(dets, info["img_size"], calibs, cls_mean_size, threshold)
    packed = torch.cat([rows.flatten(1), count.to(torch.float32).unsqueeze(1)], dim=1).cpu().numpy()      # the one copy
    ids = info["img_id"]
    ids = ids.tolist() if hasattr(ids, "tolist") else list(ids)
    results = {}
    for i, img_id in enumerate(ids):
        n = int(packed[i, -1])
        r = packed[i, :-1].reshape(-1, OUT_COLS)[:n]
        results[img_id] = [[int(v[0])] + v[1:].tolist() for v in r]
    return results
