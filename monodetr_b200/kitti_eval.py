"""KITTI object-detection metric on the device, behind the reference's function names (SURVEY.md 2).

  get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None)
                                       lib/datasets/kitti/kitti_eval_python/eval.py:717-825
  do_eval(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos=False, PR_detail_dict=None, DIForDIS=True)
                                       eval.py:656-696
  get_label_anno(path) / get_label_annos(folder, image_ids=None)
                                       lib/datasets/kitti/kitti_eval_python/kitti_common.py:294-347
  evaluate(results_dir, label_dir, image_ids, classes, logger)
                                       lib/datasets/kitti/kitti_dataset.py:101-116 (KITTI_Dataset.eval)

The reference computes the metric with JIT-compiled CPU loops plus one JIT-compiled CUDA kernel for the rotated IoU.  Here the annotations of
all images are packed once into CSR tables (`pack`), uploaded in one copy, and every configuration of every requested class --
3 metrics x classes x 3 difficulties x 2 overlap sets -- is evaluated by csrc/kitti_eval.cu in one set of launches; one copy brings
back the (tp, fp, fn, similarity) table per score threshold.  Precision, recall, their suffix maxima and the 11- / 40-point AP
are then computed here in fp64 in the reference's order, so the AP values are bit-identical when the counts are.
There is no CPU path: without a GPU the call raises.
"""
import io
import logging
import os
import pathlib
import re

import numpy as np
import torch

from . import _lib

CLASS_NAMES = ("car", "pedestrian", "cyclist", "van", "person_sitting", "truck")     # eval.py:31, lower-cased names
CLASS_TO_NAME = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting", 5: "Truck"}
NAME_TO_CLASS = {v: k for k, v in CLASS_TO_NAME.items()}
NUM_THRESH = 41                 # MDB_KITTI_NUM_THRESH
MAX_BOXES = 1024                # MDB_KITTI_MAX_BOXES
GT_COLS = DT_COLS = 13          # MDB_KITTI_GT_COLS / MDB_KITTI_DT_COLS
# min_overlaps[overlap set, metric (bbox, bev, 3d), class] of get_official_eval_result (eval.py:718-724)
OFFICIAL_MIN_OVERLAPS = np.stack([
    np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3),
    np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]]),
])


# ---------------------------------------------------------------------------------------------------------------- label files
def get_label_anno(label_path):
    """One KITTI label / result file -> dict of arrays; dimensions reordered from the file's (h, w, l) to (l, h, w).  A 16th
    column is the detection score (zeros when absent)."""
    with open(label_path, "r") as f:
        rows = [line.strip().split(" ") for line in f.readlines()]
    n = len(rows)
    anno = {
        "name": np.array([r[0] for r in rows]),
        "truncated": np.array([float(r[1]) for r in rows]),
        "occluded": np.array([int(r[2]) for r in rows]),
        "alpha": np.array([float(r[3]) for r in rows]),
        "bbox": np.array([[float(v) for v in r[4:8]] for r in rows]).reshape(-1, 4),
        "dimensions": np.array([[float(v) for v in r[8:11]] for r in rows]).reshape(-1, 3)[:, [2, 0, 1]],
        "location": np.array([[float(v) for v in r[11:14]] for r in rows]).reshape(-1, 3),
        "rotation_y": np.array([float(r[14]) for r in rows]).reshape(-1),
    }
    if n and len(rows[0]) == 16:
        anno["score"] = np.array([float(r[15]) for r in rows])
    else:
        anno["score"] = np.zeros([len(anno["bbox"])])
    return anno


def get_label_annos(label_folder, image_ids=None):
    """Files `%06d.txt` of `label_folder` for `image_ids` (a list, or an int n meaning range(n)); None = every such file in
    ascending id order."""
    if image_ids is None:
        ids = [int(p.stem) for p in pathlib.Path(label_folder).glob("*.txt") if re.match(r"^\d{6}.txt$", p.name)]
        image_ids = sorted(ids)
    if not isinstance(image_ids, list):
        image_ids = list(range(image_ids))
    return [get_label_anno(os.path.join(label_folder, "%06d.txt" % i)) for i in image_ids]


# ---------------------------------------------------------------------------------------------------------------- host packing
def _class_code(name):
    name = str(name).lower()
    return CLASS_NAMES.index(name) if name in CLASS_NAMES else -1


def _col(a, key, n, width=1):
    return np.asarray(a[key], dtype=np.float64).reshape(n, width)


def pack(gt_annos, dt_annos):
    """CSR tables of include/monodetr_b200.h (mdb_kitti_*): offsets, gt_f / gt_i / dt_f / dt_cls, and the HOST sizes."""
    if len(gt_annos) != len(dt_annos):
        raise ValueError("kitti_eval: gt_annos and dt_annos must list the same images")
    if len(gt_annos) == 0:
        raise ValueError("kitti_eval: no images")
    ng = np.array([len(a["name"]) for a in gt_annos], dtype=np.int64)
    nd = np.array([len(a["name"]) for a in dt_annos], dtype=np.int64)
    gt_off = np.concatenate([[0], np.cumsum(ng)]).astype(np.int32)
    dt_off = np.concatenate([[0], np.cumsum(nd)]).astype(np.int32)
    ov_off = np.concatenate([[0], np.cumsum(ng * nd)]).astype(np.int64)
    gt_f = [np.concatenate([_col(a, "bbox", n, 4), _col(a, "alpha", n), _col(a, "truncated", n), _col(a, "location", n, 3),
                            _col(a, "dimensions", n, 3), _col(a, "rotation_y", n)], 1) for a, n in zip(gt_annos, ng)]
    dt_f = [np.concatenate([_col(a, "bbox", n, 4), _col(a, "alpha", n), _col(a, "score", n), _col(a, "location", n, 3),
                            _col(a, "dimensions", n, 3), _col(a, "rotation_y", n)], 1) for a, n in zip(dt_annos, nd)]
    gt_i = [np.stack([np.asarray(a["occluded"], dtype=np.int64).reshape(n),
                      np.array([_class_code(s) for s in a["name"]], dtype=np.int64).reshape(n),
                      np.array([s == "DontCare" for s in a["name"]], dtype=np.int64).reshape(n)], 1) for a, n in zip(gt_annos, ng)]
    dt_cls = [np.array([_class_code(s) for s in a["name"]], dtype=np.int64).reshape(n) for a, n in zip(dt_annos, nd)]
    return {
        "gt_off": gt_off, "dt_off": dt_off, "ov_off": ov_off,
        "gt_f": np.ascontiguousarray(np.concatenate(gt_f, 0), dtype=np.float64).reshape(-1, GT_COLS),
        "gt_i": np.ascontiguousarray(np.concatenate(gt_i, 0), dtype=np.int32).reshape(-1, 3),
        "dt_f": np.ascontiguousarray(np.concatenate(dt_f, 0), dtype=np.float64).reshape(-1, DT_COLS),
        "dt_cls": np.ascontiguousarray(np.concatenate(dt_cls, 0), dtype=np.int32),
        "n_img": len(gt_annos), "n_gt": int(ng.sum()), "n_dt": int(nd.sum()), "n_ov": int(ov_off[-1]),
        "max_gt": int(ng.max()), "max_dt": int(nd.max()),
    }


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def _upload(arrays, device):
    """One host->device copy of several arrays; returns typed device views in the same order (16-byte aligned)."""
    offs, size = [], 0
    for a in arrays:
        offs.append(size)
        size += (a.nbytes + 15) // 16 * 16
    host = np.zeros(max(size, 16), dtype=np.uint8)
    for a, o in zip(arrays, offs):
        host[o:o + a.nbytes] = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    dev = torch.from_numpy(host).to(device)
    return [dev[o:o + a.nbytes].view(getattr(torch, a.dtype.name)) for a, o in zip(arrays, offs)]


def _launch_overlaps(p, d):
    ov = torch.empty(3 * max(p["n_ov"], 1), dtype=torch.float64, device=d["gt_f"].device)
    _lib.call("mdb_kitti_overlaps", d["gt_off"], d["dt_off"], d["ov_off"], p["n_img"], p["max_gt"], p["max_dt"], p["n_ov"],
              d["gt_f"], d["dt_f"], ov)
    return ov


def _to_device(p, classes=None, min_overlaps=None):
    names = ["gt_off", "dt_off", "ov_off", "gt_f", "gt_i", "dt_f", "dt_cls"]
    arrays = [p[k] for k in names]
    if classes is not None:
        names += ["classes", "min_overlaps"]
        arrays += [np.asarray(classes, dtype=np.int32), np.ascontiguousarray(min_overlaps, dtype=np.float64)]
    return dict(zip(names, _upload(arrays, _device())))


def image_overlaps(gt_annos, dt_annos):
    """Per-image overlap blocks, the parts of calculate_iou_partly(dt_annos, gt_annos, metric) (eval.py:415-489) that the
    reference reads: [metric][image] -> (n_dt, n_gt) fp64 array, metric 0 = bbox, 1 = BEV, 2 = 3d."""
    p = pack(gt_annos, dt_annos)
    ov = _launch_overlaps(p, _to_device(p)).cpu().numpy()
    n_ov, off = p["n_ov"], p["ov_off"]
    out = []
    for m in range(3):
        blocks = []
        for b in range(p["n_img"]):
            g = p["gt_off"][b + 1] - p["gt_off"][b]
            n = p["dt_off"][b + 1] - p["dt_off"][b]
            blocks.append(ov[m * n_ov + off[b]: m * n_ov + off[b + 1]].reshape(n, g))
        out.append(blocks)
    return out


def eval_counts(gt_annos, dt_annos, classes, min_overlaps, compute_aos):
    """The device pipeline: (n_cfg, 1 + 4 * 41) fp64 table, cfg = ((metric * n_cls + m) * 3 + difficulty) * 2 + k, row =
    [T, (tp, fp, fn, similarity) per threshold].  Six launches, one upload, one download."""
    classes = [int(c) for c in classes]
    if not classes or any(c not in CLASS_TO_NAME for c in classes):
        raise ValueError(f"kitti_eval: classes must be codes in 0..5, got {classes}")
    min_overlaps = np.asarray(min_overlaps, dtype=np.float64)
    if min_overlaps.shape != (2, 3, len(classes)):
        raise ValueError("kitti_eval: min_overlaps must have shape (2, 3, len(classes))")
    p = pack(gt_annos, dt_annos)
    d = _to_device(p, classes, min_overlaps)
    dev = d["gt_f"].device
    ov = _launch_overlaps(p, d)
    n_cls = len(classes)
    need = _lib.lib().mdb_kitti_eval_workspace_bytes(p["n_img"], p["n_gt"], p["n_dt"], n_cls, int(compute_aos))
    if need < 0:
        _lib.check(int(need), "mdb_kitti_eval_workspace_bytes")
    ws = torch.empty(max(int(need), 1), dtype=torch.uint8, device=dev)
    n_cfg = 18 * n_cls
    result = torch.empty(n_cfg, 1 + 4 * NUM_THRESH, dtype=torch.float64, device=dev)
    _lib.call("mdb_kitti_eval", d["gt_off"], d["dt_off"], d["ov_off"], p["n_img"], p["n_gt"], p["n_dt"], p["max_gt"], p["max_dt"],
              p["n_ov"], d["gt_f"], d["gt_i"], d["dt_f"], d["dt_cls"], ov, d["classes"], d["min_overlaps"], n_cls,
              int(compute_aos), ws, int(need), result, launches=5)
    table = result.cpu().numpy()
    if (table[:, 0] > NUM_THRESH).any():
        raise RuntimeError("kitti_eval: more than 41 score thresholds in a configuration (the reference fails on this input too)")
    return table


# ---------------------------------------------------------------------------------------------------------------- AP from counts
def _curves(table, n_cls, compute_aos):
    """precision / recall / aos (3 metrics, n_cls, 3, 2, 41) as eval_class (eval.py:614-624) builds them."""
    t = table.reshape(3, n_cls, 3, 2, 1 + 4 * NUM_THRESH)
    n_thr = t[..., 0].astype(np.int64)
    pr = t[..., 1:].reshape(3, n_cls, 3, 2, NUM_THRESH, 4)
    used = np.arange(NUM_THRESH) < n_thr[..., None]
    tp, fp, fn, sim = pr[..., 0], pr[..., 1], pr[..., 2], pr[..., 3]
    with np.errstate(divide="ignore", invalid="ignore"):
        recall = np.where(used, tp / (tp + fn), 0.0)
        precision = np.where(used, tp / (tp + fp), 0.0)
        aos = np.where(used, sim / (tp + fp), 0.0) if compute_aos else np.zeros_like(precision)

    def suffix_max(x):          # precision[i] = max(precision[i:]); the unused tail is 0 and every value >= 0 or NaN
        return np.maximum.accumulate(x[..., ::-1], axis=-1)[..., ::-1].copy()
    return suffix_max(precision), suffix_max(recall), suffix_max(aos)


def _map11(prec):               # eval.py:633-637
    s = 0
    for i in range(0, prec.shape[-1], 4):
        s = s + prec[..., i]
    return s / 11 * 100


def _map40(prec):               # eval.py:640-644
    s = 0
    for i in range(1, prec.shape[-1]):
        s = s + prec[..., i]
    return s / 40 * 100


def do_eval(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos=False, PR_detail_dict=None, DIForDIS=True):
    """(mAP_bbox, mAP_bev, mAP_3d, mAP_aos, mAP_bbox_R40, mAP_bev_R40, mAP_3d_R40, mAP_aos_R40), each (n_cls, 3 difficulties,
    2 overlap sets); the aos pair is None without compute_aos.  min_overlaps (2, 3, n_cls).  All metrics and classes in one
    device call."""
    if not DIForDIS:
        raise NotImplementedError("kitti_eval: the distance-binned evaluation (DIForDIS=False) is not implemented")
    n_cls = len(current_classes)
    table = eval_counts(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos)
    precision, _, aos = _curves(table, n_cls, compute_aos)
    out = {}
    for m, key in enumerate(("bbox", "bev", "3d")):
        out[key] = (_map11(precision[m]), _map40(precision[m]))
        if PR_detail_dict is not None:
            PR_detail_dict[key] = precision[m]
    mAP_aos = mAP_aos_R40 = None
    if compute_aos:
        mAP_aos, mAP_aos_R40 = _map11(aos[0]), _map40(aos[0])
        if PR_detail_dict is not None:
            PR_detail_dict["aos"] = aos[0]
    return (out["bbox"][0], out["bev"][0], out["3d"][0], mAP_aos, out["bbox"][1], out["bev"][1], out["3d"][1], mAP_aos_R40)


def _line(text):
    s = io.StringIO()
    print(text, file=s)
    return s.getvalue()


def _official(gt_annos, dt_annos, current_classes, PR_detail_dict=None):
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    classes = [NAME_TO_CLASS[c] if isinstance(c, str) else c for c in current_classes]
    min_overlaps = OFFICIAL_MIN_OVERLAPS[:, :, classes]
    compute_aos = False                                     # eval.py:745-751: the first image with detections decides
    for anno in dt_annos:
        if anno["alpha"].shape[0] != 0:
            compute_aos = bool(anno["alpha"][0] != -10)
            break
    bbox, bev, d3, aos, bbox40, bev40, d340, aos40 = do_eval(gt_annos, dt_annos, classes, min_overlaps, compute_aos,
                                                             PR_detail_dict=PR_detail_dict)
    texts, ret = [], {}
    for j, c in enumerate(classes):
        name, text = CLASS_TO_NAME[c], ""
        for i in range(min_overlaps.shape[0]):
            thr = "{:.2f}, {:.2f}, {:.2f}:".format(*min_overlaps[i, :, j])
            for tag, curves in (("AP", (bbox, bev, d3, aos)), ("AP_R40", (bbox40, bev40, d340, aos40))):
                text += _line(f"{name} {tag}@{thr}")
                for label, v in zip(("bbox", "bev ", "3d  "), curves[:3]):
                    text += _line(f"{label} AP:{v[j, 0, i]:.4f}, {v[j, 1, i]:.4f}, {v[j, 2, i]:.4f}")
                if compute_aos:
                    v = curves[3]
                    text += _line(f"aos  AP:{v[j, 0, i]:.2f}, {v[j, 1, i]:.2f}, {v[j, 2, i]:.2f}")
                    if i == 0:
                        sfx = "" if tag == "AP" else "_R40"
                        for l, diff in enumerate(("easy", "moderate", "hard")):
                            ret[f"{name}_aos_{diff}{sfx}"] = v[j, l, 0]
            if i == 0:
                for sfx, curves in (("", (d3, bev, bbox)), ("_R40", (d340, bev40, bbox40))):
                    for key, v in zip(("3d", "bev", "image"), curves):
                        for l, diff in enumerate(("easy", "moderate", "hard")):
                            ret[f"{name}_{key}_{diff}{sfx}"] = v[j, l, 0]
        texts.append(text)
    return texts, ret, d340[0, 1, 0], classes


def get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None):
    """(result string, dict of APs, AP3d R40 of the first class at moderate difficulty and the strict overlap set), as the
    reference.  current_classes: a class code, a name ('Car', ...) or a list of them."""
    texts, ret, first, _ = _official(gt_annos, dt_annos, current_classes, PR_detail_dict)
    return "".join(texts), ret, first


def evaluate(results_dir, label_dir, image_ids, classes=("Car", "Pedestrian", "Cyclist"), logger=None):
    """KITTI_Dataset.eval: reads the detections of `results_dir` (every %06d.txt) and the labels of `image_ids` from `label_dir`,
    logs each class's result string and returns Car AP3d R40 at moderate difficulty (0 when 'Car' is not evaluated).  All
    classes are evaluated in one device call."""
    logger = logger or logging.getLogger(__name__)
    logger.info("==> Loading detections and GTs...")
    dt_annos = get_label_annos(results_dir)
    gt_annos = get_label_annos(label_dir, [int(i) for i in image_ids])
    logger.info("==> Evaluating (official) ...")
    texts, ret, _, codes = _official(gt_annos, dt_annos, list(classes))
    for t in texts:
        logger.info(t)
    return ret["Car_3d_moderate_R40"] if NAME_TO_CLASS["Car"] in codes else 0
