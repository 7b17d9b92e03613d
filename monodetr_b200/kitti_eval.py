"""KITTI object-detection metric on the device, behind the reference's function names (SURVEY.md 2).

  get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None)
                                       lib/datasets/kitti/kitti_eval_python/eval.py:717-825
  get_distance_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None)
                                       eval.py:828-936 (AP per distance bin 0-30 / 30-50 / 50-70 m)
  do_eval(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos=False, PR_detail_dict=None, DIForDIS=True)
                                       eval.py:656-696 (DIForDIS=False: distance bins, eval.py:85-159)
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

`GroundTruth` + `DeviceEvaluator` run the validation pass without result files: the decoded detections of each batch are
collected into a device table (csrc/kitti_eval.cu mdb_kitti_collect_dets_f32), compacted at the end of the pass and evaluated by
the same kernels (`eval_device_tables`); `DeviceEvaluator.distance_result` gives the distance-binned report of the same table.
"""
import io
import logging
import os
import pathlib
import re

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from .ddp import rank_world

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


def _offsets(counts, dtype=np.int32):
    return np.concatenate([[0], np.cumsum(counts)]).astype(dtype)


def pack_gt(gt_annos):
    """The ground-truth half of `pack`: gt_off, gt_f, gt_i, n_gt, max_gt and the per-image counts `ng`."""
    if len(gt_annos) == 0:
        raise ValueError("kitti_eval: no images")
    ng = np.array([len(a["name"]) for a in gt_annos], dtype=np.int64)
    gt_f = [np.concatenate([_col(a, "bbox", n, 4), _col(a, "alpha", n), _col(a, "truncated", n), _col(a, "location", n, 3),
                            _col(a, "dimensions", n, 3), _col(a, "rotation_y", n)], 1) for a, n in zip(gt_annos, ng)]
    gt_i = [np.stack([np.asarray(a["occluded"], dtype=np.int64).reshape(n),
                      np.array([_class_code(s) for s in a["name"]], dtype=np.int64).reshape(n),
                      np.array([s == "DontCare" for s in a["name"]], dtype=np.int64).reshape(n)], 1) for a, n in zip(gt_annos, ng)]
    return {"gt_off": _offsets(ng), "ng": ng,
            "gt_f": np.ascontiguousarray(np.concatenate(gt_f, 0), dtype=np.float64).reshape(-1, GT_COLS),
            "gt_i": np.ascontiguousarray(np.concatenate(gt_i, 0), dtype=np.int32).reshape(-1, 3),
            "n_img": len(gt_annos), "n_gt": int(ng.sum()), "max_gt": int(ng.max())}


def pack_dt(dt_annos):
    """The detection half of `pack`: dt_off, dt_f, dt_cls, n_dt, max_dt and the per-image counts `nd`."""
    nd = np.array([len(a["name"]) for a in dt_annos], dtype=np.int64)
    dt_f = [np.concatenate([_col(a, "bbox", n, 4), _col(a, "alpha", n), _col(a, "score", n), _col(a, "location", n, 3),
                            _col(a, "dimensions", n, 3), _col(a, "rotation_y", n)], 1) for a, n in zip(dt_annos, nd)]
    dt_cls = [np.array([_class_code(s) for s in a["name"]], dtype=np.int64).reshape(n) for a, n in zip(dt_annos, nd)]
    return {"dt_off": _offsets(nd), "nd": nd,
            "dt_f": np.ascontiguousarray(np.concatenate(dt_f, 0), dtype=np.float64).reshape(-1, DT_COLS),
            "dt_cls": np.ascontiguousarray(np.concatenate(dt_cls, 0), dtype=np.int32),
            "n_dt": int(nd.sum()), "max_dt": int(nd.max())}


def pair_sizes(ng, nd):
    """ov_off (per-image overlap block offsets) and n_ov from the per-image gt / detection counts."""
    ov_off = _offsets(np.asarray(ng, np.int64) * np.asarray(nd, np.int64), np.int64)
    return {"ov_off": ov_off, "n_ov": int(ov_off[-1])}


def pack(gt_annos, dt_annos):
    """CSR tables of include/monodetr_b200.h (mdb_kitti_*): offsets, gt_f / gt_i / dt_f / dt_cls, and the HOST sizes."""
    if len(gt_annos) != len(dt_annos):
        raise ValueError("kitti_eval: gt_annos and dt_annos must list the same images")
    g, d = pack_gt(gt_annos), pack_dt(dt_annos)
    p = {**g, **d, **pair_sizes(g["ng"], d["nd"])}
    del p["ng"], p["nd"]
    return p


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


def _check_classes(classes, min_overlaps):
    classes = [int(c) for c in classes]
    if not classes or any(c not in CLASS_TO_NAME for c in classes):
        raise ValueError(f"kitti_eval: classes must be codes in 0..5, got {classes}")
    min_overlaps = np.asarray(min_overlaps, dtype=np.float64)
    if min_overlaps.shape != (2, 3, len(classes)):
        raise ValueError("kitti_eval: min_overlaps must have shape (2, 3, len(classes))")
    return classes, min_overlaps


def eval_counts(gt_annos, dt_annos, classes, min_overlaps, compute_aos, by_distance=False):
    """The device pipeline: (n_cfg, 1 + 4 * 41) fp64 table, cfg = ((metric * n_cls + m) * 3 + difficulty) * 2 + k, row =
    [T, (tp, fp, fn, similarity) per threshold].  by_distance: the third index is the distance bin (0-30, 30-50, 50-70 m) of
    clean_data_by_distance instead of the difficulty.  Six launches, one upload, one download."""
    classes, min_overlaps = _check_classes(classes, min_overlaps)
    p = pack(gt_annos, dt_annos)
    return eval_device_tables(_to_device(p, classes, min_overlaps), p, len(classes), compute_aos, by_distance)


def eval_device_tables(d, p, n_cls, compute_aos, by_distance=False):
    """The counts table of `eval_counts` from tables already on the device: `d` holds the device arrays gt_off, dt_off, ov_off,
    gt_f, gt_i, dt_f, dt_cls, classes and min_overlaps, `p` the HOST sizes n_img, n_gt, n_dt, n_ov, max_gt, max_dt.  Every
    evaluation (annotation lists or the device table of `DeviceEvaluator`) launches the eval kernels here: six launches, one
    download.  by_distance selects mdb_kitti_eval_distance (distance bins) over mdb_kitti_eval (difficulties)."""
    dev = d["gt_f"].device
    ov = _launch_overlaps(p, d)
    need = _lib.lib().mdb_kitti_eval_workspace_bytes(p["n_img"], p["n_gt"], p["n_dt"], n_cls, int(compute_aos))
    if need < 0:
        _lib.check(int(need), "mdb_kitti_eval_workspace_bytes")
    ws = torch.empty(max(int(need), 1), dtype=torch.uint8, device=dev)
    n_cfg = 18 * n_cls
    result = torch.empty(n_cfg, 1 + 4 * NUM_THRESH, dtype=torch.float64, device=dev)
    _lib.call("mdb_kitti_eval_distance" if by_distance else "mdb_kitti_eval", d["gt_off"], d["dt_off"], d["ov_off"], p["n_img"], p["n_gt"], p["n_dt"], p["max_gt"], p["max_dt"],
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
    2 overlap sets); the aos pair is None without compute_aos.  min_overlaps (2, 3, n_cls).  DIForDIS=False: the 3 distance bins
    0-30 / 30-50 / 50-70 m (clean_data_by_distance) in place of the difficulties.  All metrics and classes in one device call."""
    table = eval_counts(gt_annos, dt_annos, current_classes, min_overlaps, compute_aos, by_distance=not DIForDIS)
    return _aps(table, len(current_classes), compute_aos, PR_detail_dict)


def _aps(table, n_cls, compute_aos, PR_detail_dict=None):
    """do_eval's result from the counts table."""
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


def _class_codes(current_classes):
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    return [NAME_TO_CLASS[c] if isinstance(c, str) else c for c in current_classes]


DIFFICULTY_KEYS = ("easy", "moderate", "hard")          # ret_dict key parts of the third index: get_official_eval_result
DISTANCE_KEYS = ("30m", "50m", "70m")                    # and get_distance_eval_result (eval.py:890-934)


def _official(gt_annos, dt_annos, current_classes, PR_detail_dict=None, by_distance=False):
    classes = _class_codes(current_classes)
    min_overlaps = OFFICIAL_MIN_OVERLAPS[:, :, classes]
    compute_aos = False                                     # eval.py:745-751: the first image with detections decides
    for anno in dt_annos:
        if anno["alpha"].shape[0] != 0:
            compute_aos = bool(anno["alpha"][0] != -10)
            break
    aps = do_eval(gt_annos, dt_annos, classes, min_overlaps, compute_aos, PR_detail_dict=PR_detail_dict, DIForDIS=not by_distance)
    return _report(classes, min_overlaps, aps, compute_aos, DISTANCE_KEYS if by_distance else DIFFICULTY_KEYS)


def _report(classes, min_overlaps, aps, compute_aos, levels=DIFFICULTY_KEYS):
    """get_official_eval_result's (levels = DIFFICULTY_KEYS) or get_distance_eval_result's (DISTANCE_KEYS) per-class result
    strings, ret_dict and first value from do_eval's arrays; the two reports differ only in the ret_dict keys."""
    bbox, bev, d3, aos, bbox40, bev40, d340, aos40 = aps
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
                        for l, diff in enumerate(levels):
                            ret[f"{name}_aos_{diff}{sfx}"] = v[j, l, 0]
            if i == 0:
                for sfx, curves in (("", (d3, bev, bbox)), ("_R40", (d340, bev40, bbox40))):
                    for key, v in zip(("3d", "bev", "image"), curves):
                        for l, diff in enumerate(levels):
                            ret[f"{name}_{key}_{diff}{sfx}"] = v[j, l, 0]
        texts.append(text)
    return texts, ret, d340[0, 1, 0], classes


def get_official_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None):
    """(result string, dict of APs, AP3d R40 of the first class at moderate difficulty and the strict overlap set), as the
    reference.  current_classes: a class code, a name ('Car', ...) or a list of them."""
    texts, ret, first, _ = _official(gt_annos, dt_annos, current_classes, PR_detail_dict)
    return "".join(texts), ret, first


def get_distance_eval_result(gt_annos, dt_annos, current_classes, PR_detail_dict=None):
    """(result string, dict of APs) of the distance-binned evaluation, as the reference (eval.py:828-936): the report of
    get_official_eval_result with the bins 0-30 / 30-50 / 50-70 m in place of easy / moderate / hard, and ret_dict keys
    `<Class>_{3d,bev,image,aos}_{30m,50m,70m}[_R40]`.  Every bin uses the hard level's occlusion / truncation / height limits."""
    texts, ret, _, _ = _official(gt_annos, dt_annos, current_classes, PR_detail_dict, by_distance=True)
    return "".join(texts), ret


def evaluate(results_dir, label_dir, image_ids, classes=("Car", "Pedestrian", "Cyclist"), logger=None):
    """KITTI_Dataset.eval: reads the detections of `results_dir` (every %06d.txt) and the labels of `image_ids` from `label_dir`,
    logs each class's result string and returns Car AP3d R40 at moderate difficulty (0 when 'Car' is not evaluated).  All
    classes are evaluated in one device call."""
    logger = logger or logging.getLogger(__name__)
    logger.info("==> Loading detections and GTs...")
    dt_annos = get_label_annos(results_dir)
    gt_annos = get_label_annos(label_dir, [int(i) for i in image_ids])
    logger.info("==> Evaluating (official) ...")
    return _log_result(logger, *_official(gt_annos, dt_annos, list(classes)))


def _log_result(logger, texts, ret, first, codes):
    for t in texts:
        logger.info(t)
    return ret["Car_3d_moderate_R40"] if NAME_TO_CLASS["Car"] in codes else 0


# ---------------------------------------------------------------------------------------------------------------- validation pass
TESTER_CLASS_NAMES = ("Pedestrian", "Car", "Cyclist")   # kitti_dataset.py:30: the decode class id indexes this list
ROW_COLS = 14                                            # decode.OUT_COLS
COLLECT_MAX_BATCH = 512                                  # MDB_KITTI_COLLECT_MAX_BATCH
COLLECT_MAX_CLASSES = 8                                  # MDB_KITTI_COLLECT_MAX_CLASSES
# result-file field order (tester_helper.py:125-132: alpha, bbox, h w l, location, ry, score) as dt_f columns
_FILE_FROM_DT = [4, 0, 1, 2, 3, 10, 11, 9, 6, 7, 8, 12, 5]


_RESULT_LINE = "{} 0.0 0" + " {:.2f}" * DT_COLS + "\n"


def result_file_text(rows, class_names):
    """The text Tester.save_results (tester_helper.py:125-132) writes for one image: rows [class id, value, ...] as
    decode_detections returns them, the class id indexing `class_names`."""
    return "".join("{} 0.0 0".format(class_names[int(r[0])]) + "".join(" {:.2f}".format(v) for v in r[1:]) + "\n" for r in rows)


def _carve(specs, device):
    """One device buffer holding several arrays, each 16-byte aligned: (buffer, typed views, byte offsets)."""
    offs, size = [], 0
    for dtype, shape in specs:
        offs.append(size)
        size += (int(np.prod(shape)) * torch.empty(0, dtype=dtype).element_size() + 15) // 16 * 16
    buf = torch.zeros(max(size, 16), dtype=torch.uint8, device=device)
    views = [buf[o:o + int(np.prod(s)) * torch.empty(0, dtype=t).element_size()].view(t).view(*s)
             for (t, s), o in zip(specs, offs)]
    return buf, views, offs


class GroundTruth:
    """The labels of a split, parsed once at fp64 (as KITTI_Dataset.eval parses them with kitti_common.get_label_annos) and kept
    on the device in the CSR form of mdb_kitti_eval, so that every validation pass reuses them.  Image i is the i-th id of
    `image_ids`."""

    def __init__(self, gt_annos, image_ids=None, device=None):
        p = pack_gt(gt_annos)
        self.image_ids = list(range(len(gt_annos))) if image_ids is None else [int(i) for i in image_ids]
        if len(self.image_ids) != len(gt_annos):
            raise ValueError("GroundTruth: image_ids and gt_annos must have the same length")
        self.ng = p["ng"]
        self.n_img, self.n_gt, self.max_gt = p["n_img"], p["n_gt"], p["max_gt"]
        self.device = device or _device()
        self.gt_off, self.gt_f, self.gt_i = _upload([p["gt_off"], p["gt_f"], p["gt_i"]], self.device)

    @classmethod
    def from_annos(cls, gt_annos, image_ids=None, device=None):
        return cls(gt_annos, image_ids, device)

    @classmethod
    def from_kitti(cls, root_dir, split, device=None):
        """Every image of ImageSets/<split>.txt, labels from training/label_2 (kitti_dataset.py:49-60)."""
        if split == "test":
            raise ValueError("GroundTruth.from_kitti: the test split has no labels")
        with open(os.path.join(root_dir, "ImageSets", split + ".txt")) as f:
            ids = [int(x.strip()) for x in f.readlines()]
        return cls(get_label_annos(os.path.join(root_dir, "training", "label_2"), ids), ids, device)


class DeviceEvaluator:
    """One validation pass on the device: the decoded detections of every image go into a padded device table in the form the
    result files would give them back (values rounded as '{:.2f}' and parsed again), and the KITTI AP is computed from that table
    with the kernels of `evaluate`.  The result files are only needed for submission (`write_results`).

    Images are paired by their position in the split (`slots`): the reference pairs the sorted ids of its result files with the
    split's id list, and the two orders agree because KITTI's ImageSets files list ids in ascending order.

      gt           GroundTruth of the split, or None (no `result()`, e.g. the test split: then pass `image_ids`)
      classes      the classes `result()` evaluates (KITTI_Dataset.writelist), names or codes
      class_names  the decode class id -> name list of the tester (kitti_dataset.py:30)

    `add` runs extract + decode + collect (three launches on the current stream, no host synchronisation); `result` copies the
    per-image counts to the host once, compacts the table and runs the eval; `reset` starts the next pass; `merge` combines
    the tables of a pass whose images were split over the ranks of a process group."""

    def __init__(self, gt, classes=("Car",), topk=50, threshold=0.2, cls_mean_size=None, class_names=TESTER_CLASS_NAMES,
                 image_ids=None, device=None):
        from .labels import CLS_MEAN_SIZE
        self.gt = gt
        if image_ids is None:
            if gt is None:
                raise ValueError("DeviceEvaluator: pass a GroundTruth or image_ids")
            image_ids = gt.image_ids
        self.image_ids = [int(i) for i in image_ids]
        if gt is not None and len(self.image_ids) != gt.n_img:
            raise ValueError("DeviceEvaluator: image_ids must list the images of gt")
        self.n_img = len(self.image_ids)
        self.classes = _class_codes(list(classes) if isinstance(classes, (list, tuple)) else classes)
        self.min_overlaps = OFFICIAL_MIN_OVERLAPS[:, :, self.classes]
        _check_classes(self.classes, self.min_overlaps)
        self.class_names = list(class_names)
        codes = [_class_code(n) for n in self.class_names]
        if any(c < 0 for c in codes) or len(set(codes)) != len(codes) or len(codes) > COLLECT_MAX_CLASSES:
            raise ValueError(f"DeviceEvaluator: class_names must be distinct KITTI class names, got {self.class_names}")
        self.codes = np.array(codes, np.int32)
        self.topk, self.threshold = int(topk), float(threshold)
        if not 1 <= self.topk <= MAX_BOXES:
            raise ValueError(f"DeviceEvaluator: topk must be in 1..{MAX_BOXES}")
        self.device = device or (gt.device if gt is not None else _device())
        mean = np.asarray(CLS_MEAN_SIZE if cls_mean_size is None else cls_mean_size, np.float32)
        self.cls_mean_size = torch.from_numpy(mean).to(self.device)     # uploaded once: a per-batch upload would synchronise
        self._buf, (self.slot_info, self.table_f, self.table_cls), self._offs = _carve(
            [(torch.int32, (3, self.n_img)), (torch.float64, (self.n_img, self.topk, DT_COLS)),
             (torch.int32, (self.n_img, self.topk))], self.device)
        self._eval_consts = None

    def reset(self):
        """Starts a pass.  In a single process only the per-slot counts are cleared.  With torch.distributed initialised and
        more than one rank, the whole table is zeroed, so that the rows this rank does not add stay zero for `merge`."""
        if rank_world()[1] > 1:
            self._buf.zero_()
        else:
            self.slot_info.zero_()

    def merge(self):
        """Gives every rank the table of the whole pass, after each rank has added its own images: one all-reduce (sum) of
        the table on the process group's backend.  Nothing happens in a single process.

        The sum is exact.  `reset` zeroed every byte, and an image's rows and slot_info entries are written only by the rank
        that added it, so when every image is added once, every byte of the table is non-zero on at most one rank.  The
        buffer is summed as int64 words: an integer sum of words whose non-zero bytes are disjoint is their bitwise OR, with
        no carry, so each rank's bits arrive unchanged.  A float sum would not do: it turns a -0.0 (a rounded value such as
        -0.001) into +0.0, and the result file would print "0.00" for the reference's "-0.00".  An image added on two
        ranks, or on none, still shows in slot_info's add count (small int32s, summed without carry), so `result()` and
        `write_results()` raise as in a single process."""
        if rank_world()[1] > 1:
            dist.all_reduce(self._buf.view(torch.int64), op=dist.ReduceOp.SUM)

    # ------------------------------------------------------------------------------------------------------------ per batch
    def add(self, outputs, slots, img_size, calibs):
        """outputs: MonoDETR.forward's dict of one batch; slots: the batch images' positions in the split (host integers);
        img_size (B, 2) and calibs (B, 3, 4) or Calibration objects, as decode_detections takes them."""
        from . import decode
        dets = decode.extract_dets_from_outputs(outputs, topk=self.topk)
        rows, count = decode.decode_detections_device(dets, img_size, calibs, self.cls_mean_size, self.threshold)
        self.add_rows(rows, count, slots)

    def add_rows(self, rows, count, slots):
        """rows (B, topk, 14) / count (B) as decode_detections_device returns them."""
        if isinstance(slots, torch.Tensor) and slots.device.type != "cpu":
            raise TypeError("DeviceEvaluator: slots must be host integers (reading device slots would synchronise)")
        slots = np.ascontiguousarray(np.asarray(slots, dtype=np.int64).reshape(-1)).astype(np.int32)
        if rows.shape != (len(slots), self.topk, ROW_COLS) or count.shape != (len(slots),):
            raise ValueError(f"DeviceEvaluator: rows (B, {self.topk}, {ROW_COLS}) and count (B,) expected for {len(slots)} slots")
        rows, count = rows.float().contiguous(), count.int().contiguous()
        with torch.cuda.device(self.device):
            _lib.call("mdb_kitti_collect_dets_f32", rows, count, slots.ctypes.data, len(slots), self.topk, self.n_img,
                      self.codes.ctypes.data, len(self.codes), self.table_f, self.table_cls, self.slot_info,
                      launches=-(-len(slots) // COLLECT_MAX_BATCH))

    # ------------------------------------------------------------------------------------------------------------ end of a pass
    def _host_info(self, nbytes=None):
        """One device->host copy of the buffer's first `nbytes` (all of it by default): (slot_info, bytes)."""
        host = self._buf[:nbytes].cpu().numpy() if nbytes else self._buf.cpu().numpy()
        info = host[:3 * self.n_img * 4].view(np.int32).reshape(3, self.n_img)
        added = info[1]
        if (added != 1).any():
            twice, missing = np.flatnonzero(added > 1), np.flatnonzero(added == 0)
            msg = []
            if len(twice):
                msg.append(f"{len(twice)} image(s) added more than once (first id {self.image_ids[twice[0]]})")
            if len(missing):
                msg.append(f"{len(missing)} image(s) never added (first id {self.image_ids[missing[0]]})")
            raise ValueError("DeviceEvaluator: " + "; ".join(msg))
        return info, host

    def counts_table(self, by_distance=False):
        """The (n_cfg, 1 + 4 * 41) counts table of eval_counts for this pass (by_distance: the distance-binned one), and
        compute_aos."""
        if self.gt is None:
            raise ValueError("DeviceEvaluator: no GroundTruth, nothing to evaluate against")
        info, _ = self._host_info(3 * self.n_img * 4)                         # the one synchronisation of the pass
        nd = info[0].astype(np.int64)
        with_dets = np.flatnonzero(nd)
        compute_aos = bool(info[2][with_dets[0]]) if len(with_dets) else False   # eval.py:745-751
        sizes = {"n_img": self.n_img, "n_gt": self.gt.n_gt, "n_dt": int(nd.sum()), "max_gt": self.gt.max_gt,
                 "max_dt": int(nd.max()), **pair_sizes(self.gt.ng, nd)}
        if self._eval_consts is None:
            self._eval_consts = _upload([np.asarray(self.classes, np.int32), self.min_overlaps], self.device)
        dt_off, ov_off = _upload([_offsets(nd), sizes["ov_off"]], self.device)
        dt_f = torch.empty(max(sizes["n_dt"], 1), DT_COLS, dtype=torch.float64, device=self.device)
        dt_cls = torch.empty(max(sizes["n_dt"], 1), dtype=torch.int32, device=self.device)
        d = {"gt_off": self.gt.gt_off, "dt_off": dt_off, "ov_off": ov_off, "gt_f": self.gt.gt_f, "gt_i": self.gt.gt_i,
             "dt_f": dt_f, "dt_cls": dt_cls, "classes": self._eval_consts[0], "min_overlaps": self._eval_consts[1]}
        with torch.cuda.device(self.device):
            _lib.call("mdb_kitti_compact_dets", dt_off, self.table_f, self.table_cls, self.n_img, self.topk, dt_f, dt_cls)
            return eval_device_tables(d, sizes, len(self.classes), compute_aos, by_distance), compute_aos

    def result(self, logger=None):
        """What `evaluate` (KITTI_Dataset.eval) returns for this pass -- Car AP3d R40 at moderate difficulty, 0 when 'Car' is not
        among `classes` -- with the same log lines.  ValueError if an image was added twice or never."""
        logger = logger or logging.getLogger(__name__)
        logger.info("==> Loading detections and GTs...")
        table, compute_aos = self.counts_table()
        logger.info("==> Evaluating (official) ...")
        aps = _aps(table, len(self.classes), compute_aos)
        return _log_result(logger, *_report(self.classes, self.min_overlaps, aps, compute_aos))

    def distance_result(self, logger=None):
        """What get_distance_eval_result returns for this pass's detections and `classes` -- (result string, ret_dict) -- from
        the device table, without result files.  With a logger, each class's part of the result string is logged.  The same
        errors as `result`."""
        table, compute_aos = self.counts_table(by_distance=True)
        aps = _aps(table, len(self.classes), compute_aos)
        texts, ret, _, _ = _report(self.classes, self.min_overlaps, aps, compute_aos, DISTANCE_KEYS)
        if logger is not None:
            for t in texts:
                logger.info(t)
        return "".join(texts), ret

    def result_lines(self, class_names=None):
        """{image id: text of its result file} as the reference's Tester.save_results writes it, from one device->host copy."""
        names = self.class_names if class_names is None else list(class_names)
        decode_id = {int(c): i for i, c in enumerate(self.codes)}
        info, host = self._host_info()
        f = host[self._offs[1]:self._offs[1] + self.table_f.numel() * 8].view(np.float64).reshape(self.n_img, self.topk, DT_COLS)
        c = host[self._offs[2]:self._offs[2] + self.table_cls.numel() * 4].view(np.int32).reshape(self.n_img, self.topk)
        fmt = _RESULT_LINE
        out = {}
        for s, img_id in enumerate(self.image_ids):
            n = int(info[0, s])
            vals = f[s, :n][:, _FILE_FROM_DT].tolist()
            out[img_id] = "".join(fmt.format(names[decode_id[int(k)]], *v) for k, v in zip(c[s, :n], vals))
        return out

    def write_results(self, results_dir, class_names=None):
        """Writes <results_dir>/%06d.txt for every image, byte-identical to the reference's Tester.save_results
        (tester_helper.py:112-132) on the same decoded rows.  Works without a GroundTruth (test split)."""
        os.makedirs(results_dir, exist_ok=True)
        for img_id, text in self.result_lines(class_names).items():
            with open(os.path.join(results_dir, "{:06d}.txt".format(img_id)), "w") as f:
                f.write(text)
