"""CPU numpy restatement of the KITTI evaluation (the reference's lib/datasets/kitti/kitti_eval_python/eval.py and
rotate_iou.py), the yardstick of monodetr_b200/kitti_eval.py and csrc/kitti_eval.cu.

Arithmetic as in the reference: fp64 for the 2-d overlap, the 3-d height overlap / volumes and the statistics; the rotated
(bird's-eye-view) intersection in fp32 scalar arithmetic (np.float32 operands; under NumPy >= 2 a Python float combined with a
float32 stays float32, as in numba's CUDA simulator that produced tests/golden/kitti_eval.npz).  Pinned against that file by
tests/test_oracle_kitti_eval.py.  The statistics loops are vectorised over detections and thresholds, never reordered in a way
that changes a result: every choice keeps the reference's lowest-index rule and every fp64 sum keeps its order.
"""
import math

import numpy as np

CLASS_NAMES = ("car", "pedestrian", "cyclist", "van", "person_sitting", "truck")   # eval.py:31
MIN_HEIGHT = (40, 25, 25)                                                          # eval.py:32-34
MAX_OCCLUSION = (0, 1, 2)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
N_SAMPLE_PTS = 41                                                                  # eval.py:552
NO_DETECTION = -10000000                                                           # eval.py:259
F32 = np.float32


# ------------------------------------------------------------------------------------------------------------------ overlaps
def image_box_overlap(boxes, qboxes, criterion=-1):
    """eval.py:162-189: (N, K) fp64, boxes (N, 4), qboxes (K, 4) as x0 y0 x1 y1."""
    out = np.zeros((len(boxes), len(qboxes)), dtype=np.float64)
    for k, q in enumerate(qboxes):
        qarea = (q[2] - q[0]) * (q[3] - q[1])
        for n, b in enumerate(boxes):
            iw = min(b[2], q[2]) - max(b[0], q[0])
            if iw > 0:
                ih = min(b[3], q[3]) - max(b[1], q[1])
                if ih > 0:
                    barea = (b[2] - b[0]) * (b[3] - b[1])
                    ua = barea + qarea - iw * ih if criterion == -1 else (barea if criterion == 0 else qarea)
                    out[n, k] = iw * ih / ua
    return out


def _corners(rb):
    """rotate_iou.py:204-228: 4 corners of [x, y, dx, dy, angle] (fp32)."""
    a_cos, a_sin = F32(math.cos(float(rb[4]))), F32(math.sin(float(rb[4])))
    hx, hy = -rb[2] / F32(2), -rb[3] / F32(2)
    xs, ys = (hx, hx, -hx, -hx), (hy, -hy, -hy, hy)
    c = []
    for x, y in zip(xs, ys):
        c.append(a_cos * x + a_sin * y + rb[0])
        c.append(-a_sin * x + a_cos * y + rb[1])
    return c


def _in_quad(px, py, c):
    """rotate_iou.py:161-177."""
    ab0, ab1, ad0, ad1 = c[2] - c[0], c[3] - c[1], c[6] - c[0], c[7] - c[1]
    ap0, ap1 = px - c[0], py - c[1]
    abab, abap = ab0 * ab0 + ab1 * ab1, ab0 * ap0 + ab1 * ap1
    adad, adap = ad0 * ad0 + ad1 * ad1, ad0 * ap0 + ad1 * ap1
    return abab >= abap and abap >= 0 and adad >= adap and adap >= 0


def _segment(p1, p2, i, j):
    """rotate_iou.py:73-116: intersection of edge i of p1 with edge j of p2, or None."""
    A0, A1 = p1[2 * i], p1[2 * i + 1]
    B0, B1 = p1[2 * ((i + 1) % 4)], p1[2 * ((i + 1) % 4) + 1]
    C0, C1 = p2[2 * j], p2[2 * j + 1]
    D0, D1 = p2[2 * ((j + 1) % 4)], p2[2 * ((j + 1) % 4) + 1]
    BA0, BA1, DA0, CA0, DA1, CA1 = B0 - A0, B1 - A1, D0 - A0, C0 - A0, D1 - A1, C1 - A1
    acd = DA1 * CA0 > CA1 * DA0
    bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0)
    if acd == bcd:
        return None
    abc = CA1 * BA0 > BA1 * CA0
    abd = DA1 * BA0 > BA1 * DA0
    if abc == abd:
        return None
    DC0, DC1 = D0 - C0, D1 - C1
    ABBA, CDDC = A0 * B1 - B0 * A1, C0 * D1 - D0 * C1
    DH = BA1 * DC0 - BA0 * DC1
    return (ABBA * DC0 - BA0 * CDDC) / DH, (ABBA * DC1 - BA1 * CDDC) / DH


def _triangle_area(a, b, c):
    """rotate_iou.py:17-20: signed area of the triangle (a, b, c)."""
    return ((a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0])) / F32(2)


def rotated_intersection(rb1, rb2):
    """rotate_iou.py:231-245: area of the intersection of two rotated boxes, fp32 (rb = [x, y, dx, dy, angle] float32)."""
    c1, c2 = _corners(rb1), _corners(rb2)
    pts = []
    for i in range(4):                                               # rotate_iou.py:180-201
        if _in_quad(c1[2 * i], c1[2 * i + 1], c2):
            pts.append([c1[2 * i], c1[2 * i + 1]])
        if _in_quad(c2[2 * i], c2[2 * i + 1], c1):
            pts.append([c2[2 * i], c2[2 * i + 1]])
    for i in range(4):
        for j in range(4):
            t = _segment(c1, c2, i, j)
            if t is not None:
                pts.append(list(t))
    # The reference's int_pts holds 8 points.  A degenerate pair can give more (the same box with its heading flipped between
    # float32(pi / 2) and float32(-pi / 2)): the reference's simulator run raises there and its GPU run writes past a local
    # array.  Here, as in csrc/kitti_eval.cu, the first 8 candidates in the reference's order are kept.
    pts = pts[:8]
    n = len(pts)
    if n > 0:                                                        # rotate_iou.py:33-70 (insertion sort by pseudo-angle)
        cx, cy = F32(0), F32(0)
        for p in pts:
            cx, cy = cx + p[0], cy + p[1]
        cx, cy = cx / F32(n), cy / F32(n)
        vs = []
        for p in pts:
            v0, v1 = p[0] - cx, p[1] - cy
            d = F32(math.sqrt(float(v0 * v0 + v1 * v1)))
            with np.errstate(invalid="ignore", divide="ignore"):          # a repeated vertex: 0 / 0, as in the reference
                v0, v1 = v0 / d, v1 / d
            if v1 < 0:
                v0 = F32(-2) - v0
            vs.append(v0)
        for i in range(1, n):
            if vs[i - 1] > vs[i]:
                tmp, tp = vs[i], pts[i]
                j = i
                while j > 0 and vs[j - 1] > tmp:
                    vs[j], pts[j] = vs[j - 1], pts[j - 1]
                    j -= 1
                vs[j], pts[j] = tmp, tp
    area = F32(0)                                                    # rotate_iou.py:17-30
    for i in range(n - 2):
        area = area + abs(_triangle_area(pts[0], pts[i + 1], pts[i + 2]))
    return area


def image_overlaps(gt, dt):
    """The three (n_dt, n_gt) blocks of one image, as calculate_iou_partly(dt_annos, gt_annos, metric) (eval.py:415-489,
    called from :550) returns them: bbox fp64; BEV and 3d rounded through fp32, widened to fp64."""
    ng, nd = len(gt["name"]), len(dt["name"])
    o2 = image_box_overlap(np.asarray(dt["bbox"], np.float64).reshape(nd, 4), np.asarray(gt["bbox"], np.float64).reshape(ng, 4))

    def box7(a, n):       # [x, y, z, l, h, w, ry]
        return np.concatenate([np.asarray(a["location"], np.float64).reshape(n, 3), np.asarray(a["dimensions"], np.float64).reshape(n, 3),
                               np.asarray(a["rotation_y"], np.float64).reshape(n, 1)], 1)
    g7, d7 = box7(gt, ng), box7(dt, nd)
    g5, d5 = g7[:, [0, 2, 3, 5, 6]].astype(np.float32), d7[:, [0, 2, 3, 5, 6]].astype(np.float32)
    obev = np.zeros((nd, ng), np.float32)
    o3 = np.zeros((nd, ng), np.float32)
    for j in range(nd):
        for i in range(ng):
            inter = rotated_intersection(g5[i], d5[j])              # devRotateIoUEval(query = gt, box = dt)
            obev[j, i] = inter / (g5[i, 2] * g5[i, 3] + d5[j, 2] * d5[j, 3] - inter)
            r = inter                                                # eval.py:197-223, boxes = dt, qboxes = gt
            if r > 0:
                iw = min(d7[j, 1], g7[i, 1]) - max(d7[j, 1] - d7[j, 4], g7[i, 1] - g7[i, 4])
                if iw > 0:
                    area1 = d7[j, 3] * d7[j, 4] * d7[j, 5]
                    area2 = g7[i, 3] * g7[i, 4] * g7[i, 5]
                    inc = iw * float(r)
                    r = inc / (area1 + area2 - inc)
                else:
                    r = 0.0
            o3[j, i] = r
    return o2, obev.astype(np.float64), o3.astype(np.float64)


# ------------------------------------------------------------------------------------------------------------------ statistics
def clean_data(gt, dt, cls, difficulty):
    """eval.py:30-82 -> (num_valid_gt, ignored_gt int array, ignored_dt int array, dc_bboxes (n, 4))."""
    name = CLASS_NAMES[cls]
    ign_gt, dc = [], []
    num_valid = 0
    for i, gname in enumerate(gt["name"]):
        low = gname.lower()
        valid = 1 if low == name else (0 if (name == "pedestrian" and low == "person_sitting") or (name == "car" and low == "van") else -1)
        height = gt["bbox"][i][3] - gt["bbox"][i][1]
        ignore = (gt["occluded"][i] > MAX_OCCLUSION[difficulty] or gt["truncated"][i] > MAX_TRUNCATION[difficulty]
                  or height <= MIN_HEIGHT[difficulty])
        if valid == 1 and not ignore:
            ign_gt.append(0)
            num_valid += 1
        elif valid == 0 or (ignore and valid == 1):
            ign_gt.append(1)
        else:
            ign_gt.append(-1)
        if gname == "DontCare":
            dc.append(gt["bbox"][i])
    ign_dt = []
    for i, dname in enumerate(dt["name"]):
        height = abs(dt["bbox"][i][3] - dt["bbox"][i][1])
        ign_dt.append(1 if height < MIN_HEIGHT[difficulty] else (0 if dname.lower() == name else -1))
    return (num_valid, np.array(ign_gt, np.int64), np.array(ign_dt, np.int64),
            np.array(dc, np.float64).reshape(-1, 4))


def get_thresholds(scores, num_gt):
    """eval.py:9-27: score thresholds (descending) for 41 recall sample points."""
    scores = np.sort(np.asarray(scores, np.float64))[::-1]
    current, out = 0.0, []
    n = len(scores)
    for i, s in enumerate(scores):
        l_recall = (i + 1) / num_gt
        r_recall = (i + 2) / num_gt if i < n - 1 else l_recall
        if (r_recall - current) < (current - l_recall) and i < n - 1:
            continue
        out.append(s)
        current += 1 / (N_SAMPLE_PTS - 1.0)
    return out


def tp_scores(ov, ign_gt, ign_dt, scores, min_overlap):
    """eval.py:233-317 with compute_fp=False: the scores of the TP matches, in gt order."""
    free = ign_dt != -1
    out = []
    for i, g in enumerate(ign_gt):
        if g == -1:
            continue
        cand = free & (ov[:, i] > min_overlap) & (scores > NO_DETECTION)
        if not cand.any():
            continue
        s = np.where(cand, scores, -np.inf)
        j = int(np.argmax(s))                                   # first index of the highest score
        free[j] = False
        if g == 1 or ign_dt[j] == 1:
            continue
        out.append(scores[j])
    return out


def statistics(ov, ign_gt, ign_dt, dt_bbox, dc, scores, gt_alpha, dt_alpha, metric, min_overlap, thresholds, compute_aos):
    """eval.py:233-350 with compute_fp=True for every threshold at once: (tp, fp, fn, similarity) arrays of len(thresholds);
    similarity is the per-image value fused_compute_statistics adds (0 where the reference skips it)."""
    T, nd = len(thresholds), len(ign_dt)
    thr = np.asarray(thresholds, np.float64)[:, None]
    free = (ign_dt != -1)[None, :] & ~(scores[None, :] < thr)               # (T, nd): not ignored, above the threshold
    ign1 = (ign_dt == 1)[None, :]
    tp, fn = np.zeros(T, np.int64), np.zeros(T, np.int64)
    sim = np.zeros(T, np.float64)
    for i, g in enumerate(ign_gt):
        if g == -1:
            continue
        if nd == 0:
            fn += g == 0
            continue
        above = free & (ov[:, i] > min_overlap)[None, :]
        valid = above & ~ign1
        has_valid = valid.any(1)
        best = np.argmax(np.where(valid, ov[:, i][None, :], -np.inf), 1)   # first index of the largest overlap
        first_ign = np.argmax(above & ign1, 1)
        has_ign = (above & ign1).any(1)
        det = np.where(has_valid, best, np.where(has_ign, first_ign, -1))
        found = det >= 0
        fn += (~found) & (g == 0)
        rows = np.nonzero(found)[0]
        free[rows, det[rows]] = False
        is_tp = found & has_valid & (g == 0)
        tp += is_tp
        if compute_aos:
            for t in np.nonzero(is_tp)[0]:
                sim[t] = sim[t] + (1.0 + math.cos(gt_alpha[i] - dt_alpha[det[t]])) / 2.0
    open_ = free & ~ign1
    fp = open_.sum(1)
    if metric == 0 and len(dc) and nd:
        hit = (image_box_overlap(dt_bbox, dc, 0) > min_overlap).any(1)
        fp = fp - (open_ & hit[None, :]).sum(1)
    return tp, fp, fn, sim


def eval_table(gt_annos, dt_annos, classes, min_overlaps, compute_aos):
    """The device's result table (include/monodetr_b200.h mdb_kitti_eval): (18 * n_cls, 1 + 4 * 41), row cfg =
    ((metric * n_cls + m) * 3 + difficulty) * 2 + k = [T, (tp, fp, fn, similarity) per threshold]."""
    n_cls = len(classes)
    ovs = [image_overlaps(g, d) for g, d in zip(gt_annos, dt_annos)]
    table = np.zeros((3, n_cls, 3, 2, 1 + 4 * N_SAMPLE_PTS))
    for m, cls in enumerate(classes):
        for l in range(3):
            cleaned = [clean_data(g, d, cls, l) for g, d in zip(gt_annos, dt_annos)]
            num_valid = sum(c[0] for c in cleaned)
            for metric in range(3):
                for k in range(2):
                    mo = min_overlaps[k, metric, m]
                    scores = []
                    for b, (g, d) in enumerate(zip(gt_annos, dt_annos)):
                        scores += tp_scores(ovs[b][metric], cleaned[b][1], cleaned[b][2], np.asarray(d["score"], np.float64), mo)
                    thresholds = get_thresholds(scores, num_valid) if scores else []
                    row = table[metric, m, l, k]
                    row[0] = len(thresholds)
                    pr = np.zeros((len(thresholds), 4))
                    for b, (g, d) in enumerate(zip(gt_annos, dt_annos)):
                        if not len(thresholds):
                            break
                        tp, fp, fn, sim = statistics(
                            ovs[b][metric], cleaned[b][1], cleaned[b][2], np.asarray(d["bbox"], np.float64).reshape(-1, 4),
                            cleaned[b][3], np.asarray(d["score"], np.float64), np.asarray(g["alpha"], np.float64),
                            np.asarray(d["alpha"], np.float64), metric, mo, thresholds, compute_aos and metric == 0)
                        pr[:, 0] += tp
                        pr[:, 1] += fp
                        pr[:, 2] += fn
                        pr[:, 3] += sim
                    row[1:1 + 4 * len(thresholds)] = pr.reshape(-1)
    return table.reshape(18 * n_cls, -1)


def do_eval(gt_annos, dt_annos, classes, min_overlaps, compute_aos):
    """eval.py:524-696 from the table: the 8 AP arrays (n_cls, 3, 2), scalar loops in the reference's order."""
    n_cls = len(classes)
    t = eval_table(gt_annos, dt_annos, classes, min_overlaps, compute_aos).reshape(3, n_cls, 3, 2, -1)
    curves = []
    for metric in range(3):
        precision = np.zeros((n_cls, 3, 2, N_SAMPLE_PTS))
        aos = np.zeros((n_cls, 3, 2, N_SAMPLE_PTS))
        for idx in np.ndindex(n_cls, 3, 2):
            row = t[(metric,) + idx]
            T = int(row[0])
            pr = row[1:].reshape(N_SAMPLE_PTS, 4)
            with np.errstate(divide="ignore", invalid="ignore"):
                for i in range(T):
                    precision[idx + (i,)] = pr[i, 0] / (pr[i, 0] + pr[i, 1])
                    if compute_aos and metric == 0:
                        aos[idx + (i,)] = pr[i, 3] / (pr[i, 0] + pr[i, 1])
            for i in range(T):
                precision[idx + (i,)] = np.max(precision[idx][i:])
                aos[idx + (i,)] = np.max(aos[idx][i:])
        curves.append((precision, aos))

    def m11(p):
        s = 0
        for i in range(0, N_SAMPLE_PTS, 4):
            s = s + p[..., i]
        return s / 11 * 100

    def m40(p):
        s = 0
        for i in range(1, N_SAMPLE_PTS):
            s = s + p[..., i]
        return s / 40 * 100
    (pb, ab), (pv, _), (p3, _) = curves
    aos11 = m11(ab) if compute_aos else None
    aos40 = m40(ab) if compute_aos else None
    return m11(pb), m11(pv), m11(p3), aos11, m40(pb), m40(pv), m40(p3), aos40


def fixture_annos(store, prefix):
    """Annotations stored flattened in tests/golden/kitti_eval.npz (tools/gen_golden_kitti_eval.py) -> list of per-image dicts
    shaped as get_label_anno returns them."""
    counts = np.asarray(store[prefix + "count"])
    off = np.concatenate([[0], np.cumsum(counts)])
    annos = []
    for b in range(len(counts)):
        s = slice(off[b], off[b + 1])
        a = {key: np.asarray(store[prefix + key])[s] for key in
             ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")}
        a["bbox"] = a["bbox"].reshape(-1, 4)
        a["dimensions"] = a["dimensions"].reshape(-1, 3)
        a["location"] = a["location"].reshape(-1, 3)
        annos.append(a)
    return annos
