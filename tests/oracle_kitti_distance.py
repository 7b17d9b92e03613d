"""CPU restatement of the reference's distance-binned KITTI cleaning (lib/datasets/kitti/kitti_eval_python/eval.py:85-159,
clean_data_by_distance with DISTANCE_COVER = False), beside oracle/kitti_eval.py's clean_data, and the counts table of
mdb_kitti_eval_distance built from it with that module's overlaps, thresholds and statistics.  Pinned against
tests/golden/kitti_distance.npz by tests/test_kitti_distance_host_logic.py."""
import numpy as np

from oracle import kitti_eval as ok

MAX_DISTANCE = (30, 50, 70)                                                        # eval.py:90


def clean_data_by_distance(gt, dt, cls, bin_):
    """eval.py:85-159 -> (num_valid_gt, ignored_gt, ignored_dt, dc_bboxes) for distance bin 0 (<= 30 m), 1 (30-50 m) or
    2 (50-70 m).  Every bin uses the hard level's limits; the distance is np.linalg.norm of the location, as in the reference."""
    name = ok.CLASS_NAMES[cls]
    ign_gt, dc = [], []
    num_valid = 0
    for i, gname in enumerate(gt["name"]):
        low = gname.lower()
        valid = 1 if low == name else (0 if (name == "pedestrian" and low == "person_sitting") or (name == "car" and low == "van") else -1)
        height = gt["bbox"][i][3] - gt["bbox"][i][1]
        dis = np.linalg.norm(gt["location"][i])
        ignore = (gt["occluded"][i] > ok.MAX_OCCLUSION[2] or gt["truncated"][i] > ok.MAX_TRUNCATION[2]
                  or height <= ok.MIN_HEIGHT[2] or dis > MAX_DISTANCE[bin_] or (bin_ > 0 and dis <= MAX_DISTANCE[bin_ - 1]))
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
        ign_dt.append(1 if height < ok.MIN_HEIGHT[2] else (0 if dname.lower() == name else -1))
    return (num_valid, np.array(ign_gt, np.int64), np.array(ign_dt, np.int64),
            np.array(dc, np.float64).reshape(-1, 4))


def eval_table_by_distance(gt_annos, dt_annos, classes, min_overlaps, compute_aos):
    """oracle.kitti_eval.eval_table with clean_data_by_distance: (18 * n_cls, 1 + 4 * 41), row cfg =
    ((metric * n_cls + m) * 3 + bin) * 2 + k = [T, (tp, fp, fn, similarity) per threshold]."""
    n_cls = len(classes)
    ovs = [ok.image_overlaps(g, d) for g, d in zip(gt_annos, dt_annos)]
    table = np.zeros((3, n_cls, 3, 2, 1 + 4 * ok.N_SAMPLE_PTS))
    for m, cls in enumerate(classes):
        for l in range(3):
            cleaned = [clean_data_by_distance(g, d, cls, l) for g, d in zip(gt_annos, dt_annos)]
            num_valid = sum(c[0] for c in cleaned)
            for metric in range(3):
                for k in range(2):
                    mo = min_overlaps[k, metric, m]
                    scores = []
                    for b, d in enumerate(dt_annos):
                        scores += ok.tp_scores(ovs[b][metric], cleaned[b][1], cleaned[b][2], np.asarray(d["score"], np.float64), mo)
                    thresholds = ok.get_thresholds(scores, num_valid) if scores else []
                    row = table[metric, m, l, k]
                    row[0] = len(thresholds)
                    if not len(thresholds):
                        continue
                    pr = np.zeros((len(thresholds), 4))
                    for b, (g, d) in enumerate(zip(gt_annos, dt_annos)):
                        tp, fp, fn, sim = ok.statistics(
                            ovs[b][metric], cleaned[b][1], cleaned[b][2], np.asarray(d["bbox"], np.float64).reshape(-1, 4),
                            cleaned[b][3], np.asarray(d["score"], np.float64), np.asarray(g["alpha"], np.float64),
                            np.asarray(d["alpha"], np.float64), metric, mo, thresholds, compute_aos and metric == 0)
                        pr[:, 0] += tp
                        pr[:, 1] += fp
                        pr[:, 2] += fn
                        pr[:, 3] += sim
                    row[1:1 + 4 * len(thresholds)] = pr.reshape(-1)
    return table.reshape(18 * n_cls, -1)
