"""numpy restatement of the validation pass's file round trip: decoded rows -> result-file lines (tester_helper.py:112-132)
-> parsed annotations (kitti_common.py:294-347) -> the device table of monodetr_b200.kitti_eval.DeviceEvaluator.

    rows_to_text(rows, n, class_names)   the text of one result file, as Tester.save_results writes it
    text_to_anno(text)                   the annotation dict kitti_common.get_label_anno returns for that text
    rows_to_table(rows, n, codes)        (dt_f (n, 13), dt_cls (n,)) by the closed form rint(x * 100) / 100 of the kernel
"""
import numpy as np

CLASS_CODES = {"car": 0, "pedestrian": 1, "cyclist": 2, "van": 3, "person_sitting": 4, "truck": 5}
DT_FROM_ROW = [2, 3, 4, 5, 1, 13, 9, 10, 11, 8, 6, 7, 12]      # dt_f column <- decoded row column


def rows_to_text(rows, n, class_names):
    out = []
    for r in np.asarray(rows, np.float32)[:n]:
        out.append("{} 0.0 0".format(class_names[int(r[0])]) + "".join(" {:.2f}".format(v) for v in r[1:].tolist()) + "\n")
    return "".join(out)


def text_to_anno(text):
    rows = [line.strip().split(" ") for line in text.splitlines(True)]
    f = np.array([[float(v) for v in r[1:]] for r in rows], np.float64).reshape(len(rows), -1 if rows else 15)
    n = len(rows)
    anno = {"name": np.array([r[0] for r in rows]), "truncated": f[:, 0] if n else np.zeros(0),
            "occluded": np.array([int(r[2]) for r in rows]), "alpha": f[:, 2] if n else np.zeros(0),
            "bbox": f[:, 3:7].reshape(-1, 4) if n else np.zeros((0, 4)),
            "dimensions": f[:, 7:10][:, [2, 0, 1]].reshape(-1, 3) if n else np.zeros((0, 3)),
            "location": f[:, 10:13].reshape(-1, 3) if n else np.zeros((0, 3)),
            "rotation_y": f[:, 13] if n else np.zeros(0)}
    anno["score"] = f[:, 14] if n and f.shape[1] == 15 else np.zeros(n)
    return anno


def text_round(x):
    """float('{:.2f}'.format(x)) of float32 values, in closed form."""
    return np.rint(np.asarray(x, np.float32).astype(np.float64) * 100.0) / 100.0


def rows_to_table(rows, n, codes):
    """codes: decode class id -> eval class code (the tester's names through CLASS_CODES)."""
    r = np.asarray(rows, np.float32)[:n]
    return text_round(r[:, DT_FROM_ROW]), np.array([codes[int(c)] for c in r[:, 0]], np.int32)
