"""Generate tests/golden/validation.npz from the UNMODIFIED reference validation pass (CPU only).

    NUMBA_ENABLE_CUDASIM=1 python tools/gen_golden_validation.py      (the variable is set here if absent)

Needs numba and the reference checkout (MONODETR_REFERENCE, default /root/reference).  Decoded rows in this repository's
format (mdb_decode_dets_f32: float32 [cls, alpha, x0, y0, x1, y1, h, w, l, X, Y, Z, ry, score], `count` leading rows per image)
go through the reference's own steps, imported in place (no reference file is edited or copied):
  * lib/helpers/tester_helper.py Tester.save_results, called on a stand-in `self`, writes the result files;
  * kitti_eval_python.kitti_common.get_label_annos parses them and a KITTI-like label folder (every class name plus DontCare);
  * kitti_eval_python.eval.get_official_eval_result evaluates each class of the writelist (the rotated IoU in numba's CUDA
    simulator), as KITTI_Dataset.eval does (kitti_dataset.py:101-116).
The rows hold values that are exact ties of the 2-decimal formatting (multiples of 1/8) and their float32 neighbours, small
negatives that print as -0.00, values of magnitude >= 2^23, many tied 2-decimal scores, images without detections or with
none above the threshold, and all three classes.  No overlap lies within MARGIN of an overlap threshold (the image is drawn
again), so that exact AP equality is a fair bar.
Stored: rows, count, ids, the written file texts, the gt label texts, the parsed annotations (flattened as
oracle.kitti_eval.fixture_annos reads them), each class's result string / ret_dict / first value, and Car AP3d R40.
"""
import os
import sys
import tempfile
import types

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gen_golden_kitti_eval import REF, draw_object, flatten, gt_line, jitter, reference, safe  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "validation.npz")
MARGIN = 1e-4
TOPK = 16
N_IMG = 48
TESTER_NAMES = ["Pedestrian", "Car", "Cyclist"]
WRITELIST = ["Car", "Pedestrian", "Cyclist"]
TEST_ID = {"Car": 0, "Pedestrian": 1, "Cyclist": 2}        # kitti_dataset.py:107


def ref_tester():
    if REF not in sys.path:
        sys.path.insert(0, REF)
    from lib.helpers.tester_helper import Tester
    return Tester


def tie(rng, x):
    """A multiple of 1/8 near x (an exact tie of '{:.2f}' when it ends in .125 / .375 / .625 / .875), or a float32 neighbour."""
    t = np.float32(np.floor(x * 8) / 8 + 0.125 * rng.integers(0, 2))
    k = rng.integers(0, 3)
    return t if k == 0 else np.nextafter(t, np.float32(np.inf if k == 1 else -np.inf), dtype=np.float32)


def det_row(rng, o):
    """A decoded row (float32) from a jittered object dict of gen_golden_kitti_eval."""
    name = o["name"] if o["name"] in TESTER_NAMES else TESTER_NAMES[rng.integers(3)]
    h, w, l = o["hwl"]
    v = [TESTER_NAMES.index(name), o["alpha"], *o["bbox"], h, w, l, *o["loc"], o["ry"], o["score"]]
    v = [float(x) + (rng.uniform(-0.004, 0.004) if i > 0 else 0.0) for i, x in enumerate(v)]
    r = np.array(v, np.float32)
    for i in range(1, 14):
        if rng.random() < 0.3:
            r[i] = tie(rng, float(r[i]))
    if rng.random() < 0.15:
        r[1] = np.float32(rng.choice([-0.004, -0.0, -0.001, 0.004]))          # prints as -0.00 / 0.00
    if rng.random() < 0.5:
        r[13] = np.float32(rng.choice([0.25, 0.3, 0.35, 0.5, 0.55, 0.7]))       # tied scores
    return r


def far_row(rng):
    """A detection far from everything: |x| >= 2^23 in the location and the 2-d box."""
    big = np.float32(2 ** 23 + rng.integers(0, 2 ** 22))
    return np.array([1, 0.5, big, 1.0e7, big + 64, 1.0e7 + 48, 1.5, 1.6, 3.9, -big, 1.5, np.float32(3.0e7), 0.1, 0.45],
                    np.float32)


def close(rng, o):
    """A detection near its object: most of them match in 3-d at the 0.7 overlap."""
    d = dict(jitter(rng, o))
    d["bbox"] = [v + rng.normal(0, 1.5) for v in o["bbox"]]
    d["hwl"] = [v + rng.normal(0, 0.03) for v in o["hwl"]]
    d["loc"] = [v + rng.normal(0, 0.05) for v in o["loc"]]
    d["ry"] = o["ry"] + rng.normal(0, 0.03)
    return d


def draw_image(rng, kc, kind):
    while True:
        objs = [draw_object(rng) for _ in range(rng.integers(0, 8))]
        dets = [det_row(rng, close(rng, o) if rng.random() < 0.6 else jitter(rng, o))
                for o in objs if o["name"] not in ("DontCare", "Misc") and rng.random() < 0.8]
        dets += [det_row(rng, dict(draw_object(rng, TESTER_NAMES[rng.integers(3)]), score=float(rng.uniform(0, 1))))
                 for _ in range(rng.integers(0, 3))]
        if kind == "far":
            dets.append(far_row(rng))
        if kind in ("none", "below"):
            dets = []
        dets = sorted(dets, key=lambda r: -float(r[13]))[:TOPK]
        rows = np.zeros((TOPK, 14), np.float32)
        if dets:
            rows[:len(dets)] = np.stack(dets)
        gl = [gt_line(o) for o in objs]
        gt = kc_parse(kc, gl)
        dt = kc_parse(kc, [line for line in dt_lines(rows, len(dets)).split("\n") if line])
        if safe(gt, dt):
            return rows, len(dets), gl


def dt_lines(rows, n):
    """Only for the margin check; the stored texts come from the reference's save_results."""
    return "".join("{} 0.0 0".format(TESTER_NAMES[int(r[0])]) + "".join(" {:.2f}".format(v) for v in r[1:].tolist()) + "\n"
                   for r in rows[:n])


def kc_parse(kc, lines):
    with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
        f.write("".join(line + "\n" for line in lines))
    try:
        return kc.get_label_anno(f.name)
    finally:
        os.unlink(f.name)


def main():
    ev, kc = reference()
    Tester = ref_tester()
    rng = np.random.default_rng(20261016)
    kinds = ["plain"] * N_IMG
    kinds[3], kinds[10], kinds[17], kinds[30] = "none", "below", "far", "none"
    images = [draw_image(rng, kc, k) for k in kinds]
    rows = np.stack([x[0] for x in images])
    count = np.array([x[1] for x in images], np.int32)
    below = kinds.index("below")
    rows[below, :] = 0.0                                    # a decoded image whose candidates all missed the threshold
    ids = np.array(sorted(rng.choice(7481, size=N_IMG, replace=False).tolist()), np.int64)
    store = {"margin": np.array(MARGIN), "topk": np.array(TOPK), "rows": rows, "count": count, "ids": ids,
             "writelist": np.array(WRITELIST), "class_names": np.array(TESTER_NAMES)}
    results = {int(i): [[int(v[0])] + v[1:].tolist() for v in rows[b, :count[b]]] for b, i in enumerate(ids)}
    with tempfile.TemporaryDirectory() as tmp:
        stand_in = types.SimpleNamespace(output_dir=tmp, dataset_type="KITTI", class_name=TESTER_NAMES)
        Tester.save_results(stand_in, results)
        res = os.path.join(tmp, "outputs", "data")
        lab = os.path.join(tmp, "label_2")
        os.makedirs(lab)
        texts = []
        for b, i in enumerate(ids):
            with open(os.path.join(res, "%06d.txt" % i)) as f:
                texts.append(f.read())
            with open(os.path.join(lab, "%06d.txt" % i), "w") as f:
                f.write("".join(line + "\n" for line in images[b][2]))
        dt = kc.get_label_annos(res)
        gt = kc.get_label_annos(lab, [int(i) for i in ids])
    store["dt_text"] = np.array(texts)
    store["gt_text"] = np.array(["".join(line + "\n" for line in x[2]) for x in images])
    flatten("gt_", gt, store)
    flatten("dt_", dt, store)
    car = 0
    for c, category in enumerate(WRITELIST):
        s, d, v = ev.get_official_eval_result(gt, dt, TEST_ID[category])
        store[f"result{c}"] = np.array(s)
        store[f"keys{c}"] = np.array(list(d.keys()))
        store[f"values{c}"] = np.array(list(d.values()), np.float64)
        store[f"first{c}"] = np.array(v)
        if category == "Car":
            car = v
    store["car"] = np.array(car)
    print("[gen_golden_validation] first values per class:", [float(store[f"first{c}"]) for c in range(3)])
    print(f"[gen_golden_validation] {N_IMG} images, {int(count.sum())} detections, "
          f"{sum(len(a['name']) for a in gt)} labels, Car AP3d R40 moderate {float(car):.4f}", flush=True)
    np.savez_compressed(OUT, **store)
    print(f"[gen_golden_validation] wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
