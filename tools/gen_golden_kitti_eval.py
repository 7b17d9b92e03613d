"""Generate tests/golden/kitti_eval.npz from the UNMODIFIED reference KITTI evaluation (CPU only).

    NUMBA_ENABLE_CUDASIM=1 python tools/gen_golden_kitti_eval.py      (the variable is set here if absent)

Needs numba and the reference checkout (MONODETR_REFERENCE, default /root/reference).  The reference's
lib/datasets/kitti/kitti_eval_python/{eval.py, rotate_iou.py, kitti_common.py} are imported in place as a package of their own
(no reference file is edited or copied); its one GPU kernel, rotate_iou_kernel_eval, runs in numba's CUDA simulator, and an
in-memory stand-in for `skimage.io` (an unused import of kitti_common.py) lets the reference's own label parser run.

Cases (all drawn from a fixed seed):
  a  ~100 KITTI-like images: all six class names + DontCare + Misc, detections jittered from gt, tied scores (2 decimals),
     boxes at the MIN_HEIGHT / truncation / occlusion edges of each difficulty
  b  edge geometry: identical, contained and touching boxes, rotation_y in {0, +-pi/2, pi} (parallel edges)
  c  images without gt, images without detections, and alpha = -10 everywhere (no AOS)
  d  a folder of label files and result files written as the reference's tester writes them, parsed by get_label_annos
Stored per case: the annotations (flattened; oracle.kitti_eval.fixture_annos reads them back), the per-image overlap blocks of the 3 metrics,
the 8 do_eval arrays for classes (0, 1, 2) together and each class's get_official_eval_result output.  No overlap of any
metric lies within MARGIN of an overlap threshold (0.25 / 0.5 / 0.7): such an image is drawn again, so that exact AP equality
is a fair bar although the BEV overlap is fp32.
"""
import importlib
import math
import os
import sys
import tempfile
import types

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")

import numpy as np  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
REF = os.environ.get("MONODETR_REFERENCE", "/root/reference")
OUT = os.path.join(ROOT, "tests", "golden", "kitti_eval.npz")
MARGIN = 1e-4
THRESHOLDS = (0.25, 0.5, 0.7)
NAMES = ["Car", "Car", "Car", "Pedestrian", "Pedestrian", "Cyclist", "Van", "Person_sitting", "Truck", "DontCare", "Misc"]
WRITE_NAMES = ["Car", "Pedestrian", "Cyclist"]


def reference():
    """The reference's kitti_eval_python package, imported in place under its own name."""
    if "skimage" not in sys.modules:
        sk = types.ModuleType("skimage")
        sk.io = types.ModuleType("skimage.io")
        sys.modules["skimage"], sys.modules["skimage.io"] = sk, sk.io
    pkg_dir = os.path.join(REF, "lib", "datasets", "kitti", "kitti_eval_python")
    pkg = types.ModuleType("kitti_eval_python")
    pkg.__path__ = [pkg_dir]
    sys.modules["kitti_eval_python"] = pkg
    ev = importlib.import_module("kitti_eval_python.eval")
    kc = importlib.import_module("kitti_eval_python.kitti_common")
    return ev, kc


def r2(x):
    return float(np.round(x, 2))


def draw_object(rng, name=None):
    name = name or NAMES[rng.integers(len(NAMES))]
    h = float(rng.choice([24.5, 25.0, 25.5, 39.5, 40.0, 40.5])) if rng.random() < 0.3 else r2(rng.uniform(15, 200))
    w = r2(rng.uniform(10, 300))
    x0, y0 = r2(rng.uniform(0, 1100)), r2(rng.uniform(100, 250))
    trunc = float(rng.choice([0.0, 0.15, 0.16, 0.3, 0.31, 0.5, 0.51])) if rng.random() < 0.5 else r2(rng.uniform(0, 0.6))
    return dict(name=name, truncated=trunc, occluded=int(rng.integers(0, 4)), alpha=r2(rng.uniform(-math.pi, math.pi)),
                bbox=[x0, y0, r2(x0 + w), r2(y0 + h)], hwl=[r2(rng.uniform(1.2, 2.0)), r2(rng.uniform(1.4, 2.0)), r2(rng.uniform(3, 5))],
                loc=[r2(rng.uniform(-15, 15)), r2(rng.uniform(1, 2)), r2(rng.uniform(5, 60))], ry=r2(rng.uniform(-math.pi, math.pi)))


def jitter(rng, o):
    d = dict(o)
    w, h = o["bbox"][2] - o["bbox"][0], o["bbox"][3] - o["bbox"][1]
    d["bbox"] = [r2(o["bbox"][0] + rng.normal(0, 0.08 * w)), r2(o["bbox"][1] + rng.normal(0, 0.08 * h)),
                 r2(o["bbox"][2] + rng.normal(0, 0.08 * w)), r2(o["bbox"][3] + rng.normal(0, 0.08 * h))]
    d["hwl"] = [r2(v + rng.normal(0, 0.1)) for v in o["hwl"]]
    d["loc"] = [r2(v + rng.normal(0, 0.4)) for v in o["loc"]]
    d["ry"] = r2(o["ry"] + rng.normal(0, 0.2))
    d["alpha"] = r2(o["alpha"] + rng.normal(0, 0.2))
    if rng.random() < 0.1:
        d["name"] = WRITE_NAMES[rng.integers(3)]
    d["score"] = r2(rng.uniform(0, 1))
    return d


def gt_line(o):
    v = [o["truncated"], o["occluded"], o["alpha"], *o["bbox"], *o["hwl"], *o["loc"], o["ry"]]
    return "{} {:.2f} {:d} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f}".format(o["name"], *v)


def dt_line(o):
    """As the reference's tester writes a detection (lib/helpers/tester_helper.py:125-132)."""
    vals = [o["alpha"], *o["bbox"], *o["hwl"], *o["loc"], o["ry"], o["score"]]
    return "{} 0.0 0".format(o["name"]) + "".join(" {:.2f}".format(v) for v in vals)


def parse(kc, lines):
    with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
        f.write("".join(l + "\n" for l in lines))
    try:
        return kc.get_label_anno(f.name)
    finally:
        os.unlink(f.name)


def safe(gt, dt):
    from oracle.kitti_eval import image_overlaps
    for o in image_overlaps(gt, dt):
        if o.size and min(np.abs(o - t).min() for t in THRESHOLDS) < MARGIN:
            return False
    return True


def draw_image(rng, kc, n_gt_max=9, p_det=0.8, n_fp_max=3, alpha_none=False):
    while True:
        objs = [draw_object(rng) for _ in range(rng.integers(0, n_gt_max + 1))]
        dets = [jitter(rng, o) for o in objs if o["name"] not in ("DontCare", "Misc") and rng.random() < p_det]
        dets += [dict(draw_object(rng, WRITE_NAMES[rng.integers(3)]), score=r2(rng.uniform(0, 1)))
                 for _ in range(rng.integers(0, n_fp_max + 1))]
        if alpha_none:
            for d in dets:
                d["alpha"] = -10.0
        gl, dl = [gt_line(o) for o in objs], [dt_line(d) for d in dets]
        gt, dt = parse(kc, gl), parse(kc, dl)
        if safe(gt, dt):
            return gt, dt, gl, dl


def geometry_images(kc):
    """Case b: crafted pairs on parallel / identical / touching edges, at the four axis-aligned headings."""
    images = []
    for k, ry in enumerate([0.0, math.pi / 2, -math.pi / 2, math.pi]):
        base = dict(name="Car", truncated=0.0, occluded=0, alpha=0.5, bbox=[100.0, 100.0, 300.0, 200.0], hwl=[1.5, 1.6, 4.0],
                    loc=[2.0, 1.5, 20.0 + k], ry=ry)
        same = dict(base, score=0.9)
        inside = dict(base, bbox=[150.0, 120.0, 250.0, 180.0], hwl=[1.5, 1.2, 3.0], score=0.8)
        touch = dict(base, bbox=[300.0, 100.0, 500.0, 200.0], loc=[2.0 + (4.0 if k % 2 == 0 else 1.6), 1.5, 20.0 + k], score=0.7)
        shifted = dict(base, bbox=[120.0, 100.0, 320.0, 200.0], loc=[2.3, 1.5, 20.0 + k], score=0.9)
        ped = dict(base, name="Pedestrian", bbox=[600.0, 150.0, 640.0, 240.0], hwl=[1.7, 0.6, 0.8], loc=[-3.0, 1.6, 15.0], ry=ry)
        for gts, dts in (([base], [same]), ([base], [inside, same]), ([base], [touch, shifted]), ([base, ped], [dict(ped, score=0.6), same])):
            gl = [gt_line(o) for o in gts]
            dl = [dt_line(d) for d in dts]
            images.append((parse(kc, gl), parse(kc, dl), gl, dl))
    return images


def flatten(prefix, annos, store):
    counts = np.array([len(a["name"]) for a in annos], np.int64)
    store[prefix + "count"] = counts
    for key in ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score"):
        vals = [np.asarray(a[key]) for a in annos]
        if key == "name":
            store[prefix + key] = np.concatenate(vals).astype(str) if counts.sum() else np.zeros(0, dtype="<U1")
        else:
            store[prefix + key] = np.concatenate(vals, 0)


def run_case(ev, name, gt, dt, store):
    print(f"[gen_golden_kitti_eval] case {name}: {len(gt)} images, {sum(len(a['name']) for a in gt)} gt, "
          f"{sum(len(a['name']) for a in dt)} detections", flush=True)
    flatten(f"{name}__gt_", gt, store)
    flatten(f"{name}__dt_", dt, store)
    for m in range(3):
        blocks = ev.calculate_iou_partly(dt, gt, m, 50)[0]
        store[f"{name}__ov{m}"] = np.concatenate([b.reshape(-1) for b in blocks]) if blocks else np.zeros(0)
    compute_aos = False
    for a in dt:
        if a["alpha"].shape[0] != 0:
            compute_aos = bool(a["alpha"][0] != -10)
            break
    mo = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3),
                   np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]])])
    res = ev.do_eval(gt, dt, [0, 1, 2], mo[:, :, [0, 1, 2]], compute_aos)
    store[f"{name}__compute_aos"] = np.array(compute_aos)
    for i, r in enumerate(res):
        store[f"{name}__do_eval{i}"] = np.zeros(0) if r is None else r
    for c in range(3):
        pr = {}
        s, d, v = ev.get_official_eval_result(gt, dt, c, PR_detail_dict=pr)
        store[f"{name}__result{c}"] = np.array(s)
        store[f"{name}__keys{c}"] = np.array(list(d.keys()))
        store[f"{name}__values{c}"] = np.array(list(d.values()), np.float64)
        store[f"{name}__first{c}"] = np.array(v)
        for k, a in pr.items():
            store[f"{name}__pr{c}_{k}"] = a


def main():
    ev, kc = reference()
    rng = np.random.default_rng(20261015)
    store = {"margin": np.array(MARGIN)}

    a = [draw_image(rng, kc) for _ in range(100)]
    run_case(ev, "a", [x[0] for x in a], [x[1] for x in a], store)

    b = geometry_images(kc)
    for x in b:
        assert safe(x[0], x[1]), "case b must keep its overlaps away from the thresholds"
    run_case(ev, "b", [x[0] for x in b], [x[1] for x in b], store)

    c = [draw_image(rng, kc, alpha_none=True) for _ in range(12)]
    c += [draw_image(rng, kc, n_gt_max=0, alpha_none=True) for _ in range(3)]            # no gt
    c += [draw_image(rng, kc, p_det=0.0, n_fp_max=0, alpha_none=True) for _ in range(3)]  # no detections
    c.insert(0, c.pop())                                                                  # the first image has no detections
    run_case(ev, "c", [x[0] for x in c], [x[1] for x in c], store)

    d = [draw_image(rng, kc, n_gt_max=6) for _ in range(20)]
    ids = sorted(rng.choice(200, size=len(d), replace=False).tolist())
    with tempfile.TemporaryDirectory() as tmp:
        lab, res = os.path.join(tmp, "label_2"), os.path.join(tmp, "data")
        os.makedirs(lab)
        os.makedirs(res)
        for i, x in zip(ids, d):
            with open(os.path.join(lab, "%06d.txt" % i), "w") as f:
                f.write("".join(l + "\n" for l in x[2]))
            with open(os.path.join(res, "%06d.txt" % i), "w") as f:
                f.write("".join(l + "\n" for l in x[3]))
        gt = kc.get_label_annos(lab, ids)
        dt = kc.get_label_annos(res)
    store["d__ids"] = np.array(ids, np.int64)
    store["d__gt_lines"] = np.array(["\n".join(x[2]) for x in d])
    store["d__dt_lines"] = np.array(["\n".join(x[3]) for x in d])
    run_case(ev, "d", gt, dt, store)

    np.savez_compressed(OUT, **store)
    print(f"[gen_golden_kitti_eval] wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
