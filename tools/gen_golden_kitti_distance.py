"""Generate tests/golden/kitti_distance.npz from the UNMODIFIED reference KITTI evaluation's distance-binned path (CPU only).

    NUMBA_ENABLE_CUDASIM=1 python tools/gen_golden_kitti_distance.py      (the variable is set here if absent)

The reference is imported in place exactly as tools/gen_golden_kitti_eval.py does it (numba's CUDA simulator for the rotated
IoU, an in-memory stand-in for `skimage.io`), and its do_eval(..., DIForDIS=False) / get_distance_eval_result run
clean_data_by_distance (eval.py:85-159) with the module's DISTANCE_COVER = False.

Cases (all drawn from a fixed seed):
  a  ~100 KITTI-like images whose gt lie 0-90 m from the camera: all six class names + DontCare (some at KITTI's
     -1000, -1000, -1000) + Misc, heights at 25 +- 0.5, occlusion 0..3, truncation at 0.5 / 0.51, detections jittered from gt
  b  gt exactly on the bin edges: integer Pythagorean locations ((30, 0, 0), (18, 0, 24), (0, 0, 50), (0, 30, 40), (0, 0, 70),
     (42, 0, 40) = 58 m) and the fp64 neighbours one ulp away of the single-axis ones; every summation order and FMA
     contraction of x*x + y*y + z*z gives the same norm there, so the device's order is a fair comparison
  c  images without gt, images without detections, and alpha = -10 everywhere (no AOS)
Random distances keep a relative margin DIST_MARGIN from 30, 50 and 70 m, and no overlap of any metric lies within MARGIN of an
overlap threshold, so that exact AP equality is a fair bar.  Stored per case: the annotations (flattened as in kitti_eval.npz;
oracle.kitti_eval.fixture_annos reads them back), the 8 do_eval(..., DIForDIS=False) arrays for classes (0, 1, 2) together, and
each class's get_distance_eval_result output with its PR_detail_dict.
"""
import math
import os
import sys

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_golden_kitti_eval as gk  # noqa: E402

OUT = os.path.join(gk.ROOT, "tests", "golden", "kitti_distance.npz")
EDGES = (30.0, 50.0, 70.0)
DIST_MARGIN = 1e-9


def near_edge(loc):
    d = float(np.linalg.norm(np.asarray(loc, np.float64)))
    return any(abs(d - e) <= DIST_MARGIN * e for e in EDGES)


def draw_object(rng, name=None):
    """gen_golden_kitti_eval.draw_object with the location spread over 0-90 m (DontCare sometimes at -1000)."""
    o = gk.draw_object(rng, name)
    if o["name"] == "DontCare" and rng.random() < 0.5:
        o["loc"] = [-1000.0, -1000.0, -1000.0]
        return o
    while True:
        d, y, th = rng.uniform(0.5, 90.0), gk.r2(rng.uniform(1, 2)), rng.uniform(-0.6, 0.6)
        r = math.sqrt(max(d * d - y * y, 0.0))
        o["loc"] = [gk.r2(r * math.sin(th)), y, gk.r2(r * math.cos(th))]
        if not near_edge(o["loc"]):
            return o


def draw_image(rng, kc, n_gt_max=9, p_det=0.8, n_fp_max=3, alpha_none=False):
    while True:
        objs = [draw_object(rng) for _ in range(rng.integers(0, n_gt_max + 1))]
        dets = [gk.jitter(rng, o) for o in objs if o["name"] not in ("DontCare", "Misc") and rng.random() < p_det]
        dets += [dict(draw_object(rng, gk.WRITE_NAMES[rng.integers(3)]), score=gk.r2(rng.uniform(0, 1)))
                 for _ in range(rng.integers(0, n_fp_max + 1))]
        if alpha_none:
            for d in dets:
                d["alpha"] = -10.0
        gt, dt = gk.parse(kc, [gk.gt_line(o) for o in objs]), gk.parse(kc, [gk.dt_line(d) for d in dets])
        if gk.safe(gt, dt):
            return gt, dt


def anno(objs, det=False):
    """In-memory annotations (no text round trip, so that a location one ulp off an edge survives)."""
    n = len(objs)
    a = {"name": np.array([o["name"] for o in objs]), "truncated": np.array([o["truncated"] for o in objs], np.float64),
         "occluded": np.array([o["occluded"] for o in objs], np.int64), "alpha": np.array([o["alpha"] for o in objs], np.float64),
         "bbox": np.array([o["bbox"] for o in objs], np.float64).reshape(n, 4),
         "dimensions": np.array([o["hwl"] for o in objs], np.float64).reshape(n, 3)[:, [2, 0, 1]],
         "location": np.array([o["loc"] for o in objs], np.float64).reshape(n, 3),
         "rotation_y": np.array([o["ry"] for o in objs], np.float64)}
    a["score"] = np.array([o["score"] for o in objs], np.float64) if det else np.zeros(n)
    return a


def edge_images():
    """Case b: one image per edge location; the gt is found by an identical detection and missed by a shifted one."""
    up, down = (lambda v: float(np.nextafter(v, np.inf))), (lambda v: float(np.nextafter(v, -np.inf)))
    locs = [(30.0, 0.0, 0.0), (up(30.0), 0.0, 0.0), (down(30.0), 0.0, 0.0), (18.0, 0.0, 24.0),
            (0.0, 0.0, 50.0), (0.0, 0.0, up(50.0)), (0.0, 0.0, down(50.0)), (0.0, 30.0, 40.0),
            (0.0, 0.0, 70.0), (0.0, 0.0, up(70.0)), (0.0, 0.0, down(70.0)), (42.0, 0.0, 40.0)]
    images = []
    for k, loc in enumerate(locs):
        for c, (name, hwl) in enumerate((("Car", [1.5, 1.6, 4.0]), ("Pedestrian", [1.7, 0.6, 0.8]), ("Cyclist", [1.7, 0.6, 1.8]))):
            o = dict(name=name, truncated=0.0, occluded=(k + c) % 3, alpha=0.3 * (c + 1), bbox=[100.0, 120.0, 260.0, 200.0 + 10 * c],
                     hwl=hwl, loc=list(loc), ry=0.25 * c)
            dets = [dict(o, score=0.9 - 0.05 * k)] if (k + c) % 4 != 3 else []
            dets.append(dict(o, name="Car", bbox=[600.0, 300.0, 700.0, 360.0], loc=[5.0, 1.5, 12.0], score=0.55 + 0.01 * c))
            gt, dt = anno([o]), anno(dets, det=True)
            assert gk.safe(gt, dt), "case b must keep its overlaps away from the thresholds"
            images.append((gt, dt))
    return images


def run_case(ev, name, gt, dt, store):
    print(f"[gen_golden_kitti_distance] case {name}: {len(gt)} images, {sum(len(a['name']) for a in gt)} gt, "
          f"{sum(len(a['name']) for a in dt)} detections", flush=True)
    gk.flatten(f"{name}__gt_", gt, store)
    gk.flatten(f"{name}__dt_", dt, store)
    compute_aos = False
    for a in dt:
        if a["alpha"].shape[0] != 0:
            compute_aos = bool(a["alpha"][0] != -10)
            break
    mo = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3),
                   np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]])])
    res = ev.do_eval(gt, dt, [0, 1, 2], mo[:, :, [0, 1, 2]], compute_aos, DIForDIS=False)
    store[f"{name}__compute_aos"] = np.array(compute_aos)
    for i, r in enumerate(res):
        store[f"{name}__do_eval{i}"] = np.zeros(0) if r is None else r
    for c in range(3):
        pr = {}
        s, d = ev.get_distance_eval_result(gt, dt, c, PR_detail_dict=pr)
        store[f"{name}__result{c}"] = np.array(s)
        store[f"{name}__keys{c}"] = np.array(list(d.keys()))
        store[f"{name}__values{c}"] = np.array(list(d.values()), np.float64)
        for k, a in pr.items():
            store[f"{name}__pr{c}_{k}"] = a


def main():
    ev, kc = gk.reference()
    assert ev.DISTANCE_COVER is False
    rng = np.random.default_rng(20261017)
    store = {"margin": np.array(gk.MARGIN), "dist_margin": np.array(DIST_MARGIN)}

    a = [draw_image(rng, kc) for _ in range(100)]
    run_case(ev, "a", [x[0] for x in a], [x[1] for x in a], store)

    b = edge_images()
    run_case(ev, "b", [x[0] for x in b], [x[1] for x in b], store)

    c = [draw_image(rng, kc, alpha_none=True) for _ in range(12)]
    c += [draw_image(rng, kc, n_gt_max=0, alpha_none=True) for _ in range(3)]            # no gt
    c += [draw_image(rng, kc, p_det=0.0, n_fp_max=0, alpha_none=True) for _ in range(3)]  # no detections
    c.insert(0, c.pop())                                                                  # the first image has no detections
    run_case(ev, "c", [x[0] for x in c], [x[1] for x in c], store)

    np.savez_compressed(OUT, **store)
    print(f"[gen_golden_kitti_distance] wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
