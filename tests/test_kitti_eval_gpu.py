"""GPU: the device KITTI evaluation (csrc/kitti_eval.cu via monodetr_b200/kitti_eval.py) against the reference's golden vectors
and against oracle/kitti_eval.py."""
import os

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib
from monodetr_b200 import kitti_eval as ke
from oracle import kitti_eval as ok

pytestmark = pytest.mark.gpu
CASES = ("a", "b", "c", "d")
MO = ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_eval.npz")))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


def check_ap(got, ref):
    for i, (g, r) in enumerate(zip(got, ref)):
        if r is None:
            assert g is None
        elif i in (3, 7):                                       # AOS: device cos against libm
            np.testing.assert_allclose(g, r, rtol=0, atol=1e-10)
        else:
            np.testing.assert_array_equal(g, r)


def random_set(rng, n_img, max_gt=8, max_dt=12):
    names = np.array(["Car", "Car", "Pedestrian", "Cyclist", "Van", "Person_sitting", "Truck", "DontCare", "Misc"])
    gts, dts = [], []
    for _ in range(n_img):
        out = []
        for n, det in ((rng.integers(0, max_gt + 1), False), (rng.integers(0, max_dt + 1), True)):
            x0, y0 = rng.uniform(0, 1100, n), rng.uniform(100, 250, n)
            h = np.where(rng.random(n) < 0.3, rng.choice([24.5, 25.0, 25.5, 39.5, 40.0, 40.5], n), rng.uniform(15, 200, n))
            a = {"name": rng.choice(names[:4] if det else names, n), "truncated": np.round(rng.uniform(0, 0.6, n), 2),
                 "occluded": rng.integers(0, 4, n), "alpha": np.round(rng.uniform(-np.pi, np.pi, n), 2),
                 "bbox": np.round(np.stack([x0, y0, x0 + rng.uniform(10, 300, n), y0 + h], 1), 2),
                 "dimensions": np.round(np.stack([rng.uniform(3, 5, n), rng.uniform(1.2, 2, n), rng.uniform(1.4, 2, n)], 1), 2),
                 "location": np.round(np.stack([rng.uniform(-15, 15, n), rng.uniform(1, 2, n), rng.uniform(5, 60, n)], 1), 2),
                 "rotation_y": np.round(rng.uniform(-np.pi, np.pi, n), 2), "score": np.round(rng.uniform(0, 1, n), 2)}
            out.append(a)
        if len(out[0]["name"]) and len(out[1]["name"]):         # detections near a gt, so that there are matches
            k = min(len(out[0]["name"]), len(out[1]["name"]))
            for key in ("bbox", "dimensions", "location"):
                out[1][key][:k] = np.round(out[0][key][:k] + rng.normal(0, 0.1, out[0][key][:k].shape), 2)
            out[1]["rotation_y"][:k] = out[0]["rotation_y"][:k]
        gts.append(out[0])
        dts.append(out[1])
    return gts, dts


@pytest.mark.parametrize("case", CASES)
def test_overlaps_match_reference(golden, case):
    gt, dt = annos(golden, case)
    blocks = ke.image_overlaps(gt, dt)
    for m in range(3):
        got = np.concatenate([b.reshape(-1) for b in blocks[m]])
        ref = golden[f"{case}__ov{m}"]
        assert got.shape == ref.shape
        np.testing.assert_array_equal(got, ref)                 # BEV / 3d: the reference's fp32 arithmetic, bit for bit


@pytest.mark.parametrize("case", CASES)
def test_ap_and_strings_match_reference(golden, case):
    gt, dt = annos(golden, case)
    got = ke.do_eval(gt, dt, [0, 1, 2], MO, bool(golden[f"{case}__compute_aos"]))
    check_ap(got, [golden[f"{case}__do_eval{i}"] if golden[f"{case}__do_eval{i}"].size else None for i in range(8)])
    for c in range(3):
        text, ret, first = ke.get_official_eval_result(gt, dt, c)
        assert text == str(golden[f"{case}__result{c}"])
        assert list(ret) == golden[f"{case}__keys{c}"].tolist()


def test_evaluate_folder(golden, tmp_path):
    ids = golden["d__ids"].tolist()
    for sub, lines in (("label", golden["d__gt_lines"]), ("res", golden["d__dt_lines"])):
        os.makedirs(tmp_path / sub)
        for i, text in zip(ids, lines):
            (tmp_path / sub / ("%06d.txt" % i)).write_text(str(text) + ("\n" if str(text) else ""))
    logged = []

    class Log:
        def info(self, s):
            logged.append(s)
    car = ke.evaluate(str(tmp_path / "res"), str(tmp_path / "label"), ids, logger=Log())
    assert car == golden["d__first0"]
    assert logged[2:] == [str(golden[f"d__result{c}"]) for c in range(3)]


def test_random_set_matches_oracle():
    rng = np.random.default_rng(7)
    gt, dt = random_set(rng, 300)
    keep = []                           # images whose overlaps keep a 1e-4 margin from every threshold (fp32 BEV)
    for b, (g, d) in enumerate(zip(gt, dt)):
        ovs = ok.image_overlaps(g, d)
        if all(o.size == 0 or min(np.abs(o - t).min() for t in (0.25, 0.5, 0.7)) >= 1e-4 for o in ovs):
            keep.append(b)
    gt, dt = [gt[b] for b in keep], [dt[b] for b in keep]
    assert len(gt) > 250
    blocks = ke.image_overlaps(gt, dt)
    for b, (g, d) in enumerate(zip(gt, dt)):
        ref = ok.image_overlaps(g, d)
        for m in range(3):
            np.testing.assert_array_equal(blocks[m][b], ref[m])
    check_ap(ke.do_eval(gt, dt, [0, 1, 2], MO, True), ok.do_eval(gt, dt, [0, 1, 2], MO, True))


def test_kitti_val_sized_set_is_reproducible():
    rng = np.random.default_rng(3769)
    gt, dt = random_set(rng, 3769, max_gt=12, max_dt=50)
    was = _lib.deterministic()
    try:
        runs = []
        for det in (False, False, True, True):
            _lib.lib().mdb_set_deterministic(int(det))
            runs.append(ke.eval_counts(gt, dt, [0, 1, 2], MO, True))
    finally:
        _lib.lib().mdb_set_deterministic(int(was))
    for r in runs[1:]:
        assert r.tobytes() == runs[0].tobytes()
    assert runs[0][:, 0].max() > 10                             # the set produces real threshold curves


def _boxes(n):
    return {"name": np.array(["Car"] * n), "truncated": np.zeros(n), "occluded": np.zeros(n, np.int64), "alpha": np.zeros(n),
            "bbox": np.tile([0.0, 0.0, 10.0, 50.0], (n, 1)), "dimensions": np.tile([4.0, 1.5, 1.6], (n, 1)),
            "location": np.tile([1.0, 1.5, 20.0], (n, 1)), "rotation_y": np.zeros(n), "score": np.full(n, 0.5)}


def test_limits_raise_naming_the_entry_point():
    with pytest.raises(RuntimeError, match="mdb_kitti_overlaps"):
        ke.do_eval([_boxes(1)], [_boxes(ke.MAX_BOXES + 1)], [0], MO[:, :, :1], True)
    classes = [0, 1, 2, 3, 4, 5, 0]                             # more than 6 classes in one call
    with pytest.raises(RuntimeError, match="mdb_kitti_eval"):
        ke.eval_counts([_boxes(1)], [_boxes(1)], classes, ke.OFFICIAL_MIN_OVERLAPS[:, :, classes], True)
