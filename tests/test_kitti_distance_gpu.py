"""GPU: the distance-binned KITTI evaluation (mdb_kitti_eval_distance via monodetr_b200/kitti_eval.py) against the reference's
golden vectors (tests/golden/kitti_distance.npz) and tests/oracle_kitti_distance.py, and DeviceEvaluator.distance_result on a
collected validation table against get_distance_eval_result on the result files written from it."""
import os

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib
from monodetr_b200 import kitti_eval as ke
from oracle import kitti_eval as ok
import oracle_kitti_distance as okd
from test_kitti_eval_gpu import check_ap, random_set
from test_validation_gpu import Log, fixture_evaluator

pytestmark = pytest.mark.gpu
CASES = ("a", "b", "c")
MO = ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_distance.npz")))


@pytest.fixture(scope="module")
def validation(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "validation.npz")))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


def check_table(got, ref):
    """T, tp, fp and fn bit for bit; the AOS similarity sums cos on the device and in libm (1e-12 relative)."""
    assert got.shape == ref.shape
    np.testing.assert_array_equal(got[:, 0], ref[:, 0])
    g, r = got[:, 1:].reshape(len(got), -1, 4), ref[:, 1:].reshape(len(ref), -1, 4)
    np.testing.assert_array_equal(g[..., :3], r[..., :3])
    np.testing.assert_allclose(g[..., 3], r[..., 3], rtol=1e-12, atol=0)


@pytest.mark.parametrize("case", CASES)
def test_counts_match_oracle(golden, case):
    gt, dt = annos(golden, case)
    aos = bool(golden[f"{case}__compute_aos"])
    got = ke.eval_counts(gt, dt, [0, 1, 2], MO, aos, by_distance=True)
    check_table(got, okd.eval_table_by_distance(gt, dt, [0, 1, 2], MO, aos))
    assert (got[:, 0] > 0).any()


@pytest.mark.parametrize("case", CASES)
def test_ap_and_strings_match_reference(golden, case):
    gt, dt = annos(golden, case)
    got = ke.do_eval(gt, dt, [0, 1, 2], MO, bool(golden[f"{case}__compute_aos"]), DIForDIS=False)
    check_ap(got, [golden[f"{case}__do_eval{i}"] if golden[f"{case}__do_eval{i}"].size else None for i in range(8)])
    for c in range(3):
        text, ret = ke.get_distance_eval_result(gt, dt, c)
        assert text == str(golden[f"{case}__result{c}"])
        assert list(ret) == golden[f"{case}__keys{c}"].tolist()
        vals, ref = np.array(list(ret.values())), golden[f"{case}__values{c}"]
        aos = np.array(["_aos_" in k for k in ret], bool)
        np.testing.assert_array_equal(vals[~aos], ref[~aos])
        np.testing.assert_allclose(vals[aos], ref[aos], rtol=0, atol=1e-10)


def test_random_set_matches_oracle():
    """Locations 5-60 m with two decimals: every bin is populated; images whose overlaps come within 1e-4 of a threshold and
    gt within 1e-9 (relative) of a bin edge are left out, as the fixture's generator does."""
    gt, dt = random_set(np.random.default_rng(11), 300)
    keep = []
    for b, (g, d) in enumerate(zip(gt, dt)):
        ovs = ok.image_overlaps(g, d)
        dis = np.linalg.norm(np.asarray(g["location"], np.float64).reshape(-1, 3), axis=1)
        if all(o.size == 0 or min(np.abs(o - t).min() for t in (0.25, 0.5, 0.7)) >= 1e-4 for o in ovs) and \
                all(np.all(np.abs(dis - e) > 1e-9 * e) for e in (30.0, 50.0, 70.0)):
            keep.append(b)
    gt, dt = [gt[b] for b in keep], [dt[b] for b in keep]
    assert len(gt) > 250
    check_table(ke.eval_counts(gt, dt, [0, 1, 2], MO, True, by_distance=True), okd.eval_table_by_distance(gt, dt, [0, 1, 2], MO, True))


def test_distance_result_of_a_collected_table_equals_the_file_path(validation, tmp_path):
    ev = fixture_evaluator(validation)
    log = Log()
    car0 = ev.result(log)
    text, ret = ev.distance_result()
    ev.write_results(str(tmp_path))
    dt = ke.get_label_annos(str(tmp_path))
    gt = ok.fixture_annos(validation, "gt_")
    ref_text, ref_ret = ke.get_distance_eval_result(gt, dt, validation["writelist"].tolist())
    assert text == ref_text
    assert list(ret) == list(ref_ret)
    assert np.array(list(ret.values())).tobytes() == np.array(list(ref_ret.values())).tobytes()
    assert any(v > 0 for v in ret.values())
    # the official result of the same pass is unchanged, before and after
    log2 = Log()
    assert ev.result(log2) == car0 == validation["car"]
    assert log.lines == log2.lines and log.lines[2:] == [str(validation[f"result{c}"]) for c in range(3)]
    # with a logger, each class's part is logged
    log3 = Log()
    assert ev.distance_result(log3) == (text, ret)
    assert "".join(log3.lines) == text and len(log3.lines) == len(ev.classes)


def test_repeated_and_reproducible_runs_are_bit_identical():
    gt, dt = random_set(np.random.default_rng(3769), 1000, max_gt=12, max_dt=50)
    was = _lib.deterministic()
    try:
        runs = []
        for det in (False, False, True, True):
            _lib.lib().mdb_set_deterministic(int(det))
            runs.append(ke.eval_counts(gt, dt, [0, 1, 2], MO, True, by_distance=True))
    finally:
        _lib.lib().mdb_set_deterministic(int(was))
    for r in runs[1:]:
        assert r.tobytes() == runs[0].tobytes()
    assert runs[0][:, 0].max() > 10
    assert runs[0].tobytes() != ke.eval_counts(gt, dt, [0, 1, 2], MO, True).tobytes()     # the bins are not the difficulties


def test_distance_entry_point_checks_its_arguments():
    i32, i64 = torch.zeros(4, dtype=torch.int32, device="cuda"), torch.zeros(4, dtype=torch.int64, device="cuda")
    f64, res = torch.zeros(4, dtype=torch.float64, device="cuda"), torch.zeros(18, 1 + 4 * 41, dtype=torch.float64, device="cuda")
    for n_img, n_cls, ws_bytes in ((0, 1, 4096), (1, 7, 4096), (1, 1, 0)):          # no image, too many classes, no workspace
        with pytest.raises(RuntimeError, match="mdb_kitti_eval_distance"):
            _lib.call("mdb_kitti_eval_distance", i32, i32, i64, n_img, 0, 0, 0, 0, 0, f64, i32, f64, i32, f64, i32, f64, n_cls, 0,
                      res if ws_bytes else None, ws_bytes, res, launches=5)
