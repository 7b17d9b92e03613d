"""CPU: the distance-binned KITTI evaluation's host logic -- do_eval(..., DIForDIS=False), get_distance_eval_result, the
configuration order, ret_dict, PR_detail_dict and the result string -- driven through the stand-in of
test_kitti_eval_host_logic.py with mdb_kitti_eval_distance computed by tests/oracle_kitti_distance.py, and that oracle pinned to
the reference's golden vectors (tests/golden/kitti_distance.npz, tools/gen_golden_kitti_distance.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib
from monodetr_b200 import kitti_eval as ke
from oracle import kitti_eval as ok
import fake_device_lib
import oracle_kitti_distance as okd
from test_kitti_eval_host_logic import KittiFakeLib, _arr

CASES = ("a", "b", "c")


class KittiDistanceFakeLib(KittiFakeLib):
    """mdb_kitti_eval_distance computed by the distance oracle; mdb_kitti_eval as in the official stand-in."""

    def mdb_kitti_eval_distance(self, gt_off, dt_off, ov_off, n_img, n_gt, n_dt, max_gt, max_dt, n_ov, gt_f, gt_i, dt_f, dt_cls,
                                overlaps, classes, min_overlaps, n_cls, compute_aos, ws, ws_bytes, result, stream):
        self.distance_evals.append((n_img, n_gt, n_dt, max_gt, max_dt, n_ov))
        gt, dt = self._unpack(gt_off, dt_off, n_img, gt_f, gt_i, dt_f, dt_cls)
        cls = _arr(classes, ctypes.c_int32, n_cls).tolist()
        mo = _arr(min_overlaps, ctypes.c_double, 6 * n_cls).reshape(2, 3, n_cls)
        table = okd.eval_table_by_distance(gt, dt, cls, mo, bool(compute_aos))
        _arr(result, ctypes.c_double, table.size)[:] = table.reshape(-1)
        return 0


@pytest.fixture
def fake(monkeypatch):
    fake_device_lib.install(monkeypatch)
    lib = KittiDistanceFakeLib(1)
    lib.evals, lib.distance_evals = [], []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(ke, "_device", lambda: torch.device("cpu"))
    return lib


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_distance.npz")))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


def _check_do_eval(got, golden, case):
    for i, g in enumerate(got):
        ref = golden[f"{case}__do_eval{i}"]
        if g is None:
            assert ref.size == 0
        else:
            np.testing.assert_array_equal(g, ref)


@pytest.mark.parametrize("case", CASES)
def test_oracle_matches_reference(golden, case):
    """The distance oracle's table, turned into APs by the host arithmetic the official fixture pins, is the reference's."""
    gt, dt = annos(golden, case)
    aos = bool(golden[f"{case}__compute_aos"])
    table = okd.eval_table_by_distance(gt, dt, [0, 1, 2], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], aos)
    _check_do_eval(ke._aps(table, 3, aos), golden, case)


def test_oracle_bins_at_the_edges(golden):
    """Case b puts gt on 30 / 50 / 70 m and one ulp either side: each lands in the bin the reference's rule gives."""
    gt, dt = annos(golden, "b")
    seen = set()
    for g, d in zip(gt, dt):
        dis = float(np.linalg.norm(g["location"][0]))
        cls = ke.NAME_TO_CLASS[str(g["name"][0])]
        bins = [l for l in range(3) if okd.clean_data_by_distance(g, d, cls, l)[1][0] == 0]
        want = [] if dis > 70 else [0 if dis <= 30 else (1 if dis <= 50 else 2)]
        assert bins == want, (g["location"][0], bins, want)
        seen.add(dis)
    for e in (30.0, 50.0, 70.0):
        assert {e, float(np.nextafter(e, np.inf)), float(np.nextafter(e, -np.inf))} <= seen


@pytest.mark.parametrize("case", CASES)
def test_distance_result_matches_reference(fake, golden, case):
    gt, dt = annos(golden, case)
    for c in range(3):
        pr = {}
        text, ret = ke.get_distance_eval_result(gt, dt, c, PR_detail_dict=pr)
        assert text == str(golden[f"{case}__result{c}"])
        assert list(ret) == golden[f"{case}__keys{c}"].tolist()
        np.testing.assert_array_equal(np.array(list(ret.values())), golden[f"{case}__values{c}"])
        prefix = f"{case}__pr{c}_"
        assert set(pr) == {k[len(prefix):] for k in golden if k.startswith(prefix)}
        for k, v in pr.items():
            np.testing.assert_array_equal(v, golden[f"{case}__pr{c}_{k}"])
    assert len(fake.distance_evals) == 3 and not fake.evals


@pytest.mark.parametrize("case", CASES)
def test_do_eval_by_distance_all_classes_in_one_call(fake, golden, case):
    gt, dt = annos(golden, case)
    got = ke.do_eval(gt, dt, [0, 1, 2], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], bool(golden[f"{case}__compute_aos"]),
                     DIForDIS=False)
    _check_do_eval(got, golden, case)
    assert len(fake.distance_evals) == 1 and not fake.evals


def test_configuration_order(fake, golden):
    """cfg = ((metric * n_cls + m) * 3 + bin) * 2 + k: the table of classes [2, 0] is the rows of [0, 1, 2] rearranged."""
    gt, dt = annos(golden, "a")
    full = ke.eval_counts(gt, dt, [0, 1, 2], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], True, by_distance=True)
    part = ke.eval_counts(gt, dt, [2, 0], ke.OFFICIAL_MIN_OVERLAPS[:, :, [2, 0]], True, by_distance=True)
    full, part = full.reshape(3, 3, 3, 2, -1), part.reshape(3, 2, 3, 2, -1)
    np.testing.assert_array_equal(part, full[:, [2, 0]])
    assert (full[..., 0] > 0).any(axis=(0, 1, 3)).all()              # every bin has thresholds somewhere


def test_official_path_is_unchanged(fake, golden):
    """DIForDIS=True (the default) still goes to mdb_kitti_eval, and get_official_eval_result keeps its difficulty keys."""
    gt, dt = annos(golden, "a")
    ke.do_eval(gt, dt, [0], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0]], True)
    ke.do_eval(gt, dt, [0], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0]], True, DIForDIS=True)
    assert len(fake.evals) == 2 and not fake.distance_evals
    _, ret, _ = ke.get_official_eval_result(gt, dt, 0)
    assert "Car_3d_moderate_R40" in ret and not any(k.endswith(("30m", "50m", "70m", "m_R40")) for k in ret)
    assert len(fake.evals) == 3 and not fake.distance_evals


def test_current_classes_forms(fake, golden):
    gt, dt = annos(golden, "a")
    ref0, ref1 = str(golden["a__result0"]), str(golden["a__result1"])
    assert ke.get_distance_eval_result(gt, dt, 0)[0] == ref0
    assert ke.get_distance_eval_result(gt, dt, "Car")[0] == ref0
    assert ke.get_distance_eval_result(gt, dt, ["Car"])[0] == ref0
    text, ret = ke.get_distance_eval_result(gt, dt, ["Car", 1])
    assert text == ref0 + ref1
    assert list(ret) == golden["a__keys0"].tolist() + golden["a__keys1"].tolist()


def test_ret_dict_keys_and_aos_rule(fake, golden):
    gt, dt = annos(golden, "a")
    _, ret = ke.get_distance_eval_result(gt, dt, "Pedestrian")
    keys = [f"Pedestrian_aos_{b}" for b in ke.DISTANCE_KEYS] + [f"Pedestrian_aos_{b}_R40" for b in ke.DISTANCE_KEYS]
    for sfx in ("", "_R40"):
        keys += [f"Pedestrian_{m}_{b}{sfx}" for m in ("3d", "bev", "image") for b in ke.DISTANCE_KEYS]
    assert list(ret) == keys
    gt_c, dt_c = annos(golden, "c")
    text, ret = ke.get_distance_eval_result(gt_c, dt_c, 0)
    assert "aos" not in text and not any("aos" in k for k in ret)
