"""CPU: oracle/kitti_eval.py against the golden vectors of the reference KITTI evaluation (tools/gen_golden_kitti_eval.py)."""
import os

import numpy as np
import pytest

from oracle import kitti_eval as ok

CASES = ("a", "b", "c", "d")
MIN_OVERLAPS = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3),
                         np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5],
                                   [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]])])[:, :, [0, 1, 2]]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_eval.npz")))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


@pytest.mark.parametrize("case", CASES)
def test_overlaps_match_reference(golden, case):
    gt, dt = annos(golden, case)
    blocks = [ok.image_overlaps(g, d) for g, d in zip(gt, dt)]
    for m in range(3):
        got = np.concatenate([b[m].reshape(-1) for b in blocks])
        ref = golden[f"{case}__ov{m}"]
        assert got.shape == ref.shape
        np.testing.assert_array_equal(got, ref)                     # the same fp64 / fp32 operations: bit-identical


@pytest.mark.parametrize("case", CASES)
def test_ap_arrays_match_reference(golden, case):
    gt, dt = annos(golden, case)
    got = ok.do_eval(gt, dt, [0, 1, 2], MIN_OVERLAPS, bool(golden[f"{case}__compute_aos"]))
    for i, g in enumerate(got):
        ref = golden[f"{case}__do_eval{i}"]
        if g is None:
            assert ref.size == 0
        else:
            np.testing.assert_array_equal(g, ref)


def test_fixture_keeps_overlaps_away_from_thresholds(golden):
    margin = float(golden["margin"])
    assert margin >= 1e-4
    for case in CASES:
        for m in range(3):
            ov = golden[f"{case}__ov{m}"]
            for t in (0.25, 0.5, 0.7):
                assert ov.size == 0 or np.abs(ov - t).min() >= margin
