"""CPU: oracle/validation.py (decoded rows -> result-file text -> parsed annotations -> device table) against the reference's
golden vectors (tests/golden/validation.npz, tools/gen_golden_validation.py); live against the reference's save_results under the
`reference` marker."""
import os
import sys
import types

import numpy as np
import pytest

from oracle import kitti_eval as ok
from oracle import validation as ov


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "validation.npz")))


def test_rows_to_text_and_annotations(golden):
    names = golden["class_names"].tolist()
    dt = ok.fixture_annos(golden, "dt_")
    for s, n in enumerate(golden["count"]):
        text = ov.rows_to_text(golden["rows"][s], int(n), names)
        assert text == str(golden["dt_text"][s])
        got = ov.text_to_anno(text)
        for k, ref in dt[s].items():
            assert np.asarray(got[k]).shape == np.asarray(ref).shape, k
            if k == "name":
                assert got[k].tolist() == ref.tolist()
            else:
                assert np.asarray(got[k], np.float64).view(np.int64).tolist() == np.asarray(ref, np.float64).view(np.int64).tolist(), k


def test_fixture_covers_the_edges(golden):
    rows, count = golden["rows"], golden["count"]
    live = np.concatenate([rows[s, :n, 1:] for s, n in enumerate(count)]).reshape(-1)
    assert (count == 0).sum() >= 2 and not rows[count == 0].any()
    assert (np.abs(live) >= 2 ** 23).any()
    ties = live[np.abs(np.float64(live) * 8 - np.round(np.float64(live) * 8)) == 0]
    assert (np.abs(np.float64(ties) * 100 - np.round(np.float64(ties) * 100)) == 0.5).sum() > 20     # exact 2-decimal ties
    assert "-0.00" in "".join(golden["dt_text"].tolist())
    assert set(np.concatenate([rows[s, :n, 0] for s, n in enumerate(count)]).astype(int)) == {0, 1, 2}
    scores = np.concatenate([rows[s, :n, 13] for s, n in enumerate(count)])
    assert len(scores) - len(np.unique(scores)) > 10
    gt_names = set(ok.fixture_annos(golden, "gt_")[0]["name"].tolist())
    for a in ok.fixture_annos(golden, "gt_"):
        gt_names |= set(a["name"].tolist())
    assert {"Car", "Pedestrian", "Cyclist", "Van", "Person_sitting", "Truck", "DontCare"} <= gt_names


def test_table_identity_on_ties_and_neighbours():
    """rint(x * 100) / 100 == float('{:.2f}'.format(x)) for float32 x, sign of zero included."""
    k = np.arange(-4000, 4000, dtype=np.float64) / 8
    x = np.concatenate([k, np.nextafter(k.astype(np.float32), np.float32(np.inf)), np.nextafter(k.astype(np.float32), np.float32(-np.inf)),
                        np.float32([-0.0, -0.004, 1.005, 3e38, -3e38, 16777217.0, -0.005])]).astype(np.float32)
    want = np.array([float("{:.2f}".format(v)) for v in x.tolist()])
    assert ov.text_round(x).view(np.int64).tolist() == want.view(np.int64).tolist()


@pytest.mark.reference
def test_live_reference_save_results(golden, tmp_path):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tools"))
    from gen_golden_validation import ref_tester
    rows, count, ids = golden["rows"], golden["count"], golden["ids"].tolist()
    names = golden["class_names"].tolist()
    results = {i: [[int(v[0])] + v[1:].tolist() for v in rows[b, :count[b]]] for b, i in enumerate(ids)}
    ref_tester().save_results(types.SimpleNamespace(output_dir=str(tmp_path), dataset_type="KITTI", class_name=names), results)
    for b, i in enumerate(ids):
        assert (tmp_path / "outputs" / "data" / ("%06d.txt" % i)).read_text() == ov.rows_to_text(rows[b], int(count[b]), names)
