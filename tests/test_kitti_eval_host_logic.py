"""CPU: monodetr_b200/kitti_eval.py's host logic -- CSR packing, class codes, configuration order, AP arithmetic, result string,
ret_dict, PR_detail_dict, the compute_aos rule, current_classes forms and the label parser -- driven through a stand-in for the
mdb_kitti_* entry points that computes with oracle/kitti_eval.py, compared with the reference's golden vectors."""
import ctypes
import os

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib
from monodetr_b200 import kitti_eval as ke
from oracle import kitti_eval as ok
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import FakeLib

CASES = ("a", "b", "c", "d")


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * max(n, 1)).from_address(int(ptr)))[:n]


def _annos(n_img, off, f, names, extra):
    """Per-image annotation dicts back from the CSR tables (the oracle reads names; class codes become lower-case names)."""
    out = []
    for b in range(n_img):
        s = slice(off[b], off[b + 1])
        a = {"name": np.array(names[s]), "bbox": f[s, 0:4], "alpha": f[s, 4], "location": f[s, 6:9],
             "dimensions": f[s, 9:12], "rotation_y": f[s, 12]}
        a.update({k: v[s] for k, v in extra.items()})
        out.append(a)
    return out


def _name(code, dontcare=0):
    return "DontCare" if dontcare else (ok.CLASS_NAMES[code] if code >= 0 else "other")


class KittiFakeLib(FakeLib):
    """mdb_kitti_* computed by the oracle from the packed host tables."""

    def _unpack(self, gt_off, dt_off, n_img, gt_f, gt_i, dt_f, dt_cls):
        go, do = _arr(gt_off, ctypes.c_int32, n_img + 1), _arr(dt_off, ctypes.c_int32, n_img + 1)
        ng, nd = int(go[-1]), int(do[-1])
        gf = _arr(gt_f, ctypes.c_double, ng * 13).reshape(ng, 13)
        df = _arr(dt_f, ctypes.c_double, nd * 13).reshape(nd, 13)
        gi = _arr(gt_i, ctypes.c_int32, ng * 3).reshape(ng, 3) if gt_i else np.zeros((ng, 3), np.int32)
        dc = _arr(dt_cls, ctypes.c_int32, nd) if dt_cls else np.zeros(nd, np.int32)
        gt = _annos(n_img, go, gf, [_name(c, d) for c, d in zip(gi[:, 1], gi[:, 2])],
                    {"truncated": gf[:, 5], "occluded": gi[:, 0]})
        dt = _annos(n_img, do, df, [_name(c) for c in dc], {"score": df[:, 5]})
        return gt, dt

    def mdb_kitti_overlaps(self, gt_off, dt_off, ov_off, n_img, max_gt, max_dt, n_ov, gt_f, dt_f, out, stream):
        gt, dt = self._unpack(gt_off, dt_off, n_img, gt_f, None, dt_f, None)
        o = _arr(out, ctypes.c_double, 3 * n_ov).reshape(3, n_ov)
        offs = _arr(ov_off, ctypes.c_int64, n_img + 1)
        for b, (g, d) in enumerate(zip(gt, dt)):
            for m, block in enumerate(ok.image_overlaps(g, d)):
                o[m, offs[b]:offs[b + 1]] = block.reshape(-1)
        return 0

    def mdb_kitti_eval_workspace_bytes(self, n_img, n_gt, n_dt, n_cls, compute_aos):
        return 256

    def mdb_kitti_eval(self, gt_off, dt_off, ov_off, n_img, n_gt, n_dt, max_gt, max_dt, n_ov, gt_f, gt_i, dt_f, dt_cls, overlaps,
                       classes, min_overlaps, n_cls, compute_aos, ws, ws_bytes, result, stream):
        self.evals.append((n_img, n_gt, n_dt, max_gt, max_dt, n_ov))
        gt, dt = self._unpack(gt_off, dt_off, n_img, gt_f, gt_i, dt_f, dt_cls)
        cls = _arr(classes, ctypes.c_int32, n_cls).tolist()
        mo = _arr(min_overlaps, ctypes.c_double, 6 * n_cls).reshape(2, 3, n_cls)
        table = ok.eval_table(gt, dt, cls, mo, bool(compute_aos))
        _arr(result, ctypes.c_double, table.size)[:] = table.reshape(-1)
        return 0


@pytest.fixture
def fake(monkeypatch):
    fake_device_lib.install(monkeypatch)
    lib = KittiFakeLib(1)
    lib.evals = []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(ke, "_device", lambda: torch.device("cpu"))
    return lib


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_eval.npz")))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


def _anno(names, boxes, alpha=0.0, score=0.5):
    n = len(names)
    return {"name": np.array(names), "truncated": np.zeros(n), "occluded": np.zeros(n, np.int64), "alpha": np.full(n, alpha),
            "bbox": np.array(boxes, np.float64).reshape(n, 4), "dimensions": np.tile([4.0, 1.5, 1.6], (n, 1)),
            "location": np.tile([1.0, 1.5, 20.0], (n, 1)), "rotation_y": np.zeros(n), "score": np.full(n, score)}


def test_pack_csr_and_class_codes():
    gt = [_anno(["Car", "DontCare", "dontcare", "Person_sitting"], [[0, 0, 10, 50]] * 4), _anno([], []),
          _anno(["VAN", "Misc"], [[1, 2, 3, 4]] * 2)]
    dt = [_anno(["Pedestrian"], [[0, 0, 1, 1]]), _anno(["Truck", "Cyclist"], [[0, 0, 1, 1]] * 2), _anno([], [])]
    p = ke.pack(gt, dt)
    np.testing.assert_array_equal(p["gt_off"], [0, 4, 4, 6])
    np.testing.assert_array_equal(p["dt_off"], [0, 1, 3, 3])
    np.testing.assert_array_equal(p["ov_off"], [0, 4, 4, 4])
    assert (p["n_img"], p["n_gt"], p["n_dt"], p["n_ov"], p["max_gt"], p["max_dt"]) == (3, 6, 3, 4, 4, 2)
    np.testing.assert_array_equal(p["gt_i"][:, 1], [0, -1, -1, 4, 3, -1])
    np.testing.assert_array_equal(p["gt_i"][:, 2], [0, 1, 0, 0, 0, 0])                 # "DontCare" is case-sensitive
    np.testing.assert_array_equal(p["dt_cls"], [1, 5, 2])
    assert p["gt_f"].shape == (6, 13) and p["dt_f"].shape == (3, 13)
    np.testing.assert_array_equal(p["gt_f"][0], [0, 0, 10, 50, 0.0, 0.0, 1.0, 1.5, 20.0, 4.0, 1.5, 1.6, 0.0])
    assert p["dt_f"][0, 5] == 0.5                                                       # score column


@pytest.mark.parametrize("case", CASES)
def test_official_result_matches_reference(fake, golden, case):
    gt, dt = annos(golden, case)
    for c in range(3):
        pr = {}
        text, ret, first = ke.get_official_eval_result(gt, dt, c, PR_detail_dict=pr)
        assert text == str(golden[f"{case}__result{c}"])
        assert list(ret) == golden[f"{case}__keys{c}"].tolist()
        np.testing.assert_array_equal(np.array(list(ret.values())), golden[f"{case}__values{c}"])
        assert first == golden[f"{case}__first{c}"] or (np.isnan(first) and np.isnan(golden[f"{case}__first{c}"]))
        prefix = f"{case}__pr{c}_"
        assert set(pr) == {k[len(prefix):] for k in golden if k.startswith(prefix)}
        for k, v in pr.items():
            np.testing.assert_array_equal(v, golden[f"{case}__pr{c}_{k}"])


@pytest.mark.parametrize("case", CASES)
def test_do_eval_all_classes_in_one_call(fake, golden, case):
    gt, dt = annos(golden, case)
    got = ke.do_eval(gt, dt, [0, 1, 2], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], bool(golden[f"{case}__compute_aos"]))
    for i, g in enumerate(got):
        ref = golden[f"{case}__do_eval{i}"]
        if g is None:
            assert ref.size == 0
        else:
            np.testing.assert_array_equal(g, ref)
    assert len(fake.evals) == 1


def test_one_device_call_counts_six_launches(fake, golden):
    gt, dt = annos(golden, "b")
    n0 = _lib.launch_count()
    ke.get_official_eval_result(gt, dt, ["Car", "Pedestrian", "Cyclist"])
    assert _lib.launch_count() - n0 == 6 and len(fake.evals) == 1


def test_current_classes_forms(fake, golden):
    gt, dt = annos(golden, "a")
    ref0, ref1 = str(golden["a__result0"]), str(golden["a__result1"])
    assert ke.get_official_eval_result(gt, dt, 0)[0] == ref0
    assert ke.get_official_eval_result(gt, dt, "Car")[0] == ref0
    assert ke.get_official_eval_result(gt, dt, ["Car"])[0] == ref0
    text, ret, first = ke.get_official_eval_result(gt, dt, ["Car", 1])
    assert text == ref0 + ref1
    assert first == golden["a__first0"]
    assert list(ret) == golden["a__keys0"].tolist() + golden["a__keys1"].tolist()


def test_compute_aos_rule(fake, golden):
    gt, dt = annos(golden, "a")
    assert "aos  AP" in ke.get_official_eval_result(gt, dt, 0)[0]
    # the first image with detections decides: alpha[0] == -10 there switches AOS off for the whole set
    first = next(i for i, d in enumerate(dt) if len(d["name"]))
    dt = [dict(d) for d in dt]
    dt[first]["alpha"] = dt[first]["alpha"].copy()
    dt[first]["alpha"][0] = -10
    text, ret, _ = ke.get_official_eval_result(gt, dt, 0)
    assert "aos" not in text and not any("aos" in k for k in ret)
    gt_c, dt_c = annos(golden, "c")
    assert "aos" not in ke.get_official_eval_result(gt_c, dt_c, 0)[0]


def test_no_detections_anywhere(fake, golden):
    gt, _ = annos(golden, "a")
    text, ret, first = ke.get_official_eval_result(gt, [_anno([], [])] * len(gt), [0, 1, 2])
    assert first == 0.0 and all(v == 0.0 for v in ret.values())
    assert "aos" not in text


def test_label_parser_matches_reference(golden, tmp_path):
    ids = golden["d__ids"].tolist()
    for sub, lines in (("label", golden["d__gt_lines"]), ("res", golden["d__dt_lines"])):
        os.makedirs(tmp_path / sub)
        for i, text in zip(ids, lines):
            (tmp_path / sub / ("%06d.txt" % i)).write_text(str(text) + ("\n" if str(text) else ""))
    (tmp_path / "res" / "notes.txt").write_text("not a result file\n")
    gt = ke.get_label_annos(str(tmp_path / "label"), ids)
    dt = ke.get_label_annos(str(tmp_path / "res"))
    for got, ref in ((gt, ok.fixture_annos(golden, "d__gt_")), (dt, ok.fixture_annos(golden, "d__dt_"))):
        assert len(got) == len(ref)
        for g, r in zip(got, ref):
            for k in r:
                assert g[k].shape == r[k].shape, k
                np.testing.assert_array_equal(g[k], r[k])


def test_evaluate_folder(fake, golden, tmp_path):
    ids = golden["d__ids"].tolist()
    for sub, lines in (("label", golden["d__gt_lines"]), ("res", golden["d__dt_lines"])):
        os.makedirs(tmp_path / sub)
        for i, text in zip(ids, lines):
            (tmp_path / sub / ("%06d.txt" % i)).write_text(str(text) + ("\n" if str(text) else ""))

    class Log:
        lines = []

        def info(self, s):
            self.lines.append(s)
    log = Log()
    car = ke.evaluate(str(tmp_path / "res"), str(tmp_path / "label"), ids, logger=log)
    assert car == golden["d__first0"]
    assert [str(golden[f"d__result{c}"]) for c in range(3)] == log.lines[2:]
    assert len(fake.evals) == 1
