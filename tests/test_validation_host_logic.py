"""CPU: the validation pass on the device (monodetr_b200.kitti_eval.GroundTruth / DeviceEvaluator, monodetr_b200.tester.Tester)
driven through a stand-in for mdb_kitti_collect_dets_f32 / mdb_kitti_compact_dets that computes with oracle/validation.py, on
top of the mdb_kitti_* stand-in of test_kitti_eval_host_logic.py; compared with the reference's golden vectors
(tests/golden/validation.npz): slot mapping, class mapping, compaction offsets, the repeated / missing image errors, the result
strings and the written bytes."""
import ctypes
import os
import types

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib
from monodetr_b200 import kitti_eval as ke
from monodetr_b200 import tester as tester_mod
from oracle import decode as od
from oracle import kitti_eval as ok
from oracle import validation as ov
import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from test_kitti_eval_host_logic import KittiFakeLib, _arr


class ValidationFakeLib(KittiFakeLib):
    """mdb_kitti_collect_dets_f32 / mdb_kitti_compact_dets on host memory, restated with oracle/validation.py."""

    def mdb_kitti_collect_dets_f32(self, rows, count, slot, B, topk, n_img, cls_code, n_code, table_f, table_cls, slot_info,
                                   stream):
        slots = _arr(slot, ctypes.c_int32, B).copy()
        if (slots < 0).any() or (slots >= n_img).any() or topk > ke.MAX_BOXES:
            return -1
        self.collects.append(B)
        r = _arr(rows, ctypes.c_float, B * topk * 14).reshape(B, topk, 14)
        cnt = _arr(count, ctypes.c_int32, B)
        codes = _arr(cls_code, ctypes.c_int32, n_code).tolist()
        tf = _arr(table_f, ctypes.c_double, n_img * topk * 13).reshape(n_img, topk, 13)
        tc = _arr(table_cls, ctypes.c_int32, n_img * topk).reshape(n_img, topk)
        info = _arr(slot_info, ctypes.c_int32, 3 * n_img).reshape(3, n_img)
        for b, s in enumerate(slots):
            n = int(cnt[b])
            tf[s, :n], tc[s, :n] = ov.rows_to_table(r[b], n, codes)
            info[0, s], info[1, s] = n, info[1, s] + 1
            info[2, s] = int(n > 0 and ov.text_round(r[b, 0, 1]) != -10.0)
        return 0

    def mdb_kitti_compact_dets(self, dt_off, table_f, table_cls, n_img, topk, dt_f, dt_cls, stream):
        off = _arr(dt_off, ctypes.c_int32, n_img + 1)
        self.compacts.append(off.copy())
        tf = _arr(table_f, ctypes.c_double, n_img * topk * 13).reshape(n_img, topk, 13)
        tc = _arr(table_cls, ctypes.c_int32, n_img * topk).reshape(n_img, topk)
        n_dt = int(off[-1])
        of = _arr(dt_f, ctypes.c_double, n_dt * 13).reshape(n_dt, 13)
        oc = _arr(dt_cls, ctypes.c_int32, n_dt)
        for s in range(n_img):
            n = off[s + 1] - off[s]
            of[off[s]:off[s + 1]], oc[off[s]:off[s + 1]] = tf[s, :n], tc[s, :n]
        return 0


@pytest.fixture
def fake(monkeypatch):
    fake_device_lib.install(monkeypatch)
    lib = ValidationFakeLib(1)
    lib.evals, lib.collects, lib.compacts = [], [], []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(ke, "_device", lambda: torch.device("cpu"))
    return lib


@pytest.fixture
def grad_mode():
    """Tester.inference() turns autograd off, as the reference's does; put it back whatever the test does."""
    was = torch.is_grad_enabled()
    yield
    torch.set_grad_enabled(was)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "validation.npz")))


class Log:
    def __init__(self):
        self.lines = []

    def info(self, s):
        self.lines.append(s)


def evaluator(golden, gt=True, **kw):
    ids = golden["ids"].tolist()
    g = ke.GroundTruth(ok.fixture_annos(golden, "gt_"), ids) if gt else None
    return ke.DeviceEvaluator(g, golden["writelist"].tolist(), topk=int(golden["topk"]),
                              class_names=golden["class_names"].tolist(), image_ids=ids, **kw)


def add_shuffled(ev, golden, batch=5, seed=0):
    """Every image once, in a shuffled order and in batches: the slot decides where an image lands."""
    rows, count = torch.from_numpy(golden["rows"]), torch.from_numpy(golden["count"])
    order = np.random.default_rng(seed).permutation(len(count))
    for i in range(0, len(order), batch):
        sl = order[i:i + batch]
        ev.add_rows(rows[sl].clone(), count[sl].clone(), sl.tolist())


def test_oracle_table_is_the_parsed_text(golden):
    codes = [ke._class_code(n) for n in golden["class_names"]]
    dt = ok.fixture_annos(golden, "dt_")
    p = ke.pack_dt(dt)
    for s, n in enumerate(golden["count"]):
        f, c = ov.rows_to_table(golden["rows"][s], int(n), codes)
        o = slice(p["dt_off"][s], p["dt_off"][s + 1])
        assert f.view(np.int64).tolist() == p["dt_f"][o].view(np.int64).tolist()     # bit for bit, -0.0 included
        assert c.tolist() == p["dt_cls"][o].tolist()


def test_result_matches_reference(fake, golden):
    ev = evaluator(golden)
    add_shuffled(ev, golden)
    log = Log()
    car = ev.result(log)
    assert car == golden["car"]
    assert log.lines[:2] == ["==> Loading detections and GTs...", "==> Evaluating (official) ..."]
    assert log.lines[2:] == [str(golden[f"result{c}"]) for c in range(3)]
    assert len(fake.evals) == 1 and len(fake.compacts) == 1
    np.testing.assert_array_equal(fake.compacts[0], np.concatenate([[0], np.cumsum(golden["count"])]))
    # the device table holds the parsed result-file values, in the split's order
    p = ke.pack_dt(ok.fixture_annos(golden, "dt_"))
    tf = ev.table_f.numpy()
    for s, n in enumerate(golden["count"]):
        o = slice(p["dt_off"][s], p["dt_off"][s + 1])
        assert tf[s, :n].view(np.int64).tolist() == p["dt_f"][o].view(np.int64).tolist()
        assert ev.table_cls.numpy()[s, :n].tolist() == p["dt_cls"][o].tolist()


def test_same_result_as_the_annotation_path(fake, golden):
    ev = evaluator(golden)
    add_shuffled(ev, golden, batch=48)
    table, aos = ev.counts_table()
    gt, dt = ok.fixture_annos(golden, "gt_"), ok.fixture_annos(golden, "dt_")
    ref = ke.eval_counts(gt, dt, [0, 1, 2], ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]], aos)
    assert aos is True
    assert table.tobytes() == ref.tobytes()


def test_write_results_bytes(fake, golden, tmp_path):
    ev = evaluator(golden, gt=False)
    add_shuffled(ev, golden, batch=7)
    ev.write_results(str(tmp_path))
    for i, text in zip(golden["ids"], golden["dt_text"]):
        assert (tmp_path / ("%06d.txt" % i)).read_bytes() == str(text).encode()
    assert sorted(os.listdir(tmp_path)) == ["%06d.txt" % i for i in golden["ids"]]
    with pytest.raises(ValueError, match="GroundTruth"):
        ev.result()


def test_repeated_and_missing_images_raise(fake, golden):
    ev = evaluator(golden)
    rows, count = torch.from_numpy(golden["rows"]), torch.from_numpy(golden["count"])
    n = len(count)
    ev.add_rows(rows[:n - 1].clone(), count[:n - 1].clone(), list(range(n - 1)))
    with pytest.raises(ValueError, match="never added"):
        ev.result()
    ev.add_rows(rows[:2].clone(), count[:2].clone(), [n - 1, 0])
    with pytest.raises(ValueError, match="more than once"):
        ev.result()
    ev.reset()
    add_shuffled(ev, golden)
    assert ev.result(Log()) == golden["car"]


def test_bad_slot_and_limits(fake, golden):
    ev = evaluator(golden)
    rows, count = torch.from_numpy(golden["rows"]), torch.from_numpy(golden["count"])
    with pytest.raises(RuntimeError, match="mdb_kitti_collect_dets_f32"):
        ev.add_rows(rows[:2].clone(), count[:2].clone(), [0, len(count)])
    with pytest.raises(ValueError, match="rows"):
        ev.add_rows(rows[:2].clone(), count[:2].clone(), [0])
    with pytest.raises(TypeError, match="host integers"):                      # reading device slots would synchronise
        ev.add_rows(rows[:1].clone(), count[:1].clone(), torch.zeros(1, dtype=torch.int32, device="meta"))
    with pytest.raises(ValueError, match="topk"):
        ke.DeviceEvaluator(None, image_ids=[0], topk=ke.MAX_BOXES + 1)
    with pytest.raises(ValueError, match="class_names"):
        ke.DeviceEvaluator(None, image_ids=[0], class_names=["Car", "Dog"])


def test_add_counts_three_launches(fake, golden):
    ev = ke.DeviceEvaluator(None, image_ids=list(range(4)), topk=50)
    h = od.synthetic_heads(3, 4, 50)
    out = {"pred_logits": torch.from_numpy(h["logits"]), "pred_boxes": torch.from_numpy(h["boxes"]),
           "pred_3d_dim": torch.from_numpy(h["dim3"]), "pred_depth": torch.from_numpy(h["depth"]),
           "pred_angle": torch.from_numpy(h["angle"])}
    n0 = _lib.launch_count()
    ev.add(out, [3, 1, 0, 2], torch.from_numpy(h["img_size"]), torch.from_numpy(h["P2"]))
    assert _lib.launch_count() - n0 == 3 and fake.collects == [4]


# ------------------------------------------------------------------------------------------------------------------ Tester
class _Heads(torch.nn.Module):
    """A stand-in model: seeded head outputs per batch, keyed by the first image's id."""

    def forward(self, images, calibs, targets, img_sizes, dn_args=None):
        h = od.synthetic_heads(int(images[0, 0, 0, 0]), images.shape[0], 50)
        return {"pred_logits": torch.from_numpy(h["logits"]), "pred_boxes": torch.from_numpy(h["boxes"]),
                "pred_3d_dim": torch.from_numpy(h["dim3"]), "pred_depth": torch.from_numpy(h["depth"]),
                "pred_angle": torch.from_numpy(h["angle"])}


def _loader(golden, tmp_path, batch=5):
    ids = golden["ids"].tolist()
    label_dir = tmp_path / "label_2"
    os.makedirs(label_dir)
    for i, text in zip(ids, golden["gt_text"]):
        (label_dir / ("%06d.txt" % i)).write_text(str(text))
    h = od.synthetic_heads(11, len(ids), 1)
    batches = []
    for b0 in range(0, len(ids), batch):
        sl = slice(b0, b0 + batch)
        n = len(ids[sl])
        inputs = torch.full((n, 3, 4, 4), float(b0 + 1))
        batches.append((inputs, torch.from_numpy(h["P2"][sl]), {}, {"img_id": torch.tensor(ids[sl]),
                                                                    "img_size": torch.from_numpy(h["img_size"][sl])}))
    ds = types.SimpleNamespace(idx_list=["%06d" % i for i in ids], label_dir=str(label_dir), writelist=["Car", "Pedestrian"],
                               class_name=["Pedestrian", "Car", "Cyclist"], cls_mean_size=od.synthetic_heads(0, 1, 1)["mean_size"],
                               split="val", max_objs=50)
    return ds, batches


class _Loader:
    def __init__(self, dataset, batches):
        self.dataset, self.batches = dataset, batches

    def __iter__(self):
        return iter(self.batches)

    def __len__(self):
        return len(self.batches)


def test_tester_matches_file_path(fake, golden, tmp_path, monkeypatch, grad_mode):
    from monodetr_b200 import decode
    ds, batches = _loader(golden, tmp_path)
    loader = _Loader(ds, batches[::-1])                                 # any batch order
    monkeypatch.chdir(tmp_path)
    log = Log()
    t = tester_mod.Tester({"topk": 50, "threshold": 0.2}, _Heads(), loader, log, {"save_path": "out/"})
    t.inference()
    car = t.evaluate()
    # the reference's way: decode_detections per batch, save_results, KITTI_Dataset.eval over the files
    ref_dir = tmp_path / "ref"
    os.makedirs(ref_dir)
    for inputs, calibs, _, info in batches:
        dets = decode.extract_dets_from_outputs(_Heads()(inputs, calibs, None, info["img_size"]), topk=50)
        res = decode.decode_detections(dets, info, calibs, ds.cls_mean_size, 0.2)
        for img_id, rows in res.items():
            text = "".join("{} 0.0 0".format(ds.class_name[int(r[0])]) + "".join(" {:.2f}".format(v) for v in r[1:]) + "\n"
                           for r in rows)
            (ref_dir / ("%06d.txt" % img_id)).write_text(text)
            assert (tmp_path / "out" / "monodetr" / "outputs" / "data" / ("%06d.txt" % img_id)).read_text() == text
    ref_log = Log()
    ref_car = ke.evaluate(str(ref_dir), ds.label_dir, golden["ids"].tolist(), ["Car", "Pedestrian"], ref_log)
    assert car == ref_car
    assert log.lines == ["==> Saving ..."] + ref_log.lines
    assert not torch.is_grad_enabled()


def test_tester_save_results_writes_the_reference_files(fake, golden, tmp_path, monkeypatch):
    """Tester.save_results on decode_detections-shaped results ({img_id: [[int cls, 13 floats], ...]}) against the files the
    reference's save_results wrote for the same rows."""
    ds, _ = _loader(golden, tmp_path)
    monkeypatch.chdir(tmp_path)
    t = tester_mod.Tester({"topk": 50}, _Heads(), _Loader(ds, []), Log(), {"save_path": "out/"})
    rows, count = golden["rows"], golden["count"]
    results = {int(i): [[int(v[0])] + v[1:].tolist() for v in rows[b, :count[b]]] for b, i in enumerate(golden["ids"])}
    t.save_results(results)
    data = tmp_path / "out" / "monodetr" / "outputs" / "data"
    assert sorted(os.listdir(data)) == ["%06d.txt" % i for i in golden["ids"]]
    for i, text in zip(golden["ids"], golden["dt_text"]):
        assert (data / ("%06d.txt" % i)).read_bytes() == str(text).encode()
