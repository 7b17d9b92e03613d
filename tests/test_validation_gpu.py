"""GPU: the validation pass on the device (mdb_kitti_collect_dets_f32 / mdb_kitti_compact_dets through
monodetr_b200.kitti_eval.DeviceEvaluator and monodetr_b200.tester.Tester) against the reference's golden vectors
(tests/golden/validation.npz) and against the file path it replaces: decode_detections, result files written as the reference's
save_results writes them, kitti_eval.evaluate over those files."""
import os
import types

import numpy as np
import pytest
import torch

from monodetr_b200 import _lib, decode
from monodetr_b200 import kitti_eval as ke
from monodetr_b200 import tester
from oracle import decode as od
from oracle import kitti_eval as ok
from oracle import monodetr_torch as om

pytestmark = pytest.mark.gpu
NAMES = ["Pedestrian", "Car", "Cyclist"]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "validation.npz")))


class Log:
    def __init__(self):
        self.lines = []

    def info(self, s):
        self.lines.append(s)


def fixture_evaluator(golden, gt=True):
    ids = golden["ids"].tolist()
    g = ke.GroundTruth(ok.fixture_annos(golden, "gt_"), ids) if gt else None
    ev = ke.DeviceEvaluator(g, golden["writelist"].tolist(), topk=int(golden["topk"]), class_names=golden["class_names"].tolist(),
                            image_ids=ids)
    rows, count = torch.from_numpy(golden["rows"]).cuda(), torch.from_numpy(golden["count"]).cuda()
    order = np.random.default_rng(1).permutation(len(ids))
    for i in range(0, len(order), 5):
        sl = order[i:i + 5]
        ev.add_rows(rows[sl], count[sl], sl.tolist())
    return ev


def test_table_is_bit_identical_to_the_parsed_files(golden):
    ev = fixture_evaluator(golden)
    p = ke.pack_dt(ok.fixture_annos(golden, "dt_"))
    tf, tc = ev.table_f.cpu().numpy(), ev.table_cls.cpu().numpy()
    info = ev.slot_info.cpu().numpy()
    assert info[0].tolist() == golden["count"].tolist() and (info[1] == 1).all()
    for s, n in enumerate(golden["count"]):
        o = slice(p["dt_off"][s], p["dt_off"][s + 1])
        assert tf[s, :n].view(np.int64).tolist() == p["dt_f"][o].view(np.int64).tolist()       # -0.0 counts
        assert tc[s, :n].tolist() == p["dt_cls"][o].tolist()


def test_result_matches_reference(golden):
    ev = fixture_evaluator(golden)
    log = Log()
    assert ev.result(log) == golden["car"]
    assert log.lines[2:] == [str(golden[f"result{c}"]) for c in range(3)]
    table, aos = ev.counts_table()
    _, ret, _, _ = ke._report(ev.classes, ev.min_overlaps, ke._aps(table, 3, aos), aos)
    keys = sum((golden[f"keys{c}"].tolist() for c in range(3)), [])
    assert list(ret) == keys
    np.testing.assert_array_equal(np.array(list(ret.values())), np.concatenate([golden[f"values{c}"] for c in range(3)]))


def test_write_results_bytes(golden, tmp_path):
    ev = fixture_evaluator(golden, gt=False)
    ev.write_results(str(tmp_path))
    for i, text in zip(golden["ids"], golden["dt_text"]):
        assert (tmp_path / ("%06d.txt" % i)).read_bytes() == str(text).encode()


def heads(seed, B, dev="cuda"):
    h = od.synthetic_heads(seed, B, 50)
    out = {"pred_logits": h["logits"], "pred_boxes": h["boxes"], "pred_3d_dim": h["dim3"], "pred_depth": h["depth"],
           "pred_angle": h["angle"]}
    return {k: torch.from_numpy(v).to(dev) for k, v in out.items()}, torch.from_numpy(h["img_size"]).to(dev), \
        torch.from_numpy(h["P2"]).to(dev)


def write_file_path(res_dir, batches, ids, mean, thr=0.2):
    """The reference's way: decode_detections per batch and one result file per image, formatted as save_results does."""
    os.makedirs(res_dir, exist_ok=True)
    for (out, size, P2), bid in zip(batches, ids):
        dets = decode.extract_dets_from_outputs(out, topk=50)
        res = decode.decode_detections(dets, {"img_id": bid, "img_size": size}, P2, mean, thr)
        for img_id, rows in res.items():
            with open(os.path.join(res_dir, "%06d.txt" % img_id), "w") as f:
                for r in rows:
                    f.write("{} 0.0 0".format(NAMES[int(r[0])]))
                    for v in r[1:]:
                        f.write(" {:.2f}".format(v))
                    f.write("\n")


def labels_near(dt_annos, rng):
    """KITTI-like labels near the detections, so that the AP is not trivially zero."""
    lines = []
    for a in dt_annos:
        out = []
        for j in range(len(a["name"])):
            if rng.random() < 0.4:
                continue
            b = a["bbox"][j] + rng.normal(0, 2.0, 4)
            l, h, w = a["dimensions"][j]
            x, y, z = a["location"][j] + rng.normal(0, 0.1, 3)
            out.append("{} {:.2f} {:d} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f} {:.2f}".format(
                a["name"][j], rng.choice([0.0, 0.2, 0.4]), int(rng.integers(0, 3)), a["alpha"][j], *b, h, w, l, x, y, z,
                a["rotation_y"][j]))
        if rng.random() < 0.2:
            out.append("DontCare -1 -1 -10 500.00 150.00 560.00 190.00 -1 -1 -1 -1000 -1000 -1000 -10")
        lines.append("".join(s + "\n" for s in out))
    return lines


def test_val_sized_set_equals_the_file_path(tmp_path):
    n_img, B = 3769, 32
    ids = sorted(np.random.default_rng(0).choice(7481, n_img, replace=False).tolist())
    mean = od.synthetic_heads(0, 1, 1)["mean_size"]
    batches, bids = [], []
    for k, b0 in enumerate(range(0, n_img, B)):
        nb = min(B, n_img - b0)
        batches.append(heads(100 + k, nb))
        bids.append(ids[b0:b0 + nb])
    write_file_path(str(tmp_path / "res"), batches, bids, mean)
    dt = ke.get_label_annos(str(tmp_path / "res"))
    os.makedirs(tmp_path / "label_2")
    for i, text in zip(ids, labels_near(dt, np.random.default_rng(1))):
        (tmp_path / "label_2" / ("%06d.txt" % i)).write_text(text)
    ref_log = Log()
    ref = ke.evaluate(str(tmp_path / "res"), str(tmp_path / "label_2"), ids, ["Car", "Pedestrian", "Cyclist"], ref_log)
    gt = ke.GroundTruth(ke.get_label_annos(str(tmp_path / "label_2"), ids), ids)
    ev = ke.DeviceEvaluator(gt, ["Car", "Pedestrian", "Cyclist"], cls_mean_size=mean)
    for (out, size, P2), k in zip(batches, range(len(batches))):
        ev.add(out, list(range(k * B, k * B + len(bids[k]))), size, P2)
    log = Log()
    got = ev.result(log)
    assert got == ref and log.lines == ref_log.lines
    assert ref > 0


def test_add_does_not_synchronise():
    ev = ke.DeviceEvaluator(None, image_ids=list(range(8)))
    out, size, P2 = heads(5, 8)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        n0 = _lib.launch_count()
        ev.add(out, [7, 6, 5, 4, 3, 2, 1, 0], size, P2)
        assert _lib.launch_count() - n0 == 3
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_limit_and_bad_slot_errors_name_the_entry_point(golden):
    ev = ke.DeviceEvaluator(None, image_ids=list(range(4)), topk=50)
    rows = torch.zeros(2, 50, 14, device="cuda")
    count = torch.zeros(2, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="mdb_kitti_collect_dets_f32"):
        ev.add_rows(rows, count, [0, 4])
    with pytest.raises(RuntimeError, match="mdb_kitti_collect_dets_f32"):
        ev.add_rows(rows, count, [-1, 0])
    big = torch.zeros(1, ke.MAX_BOXES + 1, 14, device="cuda")
    slot = np.zeros(1, np.int32)
    codes = np.zeros(3, np.int32)
    f = torch.zeros(1, ke.MAX_BOXES + 1, 13, dtype=torch.float64, device="cuda")
    c = torch.zeros(1, ke.MAX_BOXES + 1, dtype=torch.int32, device="cuda")
    info = torch.zeros(3, 1, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="mdb_kitti_collect_dets_f32"):
        _lib.call("mdb_kitti_collect_dets_f32", big, count[:1], slot.ctypes.data, 1, ke.MAX_BOXES + 1, 1, codes.ctypes.data, 3,
                  f, c, info)
    with pytest.raises(RuntimeError, match="mdb_kitti_compact_dets"):
        _lib.call("mdb_kitti_compact_dets", count, f, c, 1, ke.MAX_BOXES + 1, f, c)


class _Loader:
    def __init__(self, dataset, batches):
        self.dataset, self.batches = dataset, batches

    def __iter__(self):
        return iter(self.batches)

    def __len__(self):
        return len(self.batches)


def test_tester_with_the_small_golden_model(tmp_path, monkeypatch):
    """The small golden model in eval mode through Tester.inference() + evaluate() against decode_detections + the
    reference-format files + kitti_eval.evaluate."""
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "model_eval_small.npz"))
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG))
    model.load_state_dict(om.with_aliases(om.deterministic_state_dict()))
    model = model.cuda().eval()
    n_img, B = 6, 2
    images, calibs, sizes = om.synthetic_inputs(n_img, int(g["seed"]), H=int(g["H"]), W=int(g["W"]))
    ids = [3, 8, 15, 16, 42, 77]
    batches = [(images[b:b + B], calibs[b:b + B], {}, {"img_id": torch.tensor(ids[b:b + B]), "img_size": sizes[b:b + B]})
               for b in range(0, n_img, B)]
    with torch.no_grad():                                          # labels near the model's own detections
        outs = [model(x.cuda(), c.cuda(), None, s["img_size"].cuda()) for x, c, _, s in batches]
    mean = np.zeros((3, 3), np.float32)
    write_file_path(str(tmp_path / "ref"), [(o, s["img_size"].cuda(), c.cuda()) for o, (_, c, _, s) in zip(outs, batches)],
                    [ids[b:b + B] for b in range(0, n_img, B)], mean, thr=0.0)
    os.makedirs(tmp_path / "label_2")
    for i, text in zip(ids, labels_near(ke.get_label_annos(str(tmp_path / "ref")), np.random.default_rng(2))):
        (tmp_path / "label_2" / ("%06d.txt" % i)).write_text(text)
    ds = types.SimpleNamespace(idx_list=["%06d" % i for i in ids], label_dir=str(tmp_path / "label_2"), writelist=["Car"],
                               class_name=NAMES, cls_mean_size=mean, split="val", max_objs=50)
    monkeypatch.chdir(tmp_path)
    log = Log()
    t = tester.Tester({"topk": 50, "threshold": 0.0}, model, _Loader(ds, batches[::-1]), log, {"save_path": "out/"})
    was = torch.is_grad_enabled()
    try:
        t.inference()
    finally:
        torch.set_grad_enabled(was)
    car = t.evaluate()
    ref_log = Log()
    ref = ke.evaluate(str(tmp_path / "ref"), ds.label_dir, ids, ["Car"], ref_log)
    assert car == ref and log.lines == ["==> Saving ..."] + ref_log.lines
    for i in ids:
        name = "%06d.txt" % i
        assert (tmp_path / "out" / "monodetr" / "outputs" / "data" / name).read_bytes() == (tmp_path / "ref" / name).read_bytes()
    # save_results on what decode_detections returns writes the same files
    t.output_dir = str(tmp_path / "saved")
    for o, (_, c, _, s) in zip(outs, batches):
        dets = decode.extract_dets_from_outputs(o, topk=50)
        t.save_results(decode.decode_detections(dets, {"img_id": s["img_id"].tolist(), "img_size": s["img_size"].cuda()},
                                                c.cuda(), mean, 0.0))
    for i in ids:
        name = "%06d.txt" % i
        assert (tmp_path / "saved" / "outputs" / "data" / name).read_bytes() == (tmp_path / "ref" / name).read_bytes()
