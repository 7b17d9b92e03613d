"""GPU: monodetr_b200.detect.Detector and tools/detect.py on the synthetic KITTI folder (tests/synthetic_kitti.py) with seeded
random models, at the suite's small resolution (320 x 96) and at 1280 x 384 -- rows and counts bit for bit those the Tester
decodes for the same batches (first call eager, second captured and replayed, later ones replayed), the command line's files
byte for byte the Tester's, ragged batches, chunking, reproducible mode, a load_state_dict after capture, the graph count, and
a non-default variant."""
import importlib.util
import os

import numpy as np
import pytest
import torch
import yaml

import monodetr_b200
import synthetic_kitti as sk
from monodetr_b200 import _lib
from monodetr_b200 import dataset as ds
from monodetr_b200 import kitti_eval as ke
from monodetr_b200 import tester
from monodetr_b200.detect import Detector
from monodetr_b200.labels import KittiBatchBuilder, LabelBank

pytestmark = pytest.mark.gpu
SMALL, FULL = (320, 96), (1280, 384)
THRESH = 0.0                    # every decoded row is kept: a random model scores low
B = 2


class Log:
    def info(self, s):
        pass


class _Loader:
    def __init__(self, dataset, batches):
        self.dataset, self.batches = dataset, batches

    def __iter__(self):
        return iter(self.batches)

    def __len__(self):
        return len(self.batches)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    sk.write_tree(root)
    return root


def _model(seed=0, **over):
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(seed)
    model, _ = monodetr_b200.build_monodetr(dict(DEFAULT_MODEL_CFG, **over))
    return model.cuda().eval()


class Val:
    """The val split at one resolution: the Tester's batches (KittiBatchBuilder, as the val loader builds them), the frames on
    the host (Pillow) and on the device (ImageBank), and P2."""

    def __init__(self, tree, res, batch=B):
        self.cfg = {"type": "KITTI", "root_dir": tree, "writelist": ["Car"], "meanshape": False, "batch_size": batch}
        self.bank = ds.ImageBank(tree, "val")
        labels = LabelBank.from_kitti(tree, "val")
        self.dataset = ds.KITTI_Dataset("val", self.cfg, img_sizes=self.bank.sizes)
        builder = KittiBatchBuilder(self.cfg, "val", labels, res)
        self.res, self.P2 = res, labels.host_P2
        self.paths = [os.path.join(tree, "training", "image_2", "%06d.png" % i) for i in self.bank.img_ids]
        self.host = [ds.decode_image(p) for p in self.paths]
        self.device = self.bank.views(range(len(self.bank)))
        self.slices = [list(range(b0, min(b0 + batch, len(self.bank)))) for b0 in range(0, len(self.bank), batch)]
        self.batches = []
        for idx in self.slices:
            images = self.bank.views(idx)
            self.batches.append(builder(images, idx, [builder.sampler.sample((im.shape[1], im.shape[0])) for im in images]))

    def run_tester(self, model, save_path):
        """Tester.inference() over the batches; returns the Tester and the raw (rows, count) it decoded per batch."""
        t = tester.Tester({"topk": 50, "threshold": THRESH}, model, _Loader(self.dataset, self.batches), Log(),
                          {"save_path": save_path}, "m")
        raw, add_rows = [], t.evaluator.add_rows
        t.evaluator.add_rows = lambda rows, count, slots: (raw.append((rows.clone(), count.clone())), add_rows(rows, count, slots))
        was = torch.is_grad_enabled()
        try:
            t.inference()
        finally:
            torch.set_grad_enabled(was)
        return t, raw

    def detector(self, model, **kw):
        return Detector(model, cls_mean_size=self.dataset.cls_mean_size, topk=50, threshold=THRESH, resolution=self.res,
                        **dict(dict(max_batch=B), **kw))

    def table(self, results):
        """A DeviceEvaluator table filled with the Detector's rows, the way the Tester fills its own."""
        ev = ke.DeviceEvaluator(None, ["Car"], topk=50, threshold=THRESH, cls_mean_size=self.dataset.cls_mean_size,
                                class_names=self.dataset.class_name, image_ids=self.bank.img_ids)
        for idx, (rows, count) in zip(self.slices, results):
            ev.add_rows(rows, count, idx)
        return ev


@pytest.fixture
def repro():
    prev = monodetr_b200.set_deterministic(True)
    try:
        yield
    finally:
        monodetr_b200.set_deterministic(prev)


@pytest.mark.parametrize("res,where", [(SMALL, "host"), (FULL, "device")])
def test_matches_the_tester_eager_captured_and_replayed(tree, tmp_path, monkeypatch, res, where):
    """Default (not reproducible) mode: the eval forward has no float atomics, so replayed calls give the eager bits."""
    monkeypatch.chdir(tmp_path)
    val = Val(tree, res)
    model = _model()
    t, raw = val.run_tester(model, "out")
    frames = val.host if where == "host" else val.device
    det = val.detector(model)
    for p in range(3):                     # pass 0: batch 0 eager, batch 1 captured + replayed, batch 2 replayed
        n0 = _lib.launch_count()
        results = [det.detect_device([frames[i] for i in idx], val.P2[idx]) for idx in val.slices]
        assert (_lib.launch_count() > n0) == (p == 0)              # passes 1 and 2 launch nothing outside the graph
        assert det.live_graphs == 1
        for b, ((rows, count), (r_rows, r_count)) in enumerate(zip(results, raw)):
            assert torch.equal(count, r_count) and torch.equal(rows, r_rows), (p, b)
        assert torch.equal(val.table(results)._buf, t.evaluator._buf), p
        assert int(sum(c.sum() for _, c in results)) > 0
    host = det.detect([frames[i] for i in val.slices[0]], val.P2[val.slices[0]])
    for b, rows in enumerate(host):
        n = int(raw[0][1][b])
        assert rows.dtype == np.float32 and np.array_equal(rows, raw[0][0][b, :n].cpu().numpy())


def test_cli_files_equal_the_testers(tree, tmp_path, monkeypatch):
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.trainer import get_checkpoint_state, save_checkpoint
    monkeypatch.chdir(tmp_path)
    val = Val(tree, FULL)
    model = _model(seed=3)
    val.run_tester(model, "out")
    save_checkpoint(get_checkpoint_state(model, None, 1), str(tmp_path / "ckpt"))
    cfg = {"dataset": {"meanshape": False, "batch_size": B}, "model": dict(DEFAULT_MODEL_CFG),
           "tester": {"topk": 50, "threshold": THRESH}}
    (tmp_path / "cfg.yaml").write_text(yaml.safe_dump(cfg))
    (tmp_path / "list.txt").write_text("".join(p + "\n" for p in val.paths))
    spec = importlib.util.spec_from_file_location("detect_cli", os.path.join(os.path.dirname(__file__), "..", "tools", "detect.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    cli.main(["--config", str(tmp_path / "cfg.yaml"), "--checkpoint", str(tmp_path / "ckpt.pth"), "--images",
              str(tmp_path / "list.txt"), "--calib", os.path.join(tree, "training", "calib"), "--out", str(tmp_path / "cli")])
    ref_dir = tmp_path / "out" / "m" / "outputs" / "data"
    names = sorted(os.listdir(ref_dir))
    assert names == sorted(os.listdir(tmp_path / "cli")) and len(names) == len(val.paths)
    assert any((ref_dir / n).read_bytes() for n in names)
    for n in names:
        assert (tmp_path / "cli" / n).read_bytes() == (ref_dir / n).read_bytes(), n


def test_mixed_sizes_and_chunks(tree):
    val = Val(tree, SMALL)
    assert len({f.shape for f in val.host}) > 1
    model = _model(seed=1)
    single = val.detector(model, max_batch=1)
    one = [single.detect_device([f], val.P2[i:i + 1]) for i, f in enumerate(val.host)]
    whole = val.detector(model, max_batch=8)
    chunked = val.detector(model, max_batch=4)
    n = len(val.host)
    for _ in range(3):                     # eager, captured + replayed, replayed
        rows, count = whole.detect_device(val.host, val.P2)
        assert torch.equal(rows, torch.cat([r for r, _ in one])) and torch.equal(count, torch.cat([c for _, c in one]))
        c_rows, c_count = chunked.detect_device(val.host, val.P2)           # chunks of 4 and 2
        assert torch.equal(c_rows, rows) and torch.equal(c_count, count) and rows.shape[0] == n
    assert whole.live_graphs == 1 and chunked.live_graphs == 2


def test_reproducible_mode_replay_equals_eager(tree, repro):
    val = Val(tree, SMALL)
    model = _model(seed=2)
    det = val.detector(model)
    frames, P2 = [val.device[i] for i in val.slices[0]], val.P2[val.slices[0]]
    outs = [det.detect_device(frames, P2) for _ in range(3)]
    assert det.live_graphs == 1
    for rows, count in outs[1:]:
        assert torch.equal(rows, outs[0][0]) and torch.equal(count, outs[0][1])


def test_load_state_dict_after_capture(tree):
    """The graph splits the weights where they are and the frozen BatchNorm fold is refreshed in place, so new weights and
    BatchNorm statistics reach the replayed graph without a new capture."""
    val = Val(tree, SMALL)
    model = _model(seed=4)
    det = val.detector(model)
    frames, P2 = [val.device[i] for i in val.slices[1]], val.P2[val.slices[1]]
    before = [det.detect_device(frames, P2) for _ in range(3)]
    graph = det._graphs[B]
    new = _model(seed=5).state_dict()
    g = torch.Generator().manual_seed(0)
    for k in new:
        if k.endswith("running_var") or k.endswith("running_mean"):          # BatchNorm statistics that differ from the init
            new[k] = new[k] + 0.1 * torch.rand(new[k].shape, generator=g).to(new[k].device)
    model.load_state_dict(new)
    n0 = _lib.launch_count()
    after = det.detect_device(frames, P2)
    assert _lib.launch_count() == n0 and det._graphs[B] is graph and det.live_graphs == 1      # replayed
    fresh_model = _model(seed=6)
    fresh_model.load_state_dict(new)
    fresh = val.detector(fresh_model).detect_device(frames, P2)             # first call: eager
    assert torch.equal(after[0], fresh[0]) and torch.equal(after[1], fresh[1])
    assert not torch.equal(after[0], before[2][0])


def test_graph_count_and_no_graph(tree, monkeypatch):
    val = Val(tree, SMALL)
    model = _model(seed=7)
    det = val.detector(model, max_batch=4)
    out = {}
    for n in (1, 2):
        out[n] = [det.detect_device(val.host[:n], val.P2[:n]) for _ in range(3)]
    assert det.live_graphs == 2 and sorted(det._graphs) == [1, 2]
    n0 = _lib.launch_count()
    det.detect_device(val.host[:3], val.P2[:3])
    first = _lib.launch_count() - n0
    det.detect_device(val.host[:3], val.P2[:3])
    assert det.live_graphs == 2 and _lib.launch_count() - n0 == 2 * first                 # a third size stays eager
    n0 = _lib.launch_count()
    det.detect_device(val.host[:2], val.P2[:2])
    assert _lib.launch_count() == n0                                                        # a captured size replays
    monkeypatch.setenv("MDB_NO_GRAPH", "1")
    plain = val.detector(model, max_batch=4)
    for n in (1, 2):
        for _ in range(3):
            rows, count = plain.detect_device(val.host[:n], val.P2[:n])
            assert torch.equal(rows, out[n][2][0]) and torch.equal(count, out[n][2][1])
    assert plain.live_graphs == 0


def test_variant_dab_resnet101_dc5(tree, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    val = Val(tree, SMALL)
    model = _model(seed=8, backbone="resnet101", dilation=True, use_dab=True)
    _, raw = val.run_tester(model, "out")
    det = val.detector(model)
    for _ in range(2):
        for idx, (r_rows, r_count) in zip(val.slices, raw):
            rows, count = det.detect_device([val.host[i] for i in idx], val.P2[idx])
            assert torch.equal(rows, r_rows) and torch.equal(count, r_count)
    assert det.live_graphs == 1
