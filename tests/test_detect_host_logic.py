"""CPU: the host side of monodetr_b200.detect.Detector and tools/detect.py over the fake device library -- argument checks before
any library call, the pre-process metadata / calibs / img_sizes against the reference dataset's eval branch
(tests/golden/preprocess.npz pins get_affine_transform), frame staging, chunk and output order, from_config, and the command
line's parsing, file naming and output files."""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

import fake_device_lib
from monodetr_b200 import _lib, detect, kitti_eval
from monodetr_b200 import preprocess as pp
from monodetr_b200.labels import CLASS_NAMES, CLS_MEAN_SIZE, AugmentationSampler
from oracle import decode as od
from oracle import preprocess as op

RES = (32, 12)


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(int(ptr))).copy()


class DetectFakeLib(fake_device_lib.FakeLib):
    def mdb_warp_affine_normalize_u8(self, src, wh, pitch, trans_inv, flip, B, W, H, mean3, std3, out, stream):
        s, p = _arr(src, ctypes.c_int64, B), _arr(pitch, ctypes.c_int64, B)
        sizes = _arr(wh, ctypes.c_int32, 2 * B).reshape(B, 2)
        tinv = _arr(trans_inv, ctypes.c_double, 6 * B).reshape(B, 6)
        fl = _arr(flip, ctypes.c_uint8, B)
        self.warps.append(dict(src=s, pitch=p, wh=sizes, trans_inv=tinv, flip=fl))
        o = fake_device_lib.f32(out, B, 3, H, W)
        for b in range(B):
            w, h = (int(v) for v in sizes[b])
            img = _arr(s[b], ctypes.c_uint8, h * int(p[b])).reshape(h, int(p[b]))[:, :3 * w].reshape(h, w, 3)
            o[b].copy_(torch.from_numpy(op.preprocess(img, tinv[b], (W, H), bool(fl[b]))))
        return 0


class StubModel(torch.nn.Module):
    """Records what the forward reads; each frame's heads are seeded by its P2[0, 3], so a frame's rows do not depend on the
    batch it is in."""

    def __init__(self):
        super().__init__()
        self.w = torch.nn.Parameter(torch.zeros(3))
        self.seen = []

    def forward(self, images, calibs, targets, img_sizes, dn_args=None):
        self.seen.append(dict(images=images.clone(), calibs=calibs.clone(), img_sizes=img_sizes.clone(), dn_args=dn_args))
        hs = [od.synthetic_heads(int(c[0, 3]), 1, 50) for c in calibs]
        cat = {k: torch.from_numpy(np.concatenate([h[k] for h in hs])) for k in ("logits", "boxes", "dim3", "depth", "angle")}
        return {"pred_logits": cat["logits"], "pred_boxes": cat["boxes"], "pred_3d_dim": cat["dim3"], "pred_depth": cat["depth"],
                "pred_angle": cat["angle"]}


@pytest.fixture
def fake(monkeypatch):
    fake_device_lib.install(monkeypatch)
    lib = DetectFakeLib(1)
    lib.warps = []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(detect, "_require_cuda", lambda device: None)
    monkeypatch.setattr(pp, "_require_cuda", lambda device: None)
    monkeypatch.setattr(detect, "_pinned", lambda n: torch.empty(n, dtype=torch.uint8))
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    return lib


def _detector(model=None, **kw):
    d = detect.Detector(model or StubModel(), device="cpu", **dict(dict(resolution=RES, max_frame=(40, 20)), **kw))
    d.use_graphs = False
    return d


def _frames(sizes, seed=0):
    return op.synthetic_images(seed, sizes)


def _p2(n, seed=1):
    P2 = np.tile(np.array([[700.0, 0, 600, 45], [0, 700, 170, 0.2], [0, 0, 1, 0.003]], np.float32), (n, 1, 1))
    P2[:, 0, 3] = np.arange(n) + 100 * seed                # the stub's per-frame seed
    return P2


# ---- argument checks --------------------------------------------------------------------------------------------------------
def _bad_inputs():
    ok = _frames([(20, 10), (18, 9)])
    big = np.zeros((10, 41, 3), np.uint8)
    tall = np.zeros((21, 10, 3), np.uint8)
    nan = _p2(2)
    nan[1, 2, 2] = np.nan
    inf = _p2(2).astype(np.float64)
    inf[0, 0, 0] = 1e39                                    # finite in float64, not in float32
    return [
        ("frame 1: dtype", [ok[0], ok[1].astype(np.float32)], _p2(2)),
        ("frame 0: dtype", [torch.from_numpy(ok[0]).int(), ok[1]], _p2(2)),
        ("frame 1: shape", [ok[0], ok[1][:, :, :2]], _p2(2)),
        ("frame 0: shape", [ok[0][None], ok[1]], _p2(2)),
        ("frame 1: 41 x 10", [ok[0], big], _p2(2)),
        ("frame 0: 10 x 21", [tall, ok[1]], _p2(2)),
        ("frame 1: a numpy array", [ok[0], ok[1].tolist()], _p2(2)),
        ("P2 of frame 1 is not finite", ok, nan),
        ("P2 of frame 0 is not finite", ok, inf),
        ("P2: shape", ok, _p2(2)[:, :, :3]),
        ("P2: shape", ok, _p2(2)[0]),
        ("2 frames but 3 P2", ok, _p2(3)),
        ("list of", np.stack(ok[:1]), _p2(1)),
    ]


@pytest.mark.parametrize("case", range(13))
def test_bad_inputs_raise_before_any_library_call(fake, case):
    want, frames, P2 = _bad_inputs()[case]
    d = _detector()
    fake.calls.clear()
    for call in (d.detect, d.detect_device):
        with pytest.raises(ValueError, match=want.replace("(", r"\(")):
            call(frames, P2)
    assert not fake.calls and not d.model.seen


def test_empty_call(fake):
    d = _detector()
    assert d.detect([], np.zeros((0, 3, 4))) == []
    rows, count = d.detect_device([], np.zeros((0, 3, 4)))
    assert rows.shape == (0, 50, 14) and count.shape == (0,) and not fake.calls.get("mdb_warp_affine_normalize_u8")


def test_constructor_checks(fake):
    for kw in (dict(topk=0), dict(max_batch=0), dict(max_frame=(0, 10)), dict(cls_mean_size=np.zeros((3, 2)))):
        with pytest.raises(ValueError):
            _detector(**kw)
    m = StubModel().train()
    _detector(m)
    assert not m.training                                  # the Detector puts the model in eval mode


# ---- what the pre-process and the forward read ------------------------------------------------------------------------------
def test_eval_branch_metadata_calibs_and_img_sizes(fake):
    """trans_inv of each frame is the reference's eval branch (get_affine_transform(img_size / 2, img_size, 0, resolution,
    inv=1)): bit for bit the golden cv2 values of tests/golden/preprocess.npz and the loader's val records; calibs = P2 and
    img_sizes = (W, H) as the val loader gives them; the warp reads each frame from its slot."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "preprocess.npz"))
    res = tuple(int(v) for v in g["resolution"])
    sizes = [tuple(int(v) for v in g["sizes"][i]) for i in (0, 1)]
    for i in (0, 1):                                       # the golden cases drawn without augmentation
        assert np.array_equal(g[f"{i}.center"], np.array(sizes[i]) / 2) and np.array_equal(g[f"{i}.crop_size"], sizes[i])
    model = StubModel()
    d = _detector(model, resolution=res, max_frame=(320, 100), max_batch=4)
    frames = _frames(sizes + [(200, 60)], seed=5)
    frames[1] = torch.from_numpy(frames[1])               # host tensors and arrays alike
    P2 = _p2(3)
    d.detect(frames, P2)
    (w,) = fake.warps
    val = AugmentationSampler("val", resolution=res)
    for b, f in enumerate(frames):
        H, W = f.shape[:2]
        assert w["trans_inv"][b].view(np.int64).tolist() == val.sample((W, H)).trans_inv.reshape(6).view(np.int64).tolist()
        if b < 2:
            assert w["trans_inv"][b].view(np.int64).tolist() == g[f"{b}.trans_inv"].reshape(6).view(np.int64).tolist()
    assert w["wh"].tolist() == [[f.shape[1], f.shape[0]] for f in frames] and not w["flip"].any()
    assert w["pitch"].tolist() == [3 * f.shape[1] for f in frames]
    assert len(set(np.diff(w["src"]).tolist())) == 1      # fixed slots, one per frame
    (seen,) = model.seen
    assert seen["calibs"].dtype == torch.float32 and np.array_equal(seen["calibs"].numpy(), P2)
    assert seen["img_sizes"].dtype == torch.int64 and seen["img_sizes"].tolist() == w["wh"].tolist()
    assert seen["dn_args"] == 0
    for b, f in enumerate(frames):
        f = np.asarray(f)
        want = op.preprocess(f, val.sample((f.shape[1], f.shape[0])).trans_inv.reshape(6), res)
        assert np.array_equal(seen["images"][b].numpy(), want), b


def test_metadata_matches_the_one_call_preprocessor(fake):
    """ImageBatchPreprocessor.__call__ is metadata + one upload + launch: same words, same output."""
    frames = [torch.from_numpy(f) for f in _frames([(20, 10), (17, 9)])]
    tinv = np.stack([pp.get_affine_transform(np.array([W, H]) / 2, np.array([W, H]), 0, np.array(RES), inv=1)[1]
                     for W, H in [(20, 10), (17, 9)]])
    pre = pp.ImageBatchPreprocessor(RES, device="cpu")
    out = pre(frames, tinv, [True, False])
    buf = pre.metadata(np.full(pp.metadata_words(2) + 3, 7, np.int64), [f.data_ptr() for f in frames], [60, 51],
                       [(20, 10), (17, 9)], tinv, [True, False])
    assert buf[-3:].tolist() == [7, 7, 7]                 # nothing written past the metadata
    w = fake.warps[-1]
    assert w["src"].tolist() == buf[:2].tolist() and w["pitch"].tolist() == [60, 51] and w["flip"].tolist() == [1, 0]
    out2 = pre.launch(torch.from_numpy(buf).data_ptr(), 2, torch.empty(2, 3, RES[1], RES[0]))
    assert torch.equal(out, out2)
    with pytest.raises(ValueError):
        pre.launch(torch.from_numpy(buf).data_ptr(), 2, torch.empty(2, 3, RES[1], RES[0] + 1))


# ---- chunks and order -------------------------------------------------------------------------------------------------------
def test_chunks_run_in_order_and_keep_the_output_order(fake):
    sizes = [(20, 10), (18, 9), (40, 20), (31, 12), (20, 10), (25, 11), (33, 17)]
    frames, P2 = _frames(sizes, seed=3), _p2(7, seed=2)
    model = StubModel()
    chunked = _detector(model, max_batch=3).detect(frames, P2)
    assert [s["calibs"].shape[0] for s in model.seen] == [3, 3, 1]
    assert np.concatenate([s["calibs"].numpy() for s in model.seen]).tolist() == P2.tolist()
    whole = _detector(max_batch=8).detect(frames, P2)
    single = [_detector().detect([f], P2[i:i + 1])[0] for i, f in enumerate(frames)]
    assert len(chunked) == 7 and any(len(r) for r in chunked)
    for a, b, c in zip(chunked, whole, single):
        assert a.dtype == np.float32 and a.shape[1] == 14
        assert np.array_equal(a, b) and np.array_equal(a, c)
    rows, count = _detector(max_batch=3).detect_device(frames, P2)
    assert rows.shape == (7, 50, 14) and count.dtype == torch.int32
    assert [int(c) for c in count] == [len(r) for r in chunked]


def test_rows_are_the_decode_of_the_heads(fake):
    """detect = extract_dets_from_outputs + decode_detections_device with the Detector's topk, threshold and mean sizes."""
    frames, P2 = _frames([(20, 10), (18, 9)]), _p2(2)
    mean = np.arange(9, dtype=np.float32).reshape(3, 3) / 7
    got = _detector(topk=20, threshold=0.1, cls_mean_size=mean).detect(frames, P2)
    for b, rows in enumerate(got):
        h = od.synthetic_heads(int(P2[b, 0, 3]), 1, 50)
        dets = od.extract_dets(h["logits"], h["boxes"], h["dim3"], h["depth"], h["angle"], 20)
        want = od.decode_dets(dets, np.array([[frames[b].shape[1], frames[b].shape[0]]], np.float32), P2[b:b + 1], mean, 0.1)[0]
        assert np.array_equal(rows, np.array(want, np.float64).astype(np.float32).reshape(-1, 14))


# ---- from_config ------------------------------------------------------------------------------------------------------------
def test_from_config(fake, monkeypatch, tmp_path):
    import monodetr_b200
    built = []

    def build(cfg, criterion_builder=None):
        built.append((cfg, criterion_builder(cfg) if criterion_builder else "default"))
        return StubModel(), None
    monkeypatch.setattr(monodetr_b200, "build_monodetr", build)
    src = StubModel()
    with torch.no_grad():
        src.w.copy_(torch.tensor([1.0, 2.0, 3.0]))
    ckpt = str(tmp_path / "ckpt.pth")
    torch.save({"epoch": 3, "model_state": src.state_dict(), "optimizer_state": None}, ckpt)
    cfg = {"model": {"num_classes": 3}, "tester": {"topk": 20, "threshold": 0.05}, "dataset": {"meanshape": False}}
    d = detect.Detector.from_config(cfg, ckpt, device="cpu", resolution=RES)
    assert built == [({"num_classes": 3}, None)]           # no criterion is built
    assert (d.topk, d.threshold) == (20, 0.05) and d.resolution == RES
    assert torch.equal(d.model.w, src.w) and not d.model.training
    assert not d.cls_mean_size.any() and d.cls_mean_size.shape == (3, 3)
    d = detect.Detector.from_config(dict(cfg, dataset={"meanshape": True}), ckpt, device="cpu", topk=7)
    assert d.topk == 7 and d.threshold == 0.05
    assert np.array_equal(d.cls_mean_size.numpy(), CLS_MEAN_SIZE.astype(np.float32))
    d = detect.Detector.from_config({"model": {}}, ckpt, device="cpu")
    assert (d.topk, d.threshold) == (50, 0.2)              # configs/monodetr.yaml's tester values


# ---- the command line -------------------------------------------------------------------------------------------------------
def _cli():
    spec = importlib.util.spec_from_file_location("detect_cli", os.path.join(os.path.dirname(__file__), "..", "tools", "detect.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_cli_arguments_and_names(tmp_path):
    cli = _cli()
    base = ["--config", "c.yaml", "--checkpoint", "k.pth", "--images", "im", "--calib", "cal", "--out", "o"]
    a = cli.parse_args(base)
    assert (a.config, a.checkpoint, a.images, a.calib, a.out, a.batch) == ("c.yaml", "k.pth", "im", "cal", "o", None)
    assert cli.parse_args(base + ["--batch", "4"]).batch == 4
    for bad in (base[:-2], base + ["--batch", "0"]):
        with pytest.raises(SystemExit):
            cli.parse_args(bad)
    assert cli.result_name("/x/000123.png") == "000123.txt" and cli.result_name("7.jpg") == "000007.txt"
    assert cli.result_name("/x/frame_a.png") == "frame_a.txt"
    d = tmp_path / "imgs"
    d.mkdir()
    for n in ("b.png", "a.JPG", "c.jpeg", "notes.txt"):
        (d / n).write_bytes(b"")
    assert [os.path.basename(p) for p in cli.image_paths(str(d))] == ["a.JPG", "b.png", "c.jpeg"]
    (tmp_path / "list.txt").write_text("imgs/b.png\n\n" + str(d / "a.JPG") + "\n")
    assert cli.image_paths(str(tmp_path / "list.txt")) == [str(d / "b.png"), str(d / "a.JPG")]
    assert cli.calib_paths(["/x/a.png", "/y/b.jpg"], str(d)) == [str(d / "a.txt"), str(d / "b.txt")]
    assert cli.calib_paths(["/x/a.png", "/y/b.jpg"], "one.txt") == ["one.txt", "one.txt"]
    (tmp_path / "empty").mkdir()
    with pytest.raises(ValueError):
        cli.image_paths(str(tmp_path / "empty"))


def test_cli_writes_one_result_file_per_image(tmp_path, monkeypatch):
    from PIL import Image
    import synthetic_kitti as sk
    cli = _cli()
    sizes = [(30, 12), (25, 10), (30, 12)]
    names = ["000004", "000011", "cam_x"]
    (tmp_path / "img").mkdir()
    (tmp_path / "calib").mkdir()
    for n, im, cam in zip(names, _frames(sizes, seed=9), (0, 1, 0)):
        Image.fromarray(im).save(tmp_path / "img" / (n + ".png"))
        (tmp_path / "calib" / (n + ".txt")).write_text(sk.calib_text(cam))
    (tmp_path / "cfg.yaml").write_text("model: {}\ntester: {topk: 10, threshold: 0.3}\ndataset: {batch_size: 2}\n")
    calls = []

    class StubDetector:
        @classmethod
        def from_config(cls, cfg, checkpoint, **kw):
            calls.append(("from_config", cfg, checkpoint, kw))
            return cls()

        def detect(self, frames, P2):
            calls.append(("detect", [f.shape for f in frames], P2.copy()))
            rng = np.random.default_rng(len(calls))
            return [np.concatenate([rng.integers(0, 3, (k, 1)), rng.normal(0, 5, (k, 13))], 1).astype(np.float32)
                    for k in range(len(frames))]

    monkeypatch.setattr(detect, "Detector", StubDetector)
    out = tmp_path / "out"
    cli.main(["--config", str(tmp_path / "cfg.yaml"), "--checkpoint", "ck.pth", "--images", str(tmp_path / "img"),
              "--calib", str(tmp_path / "calib"), "--out", str(out)])
    fc, det1, det2 = calls
    assert fc[1]["tester"] == {"topk": 10, "threshold": 0.3} and fc[2] == "ck.pth"
    assert fc[3] == {"max_batch": 2, "max_frame": (30, 12)}
    assert det1[1] == [(12, 30, 3), (10, 25, 3)] and det2[1] == [(12, 30, 3)]
    assert np.array_equal(np.concatenate([det1[2], det2[2]]), np.stack([sk.p2_of(c) for c in (0, 1, 0)]))
    assert sorted(os.listdir(out)) == ["000004.txt", "000011.txt", "cam_x.txt"]
    rng = np.random.default_rng(2)
    first = [np.concatenate([rng.integers(0, 3, (k, 1)), rng.normal(0, 5, (k, 13))], 1).astype(np.float32) for k in range(2)]
    assert (out / "000004.txt").read_text() == "" and (out / "cam_x.txt").read_text() == ""
    assert (out / "000011.txt").read_text() == kitti_eval.result_file_text(first[1].tolist(), CLASS_NAMES)
    assert (out / "000011.txt").read_text().startswith(CLASS_NAMES[int(first[1][0, 0])] + " 0.0 0 ")
