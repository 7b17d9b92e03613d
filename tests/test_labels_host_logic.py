"""CPU: the host side of monodetr_b200.labels -- label and calib parsing against the reference's own parse, the augmentation
sampler's draws and stream state, record packing, the option checks -- with a stand-in for mdb_kitti_encode_targets that computes
with oracle/labels.py on host memory (tests/golden/labels.npz, tools/gen_golden_labels.py)."""
import ctypes
import os

import numpy as np
import pytest
import torch

import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import FakeLib
from monodetr_b200 import _lib
from monodetr_b200 import labels as lb
from oracle import labels as ol

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "labels.npz"))
VARIANTS = ["shipped", "all3", "clip2d", "inverse", "none", "meanshape", "val", "e2e"]
SHIPPED = {"aug_pd": True, "aug_crop": True, "random_flip": 0.5, "random_crop": 0.5, "scale": 0.05, "shift": 0.05,
           "writelist": ["Car"], "clip_2d": False, "depth_scale": "normal", "meanshape": False, "class_merging": False,
           "use_dontcare": False}


def _cfg(name):
    import json
    return dict(SHIPPED, **json.loads(str(GOLD[f"{name}.cfg"])))


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(int(ptr)))


class LabelsFakeLib(FakeLib):
    def mdb_kitti_encode_targets(self, off, objs, P2, n_bank, images, B, cfg, *outs):
        outs = outs[:-1]                                                         # (the stream)
        offsets = _arr(off, ctypes.c_int64, n_bank + 1)
        recs = _arr(objs, ctypes.c_double, int(offsets[-1]) * ol.WIDTH).reshape(-1, ol.WIDTH)
        P2s = _arr(P2, ctypes.c_float, 12 * n_bank).reshape(n_bank, 3, 4)
        im = _arr(images, ctypes.c_uint8, 72 * B).view(lb._IMAGE_DTYPE)
        c = _arr(cfg, ctypes.c_uint8, 96).view(lb._CONFIG_DTYPE)[0]
        self.encode_calls.append(dict(images=im.copy(), cfg=c.copy()))
        S = int(c["max_objs"])
        want = ol.encode_batch(offsets, recs, P2s, im["bank_index"], np.stack([im["img_w"], im["img_h"]], 1), im["flip"],
                               im["crop_scale"], im["trans"].reshape(B, 2, 3), class_mask=int(c["class_mask"]),
                               clip_2d=bool(c["clip_2d"]), depth_scale=ol.DEPTH_SCALES[int(c["depth_scale"])],
                               mean_size=c["mean_size"].reshape(3, 3), resolution=(int(c["res_w"]), int(c["res_h"])), max_objs=S)
        for k, ptr in zip(ol.KEYS, outs):
            w = want[k]
            dst = _arr(ptr, np.ctypeslib.as_ctypes_type(np.uint8 if w.dtype == bool else w.dtype), w.size).reshape(w.shape)
            dst[:] = w
        return 0


@pytest.fixture
def fake(monkeypatch):
    fake_device_lib.install(monkeypatch)
    lib = LabelsFakeLib(1)
    lib.encode_calls = []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(lb, "_require_cuda", lambda device: None)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    return lib


def _gold_bank(device="cpu"):
    offsets, recs, P2s = ol.gold_bank(GOLD)
    return lb.LabelBank(offsets, recs, P2s, GOLD["img_ids"], device=device)


def _gold_records(name):
    n = len(GOLD[f"{name}.seeds"])
    return [lb.AugRecord(tuple(GOLD["sizes"][i]), bool(GOLD[f"{name}.flip"][i]), float(GOLD[f"{name}.crop_scale"][i]),
                         GOLD[f"{name}.center"][i], GOLD[f"{name}.trans"][i], GOLD[f"{name}.trans_inv"][i]) for i in range(n)]


def _write_split(d, n=len(GOLD["sizes"])):
    for sub in ("ImageSets", "training/calib", "training/label_2"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    open(os.path.join(d, "ImageSets", "train.txt"), "w").write("".join("%06d\n" % i for i in range(n)))
    for i in range(n):
        open(os.path.join(d, "training", "label_2", "%06d.txt" % i), "w").write(str(GOLD[f"label.{i}"]))
        open(os.path.join(d, "training", "calib", "%06d.txt" % i), "w").write(str(GOLD[f"calib.{i}"]))


def test_layouts_match_the_header_and_the_oracle():
    assert lb._IMAGE_DTYPE.itemsize == 72 and lb._CONFIG_DTYPE.itemsize == 96
    assert [lb._IMAGE_DTYPE.fields[n][1] for n in ("trans", "crop_scale", "bank_index", "img_w", "img_h", "flip")] == [0, 48, 56, 60,
                                                                                                                    64, 68]
    assert [lb._CONFIG_DTYPE.fields[n][1] for n in ("class_mask", "clip_2d", "depth_scale", "res_w", "res_h", "max_objs")] == \
        [72, 76, 80, 84, 88, 92]
    assert (lb.RECORD_WIDTH, lb.CLS, lb.TRUNC, lb.X1, lb.H, lb.PX, lb.RY) == (ol.WIDTH, ol.CLS, ol.TRUNC, ol.X1, ol.H, ol.PX, ol.RY)
    assert lb.CLASS_NAMES == ol.CLASS_NAMES and lb.TARGET_KEYS == ol.KEYS and np.array_equal(lb.CLS_MEAN_SIZE, ol.CLS_MEAN_SIZE)
    assert list(lb.DEPTH_SCALES) == list(ol.DEPTH_SCALES)


def test_bank_parse_matches_the_reference_objects(tmp_path):
    _write_split(str(tmp_path))
    bank = lb.LabelBank.from_kitti(str(tmp_path), "train", device="cpu")
    offsets, recs, P2s = ol.gold_bank(GOLD)
    assert bank.img_ids == list(GOLD["img_ids"]) and bank.names == [str(c) for c in GOLD["parsed.cls"]]
    np.testing.assert_array_equal(bank.host_offsets, offsets)
    np.testing.assert_array_equal(bank.host_P2, P2s)
    assert bank.host_P2.dtype == GOLD["parsed.P2"].dtype == np.float32
    np.testing.assert_array_equal(bank.host_objects[:, :ol.RY + 1], recs[:, :ol.RY + 1])      # every field, bit for bit
    np.testing.assert_array_equal(bank.objects.numpy(), bank.host_objects)
    assert max(np.diff(offsets)) > lb.MAX_OBJS                 # the > 50-line file keeps every line


@pytest.mark.parametrize("line", ["Car 0.00 0 -1.58 587.01 173.33 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70",
                                  "Car 0.00 0 -1.58 587.01 173.33 614.12 abc 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59",
                                  "Car  0.00 0 -1.58 587.01 173.33 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59", ""])
def test_malformed_label_line_names_file_and_line(tmp_path, line):
    _write_split(str(tmp_path), 2)
    path = os.path.join(str(tmp_path), "training", "label_2", "000001.txt")
    open(path, "a").write(line + "\n")
    n = str(GOLD["label.1"]).count("\n") + 1
    with pytest.raises(ValueError, match=f"000001.txt:{n}:"):
        lb.LabelBank.from_kitti(str(tmp_path), "train", device="cpu")


def test_malformed_calib_raises(tmp_path):
    _write_split(str(tmp_path), 1)
    open(os.path.join(str(tmp_path), "training", "calib", "000000.txt"), "w").write("P0: 1\nP1: 1\nP2: 1 2 3\n")
    with pytest.raises(ValueError, match="000000.txt:3"):
        lb.LabelBank.from_kitti(str(tmp_path), "train", device="cpu")


@pytest.mark.parametrize("name", VARIANTS)
def test_sampler_makes_the_reference_draws(name):
    cfg, split = _cfg(name), str(GOLD[f"{name}.split"])
    res = tuple(int(v) for v in GOLD[f"{name}.resolution"])
    s = lb.AugmentationSampler.from_config(cfg, split, res)
    for i, seed in enumerate(GOLD[f"{name}.seeds"]):
        np.random.seed(int(seed))
        r = s.sample(GOLD["sizes"][i])
        _, keys, pos, has_gauss, gauss = np.random.get_state()
        assert np.array_equal(keys, GOLD[f"{name}.state_keys"][i]) and pos == GOLD[f"{name}.state_pos"][i]
        assert has_gauss == GOLD[f"{name}.state_gauss"][i][0] and gauss == GOLD[f"{name}.state_gauss"][i][1]
        assert r.flip == bool(GOLD[f"{name}.flip"][i]) and r.crop_scale == GOLD[f"{name}.crop_scale"][i]
        np.testing.assert_array_equal(r.center, GOLD[f"{name}.center"][i])
        # get_affine_transform solves cv2.getAffineTransform's 3-point system with numpy (tests/test_oracle_preprocess.py)
        np.testing.assert_allclose(r.trans, GOLD[f"{name}.trans"][i], rtol=0, atol=1e-9)
        np.testing.assert_allclose(r.trans_inv, GOLD[f"{name}.trans_inv"][i], rtol=0, atol=1e-9)
        assert (r.distort is not None) == (cfg["aug_pd"] and split == "train")


def test_sampler_makes_no_draw_on_val():
    s = lb.AugmentationSampler.from_config(SHIPPED, "val")
    np.random.seed(3)
    before = np.random.get_state()[1].copy(), np.random.get_state()[2]
    r = s.sample((1242, 375))
    assert np.array_equal(np.random.get_state()[1], before[0]) and np.random.get_state()[2] == before[1]
    assert not r.flip and r.crop_scale == 1 and r.distort is None


@pytest.mark.parametrize("name", ["shipped", "clip2d", "inverse", "meanshape"])
def test_encoder_packs_records_and_config(fake, name):
    bank = _gold_bank()
    recs = _gold_records(name)
    cfg = _cfg(name)
    enc = lb.TargetEncoder(cfg["writelist"], cfg["clip_2d"], cfg["depth_scale"], cfg["meanshape"],
                           tuple(int(v) for v in GOLD[f"{name}.resolution"]), device="cpu")
    idx = list(range(len(recs)))[::-1]
    n0 = _lib.launch_count()
    t = enc(bank, idx, recs[::-1])
    assert _lib.launch_count() - n0 == 1
    (call,) = fake.encode_calls
    np.testing.assert_array_equal(call["images"]["bank_index"], idx)
    assert call["cfg"]["max_objs"] == 50 and call["cfg"]["depth_scale"] == lb.DEPTH_SCALES[cfg["depth_scale"]]
    want = {k: GOLD[f"{name}.{k}"][::-1] for k in ol.KEYS}
    ol.assert_targets_match({k: v.numpy() for k, v in t.items()}, want, name)
    assert t["mask_2d"].dtype == torch.bool and t["labels"].dtype == torch.int8 and t["heading_bin"].dtype == torch.int64


def test_batch_builder_composes_both_halves(fake, monkeypatch):
    """The images go through ImageBatchPreprocessor with the records' trans_inv / flip / distort; info as default_collate."""
    seen = {}

    def fake_pre(self, images, trans_inv, flip=None, distort=None):
        seen.update(trans_inv=trans_inv, flip=flip, distort=distort)
        return torch.zeros(len(images), 3, 96, 320)

    from monodetr_b200 import preprocess as pp
    monkeypatch.setattr(pp.ImageBatchPreprocessor, "__call__", fake_pre)
    bank = _gold_bank()
    builder = lb.KittiBatchBuilder(SHIPPED, "train", bank, resolution=(320, 96), device="cpu")
    imgs = [torch.zeros(int(h), int(w), 3, dtype=torch.uint8) for w, h in GOLD["sizes"][:3]]
    np.random.seed(4)
    recs = [builder.sampler.sample((im.shape[1], im.shape[0])) for im in imgs]
    inputs, P2, targets, info = builder(imgs, [2, 0, 1], recs)
    np.testing.assert_array_equal(seen["trans_inv"], np.stack([r.trans_inv for r in recs]))
    assert seen["flip"] == [r.flip for r in recs] and seen["distort"] == [r.distort for r in recs]
    np.testing.assert_array_equal(P2.numpy(), GOLD["parsed.P2"][[2, 0, 1]])
    assert info["img_id"].tolist() == [2, 0, 1] and info["img_id"].dtype == torch.int64
    np.testing.assert_array_equal(info["img_size"].numpy(), GOLD["sizes"][:3])
    np.testing.assert_array_equal(info["bbox_downsample_ratio"].numpy(), GOLD["sizes"][:3] / np.array([10, 3]))
    np.testing.assert_array_equal(targets["img_size"].numpy(), GOLD["sizes"][:3])
    with pytest.raises(ValueError, match="drawn for an image"):
        builder(imgs, [2, 0, 1], recs[::-1])


@pytest.mark.parametrize("opt", ["aug_calib", "class_merging", "use_dontcare"])
def test_unsupported_options_raise(opt):
    with pytest.raises(NotImplementedError, match=opt):
        lb.KittiBatchBuilder(dict(SHIPPED, **{opt: True}), "train", None, device="cpu")


def test_unsupported_splits_and_classes_raise(tmp_path):
    with pytest.raises(NotImplementedError):
        lb.KittiBatchBuilder(SHIPPED, "test", None, device="cpu")
    with pytest.raises(NotImplementedError):
        lb.LabelBank.from_kitti(str(tmp_path), "test", device="cpu")
    with pytest.raises(NotImplementedError, match="Van"):
        lb.TargetEncoder(["Car", "Van"], device="cpu")
    with pytest.raises(ValueError):
        lb.TargetEncoder(["Car"], depth_scale="log", device="cpu")


@pytest.mark.parametrize("case", ["index", "negative", "empty", "nan_scale", "zero_scale", "count", "trans"])
def test_out_of_range_inputs_raise_before_launch(fake, case):
    bank = _gold_bank()
    recs = _gold_records("shipped")[:3]
    idx = [0, 1, 2]
    if case == "index":
        idx = [0, 1, len(bank)]
    elif case == "negative":
        idx = [0, -1, 2]
    elif case == "empty":
        idx, recs = [], []
    elif case == "nan_scale":
        recs[1] = recs[1]._replace(crop_scale=float("nan"))
    elif case == "zero_scale":
        recs[1] = recs[1]._replace(crop_scale=0.0)
    elif case == "count":
        recs = recs[:2]
    else:
        recs[0] = recs[0]._replace(trans=np.full((2, 3), np.inf))
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        lb.TargetEncoder(device="cpu")(bank, idx, recs)
    assert _lib.launch_count() == n0 and not fake.encode_calls


def test_bank_rejects_inconsistent_arrays():
    with pytest.raises(ValueError):
        lb.LabelBank([0, 3], np.zeros((2, lb.RECORD_WIDTH)), np.zeros((1, 3, 4)), [0], device="cpu")
    with pytest.raises(ValueError):
        lb.LabelBank.from_arrays([1], np.full((1, lb.RECORD_WIDTH), np.nan), np.zeros((1, 3, 4)), device="cpu")
    b = lb.LabelBank.from_arrays([2, 0], np.full((2, lb.RECORD_WIDTH), 0.1), np.zeros((2, 3, 4)), device="cpu")
    assert b.host_objects[0, lb.X1] == np.float32(0.1) and b.host_objects[0, lb.H] == 0.1 and len(b) == 2
