"""Host logic of monodetr_b200.dataset (no GPU): the light KITTI_Dataset under a real torch DataLoader makes the reference
loader's image order and per-item draws (tests/golden/loader.npz, tools/gen_golden_loader.py) for 0 and 2 workers over two
epochs; the datasets pickle and hold no CUDA tensor; the DeviceLoader wrapper; the errors build_dataloader raises before it
decodes anything."""
import json
import os
import pickle
import types

import numpy as np
import pytest
import torch
from PIL import Image

import synthetic_kitti as sk
from monodetr_b200 import dataset as ds

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "loader.npz"))
CFG = json.loads(str(GOLD["cfg"]))
RUNS = {"train_w0": ("train", 0, 2), "train_w2": ("train", 2, 2), "val": ("val", 0, 1), "test": ("test", 0, 1)}


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    sk.write_tree(root)
    return root


def _cfg(root, **over):
    return dict(CFG, root_dir=root, **over)


def _draw_row(rec):
    pd = rec.distort
    pd = [np.nan] * 4 + [-1, -1] if pd is None else list(pd)
    return np.concatenate([[float(rec.flip), rec.crop_scale], rec.center, np.asarray(rec.trans_inv).reshape(6), pd])


@pytest.mark.parametrize("run", list(RUNS))
def test_light_loader_makes_the_reference_order_and_draws(tree, run):
    split, workers, epochs = RUNS[run]
    sk.set_random_seed(444)
    dataset = ds.KITTI_Dataset(split, _cfg(tree))
    loader = ds.kitti_loader(dataset, CFG["batch_size"], split == "train", workers)
    for epoch in range(epochs):
        if split == "train":
            np.random.seed(np.random.get_state()[1][0] + epoch)          # Trainer.train, before each epoch
        p = f"{run}.e{epoch}"
        ids, draws, bounds = [], [], [0]
        for batch in loader:
            assert isinstance(batch, list) and all(isinstance(k, int) for k, _ in batch)
            ids += [int(dataset.idx_list[k]) for k, _ in batch]
            draws += [_draw_row(r) for _, r in batch]
            bounds.append(bounds[-1] + len(batch))
        assert ids == GOLD[p + ".ids"].tolist(), p
        assert bounds == GOLD[p + ".bounds"].tolist(), p
        # flip, crop_scale, center, trans_inv (cv2's bits) and the photometric draws
        np.testing.assert_array_equal(np.array(draws), GOLD[p + ".draws"], err_msg=p)


def test_get_affine_transform_is_cv2_bit_for_bit():
    """The reference's get_affine_transform (cv2.getAffineTransform) in every fixture that stored its matrices."""
    from monodetr_b200.preprocess import get_affine_transform
    pre = np.load(os.path.join(os.path.dirname(__file__), "golden", "preprocess.npz"))
    for i in range(len(pre["sizes"])):
        trans, trans_inv = get_affine_transform(pre[f"{i}.center"], pre[f"{i}.crop_size"], 0, pre["resolution"], inv=1)
        assert np.array_equal(trans, pre[f"{i}.trans"]) and np.array_equal(trans_inv, pre[f"{i}.trans_inv"]), i
    lab = np.load(os.path.join(os.path.dirname(__file__), "golden", "labels.npz"))
    n = 0
    for v in ("shipped", "all3", "clip2d", "inverse", "none", "meanshape", "val", "e2e"):
        for i in range(len(lab[f"{v}.seeds"])):
            size = lab["sizes"][i]
            crop = size * lab[f"{v}.crop_scale"][i] if lab[f"{v}.crop_scale"][i] != 1 else size
            trans, trans_inv = get_affine_transform(lab[f"{v}.center"][i], crop, 0, lab[f"{v}.resolution"], inv=1)
            assert np.array_equal(trans, lab[f"{v}.trans"][i]) and np.array_equal(trans_inv, lab[f"{v}.trans_inv"][i]), (v, i)
            n += 1
    assert n > 40


def _tensors(obj, seen=None):
    seen = set() if seen is None else seen
    if id(obj) in seen or isinstance(obj, types.ModuleType):
        return []
    seen.add(id(obj))
    if torch.is_tensor(obj):
        return [obj]
    if isinstance(obj, dict):
        return [t for v in obj.values() for t in _tensors(v, seen)]
    if isinstance(obj, (list, tuple)):
        return [t for v in obj for t in _tensors(v, seen)]
    if hasattr(obj, "__dict__"):
        return _tensors(vars(obj), seen)
    return []


@pytest.mark.parametrize("split", ["train", "val", "trainval", "test"])
def test_dataset_pickles_and_holds_no_tensor(tree, split):
    dataset = ds.KITTI_Dataset(split, _cfg(tree))
    dataset[0]                                                          # the lazily built sampler is not pickled
    clone = pickle.loads(pickle.dumps(dataset))
    assert not _tensors(dataset) and not _tensors(clone)
    np.random.seed(5)
    a = dataset[1]
    np.random.seed(5)
    b = clone[1]
    assert a[0] == b[0] == 1 and a[1].flip == b[1].flip and np.array_equal(a[1].trans_inv, b[1].trans_inv)


def test_dataset_attributes(tree):
    splits = {s: [int(x) for x in open(os.path.join(tree, "ImageSets", s + ".txt"))] for s in ("train", "val", "test")}
    for split, n in (("train", 14), ("val", 6), ("test", 6)):
        d = ds.KITTI_Dataset(split, _cfg(tree))
        assert len(d) == n and d.split == split and d.idx_list == ["%06d" % i for i in splits[split]]
        data = os.path.join(tree, "testing" if split == "test" else "training")
        assert d.label_dir == os.path.join(data, "label_2") and d.calib_dir == os.path.join(data, "calib")
        assert d.writelist == ["Car"] and d.class_name == ["Pedestrian", "Car", "Cyclist"]
        assert d.cls_mean_size.dtype == np.float32 and not d.cls_mean_size.any() and d.cls_mean_size.shape == (3, 3)
        assert d.resolution.tolist() == [1280, 384]
        for k, i in enumerate(splits[split]):
            with Image.open(os.path.join(data, "image_2", "%06d.png" % i)) as im:
                assert tuple(d.img_sizes[k]) == im.size
    assert ds.KITTI_Dataset("train", _cfg(tree, meanshape=True)).cls_mean_size[1, 2] == 3.88311640418
    np.random.seed(1)
    before = np.random.get_state()[1].copy()
    item, rec = ds.KITTI_Dataset("val", _cfg(tree))[2]
    assert item == 2 and np.array_equal(np.random.get_state()[1], before)           # val: no draw
    assert not rec.flip and rec.crop_scale == 1 and rec.distort is None


class _Bank:
    def views(self, idx):
        return [f"view{k}" for k in idx]


def test_device_loader_wraps_each_batch(tree):
    calls = []

    def builder(images, idx, records):
        calls.append((images, idx, records))
        return len(calls)

    dataset = ds.KITTI_Dataset("val", _cfg(tree))
    loader = ds.DeviceLoader(ds.kitti_loader(dataset, 4, False, 0), _Bank(), builder)
    assert len(loader) == 2 and loader.dataset is dataset and loader.batch_size == 4
    assert list(loader) == [1, 2]
    assert [c[1] for c in calls] == [[0, 1, 2, 3], [4, 5]]
    assert calls[1][0] == ["view4", "view5"] and [r.img_size for r in calls[1][2]] == [tuple(s) for s in dataset.img_sizes[4:]]


def test_build_dataloader_errors_come_before_decoding(tmp_path):
    missing = str(tmp_path / "nothing")
    with pytest.raises(NotImplementedError, match="Waymo dataset is not supported"):
        ds.build_dataloader(_cfg(missing, type="Waymo"))
    for opt in ("aug_calib", "class_merging", "use_dontcare"):
        with pytest.raises(NotImplementedError, match=opt):
            ds.build_dataloader(_cfg(missing, **{opt: True}))
    with pytest.raises(ValueError, match="train_split"):
        ds.build_dataloader(_cfg(missing, train_split="training"))


@pytest.mark.parametrize("mode", ["RGBA", "L", "I;16"])
def test_non_rgb_image_raises_before_the_device(tmp_path, mode):
    """On a machine without CUDA any device allocation would fail with another error: the ValueError comes first."""
    root = str(tmp_path)
    sk.write_tree(root, n_train=3, n_val=1, n_test=1, objects=(1, 3))
    bad = int(open(os.path.join(root, "ImageSets", "train.txt")).readlines()[1])
    path = os.path.join(root, "training", "image_2", "%06d.png" % bad)
    Image.open(path).convert(mode).save(path)
    with pytest.raises(ValueError, match="%06d.png" % bad):
        ds.ImageBank(root, "train", device="cuda")
    with pytest.raises(ValueError, match="%06d.png" % bad):
        ds.build_dataloader(_cfg(root), workers=0)
    with pytest.raises(ValueError, match="%06d.png" % bad):
        ds.KITTI_Dataset("train", _cfg(root))
