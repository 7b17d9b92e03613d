"""Device photometric distortion (mdb_photometric_distort_u8 through monodetr_b200.preprocess), bit-exact against the reference's
outputs (tests/golden/photometric.npz, tools/gen_golden_photometric.py) and the numpy oracle (oracle/photometric.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import photometric as ph
from oracle import preprocess as op

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "photometric.npz"))
KITTI_SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376)]


def _fixture_case(i):
    img = op.synthetic_images(int(GOLD["img_seed"]) + i, [tuple(int(v) for v in GOLD["sizes"][i])])[0]
    r = GOLD[f"{i}.record"]
    return img, ph.Params(*r[:4], int(r[4]), int(r[5]))


def test_every_fixture_case_bit_exact():
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    n = len(GOLD["sizes"])
    imgs, recs = zip(*[_fixture_case(i) for i in range(n)])
    outs = ImageBatchPreprocessor().distort([torch.from_numpy(im) for im in imgs], list(recs))
    for i, o in enumerate(outs):
        assert o.is_cuda and o.shape == imgs[i].shape
        assert np.array_equal(o.cpu().numpy(), GOLD[f"{i}.u8"]), i


def _kitti_batch():
    from monodetr_b200.preprocess import PhotometricDistort, get_affine_transform
    imgs = op.synthetic_images(21, KITTI_SIZES)
    np.random.seed(22)
    pd = PhotometricDistort()
    recs = [pd.sample() for _ in KITTI_SIZES]
    recs[1] = recs[1]._replace(contrast=1.45, saturation=1.5, contrast_last=1, perm=5)   # values far outside [0, 256)
    rng = np.random.default_rng(23)
    res = np.array([1280, 384])
    tinv, flip = [], []
    for (W, H) in KITTI_SIZES:
        size = np.array([W, H], np.float64)
        center = size / 2 + size * np.clip(rng.standard_normal(2) * 0.1, -0.2, 0.2)
        tinv.append(get_affine_transform(center, size * np.clip(rng.standard_normal() * 0.4 + 1, 0.6, 1.4), 0, res, inv=1)[1])
        flip.append(bool(rng.integers(0, 2)))
    flip[0], flip[1] = True, False
    return imgs, recs, np.stack(tinv), flip


def test_kitti_sized_ragged_batch_against_oracle():
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    imgs, recs, tinv, flip = _kitti_batch()
    srcs = [torch.from_numpy(im).cuda() if i % 2 else torch.from_numpy(im.copy()) for i, im in enumerate(imgs)]
    before = [s.clone() for s in srcs]
    pre = ImageBatchPreprocessor(resolution=(1280, 384))
    alone = pre.distort(srcs, recs)
    full = pre(srcs, tinv, flip, distort=recs).cpu().numpy()
    torch.cuda.synchronize()
    n_wrap = 0
    for i, im in enumerate(imgs):
        want = ph.distort_float(im, ph.Params(*recs[i]))
        n_wrap += int(((want < 0) | (want >= 256)).sum())
        want = ph.to_u8(want)
        got = alone[i].cpu().numpy()
        assert np.array_equal(got, want), (i, (got != want).sum())
        full_want = op.preprocess(want, tinv[i].reshape(-1), (1280, 384), flip[i])
        assert np.array_equal(full[i], full_want), i
        assert torch.equal(srcs[i], before[i])                     # the caller's images are untouched
    assert n_wrap > 0


def test_without_distort_unchanged():
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    from monodetr_b200 import _lib
    imgs, recs, tinv, flip = _kitti_batch()
    srcs = [torch.from_numpy(im) for im in imgs]
    pre = ImageBatchPreprocessor(resolution=(1280, 384))
    n0 = _lib.launch_count()
    out = pre(srcs, tinv, flip).cpu().numpy()
    assert _lib.launch_count() - n0 == 1
    pre(srcs, tinv, flip, distort=recs)
    assert _lib.launch_count() - n0 == 3
    for i, im in enumerate(imgs):
        assert np.array_equal(out[i], op.preprocess(im, tinv[i].reshape(-1), (1280, 384), flip[i])), i


def test_getitem_end_to_end_fixture():
    from monodetr_b200.preprocess import ImageBatchPreprocessor, PhotometricDistort, get_affine_transform
    src = op.synthetic_images(int(GOLD["e2e.img_seed"]), [tuple(int(v) for v in GOLD["e2e.size"])])[0]
    res = tuple(int(v) for v in GOLD["e2e.res"])
    K = len(GOLD["e2e.seeds"])
    recs, flips, tinvs = [], [], []
    for k in range(K):
        rec, flip, tinv = ph.replay_getitem(GOLD, k, PhotometricDistort().sample, get_affine_transform)
        assert ph.state_matches(GOLD, f"e2e.{k}.")
        recs.append(rec), flips.append(flip), tinvs.append(tinv)
    out = ImageBatchPreprocessor(resolution=res)([torch.from_numpy(src)] * K, np.stack(tinvs), flips, distort=recs).cpu().numpy()
    for k in range(K):
        assert np.array_equal(out[k], op.normalize(GOLD[f"e2e.{k}.u8"])), k


def test_same_bits_in_reproducible_mode():
    import monodetr_b200
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    imgs, recs, tinv, flip = _kitti_batch()
    srcs = [torch.from_numpy(im).cuda() for im in imgs]
    pre = ImageBatchPreprocessor(resolution=(1280, 384))
    a = pre(srcs, tinv, flip, distort=recs)
    prev = monodetr_b200.set_deterministic(True)
    try:
        b = pre(srcs, tinv, flip, distort=recs)
        c = pre.distort(srcs, recs)
    finally:
        monodetr_b200.set_deterministic(prev)
    assert torch.equal(a, b)
    for i, im in enumerate(imgs):
        assert np.array_equal(c[i].cpu().numpy(), ph.distort(im, ph.Params(*recs[i])))


def test_errors():
    from monodetr_b200 import _lib
    from monodetr_b200.preprocess import ImageBatchPreprocessor
    pre = ImageBatchPreprocessor(resolution=(64, 32))
    img = [torch.zeros(8, 8, 3, dtype=torch.uint8)]
    for bad in [(0.0, 1.0, 1.0, 0.0, 0, 6), (0.0, 1.0, 1.0, 0.0, 3, 0), (float("nan"), 1.0, 1.0, 0.0, 0, 0)]:
        with pytest.raises(ValueError):
            pre(img, np.eye(2, 3)[None], None, distort=[bad])
        with pytest.raises(ValueError):
            pre.distort(img, [bad])
    with pytest.raises(ValueError):
        pre(img, np.eye(2, 3)[None], None, distort=[])
    with pytest.raises(RuntimeError):
        ImageBatchPreprocessor(device="cpu").distort(img, [(0.0, 1.0, 1.0, 0.0, 0, 0)])
    meta = torch.zeros(64, dtype=torch.int64, device="cuda")
    p = meta.data_ptr()
    with pytest.raises(RuntimeError, match="mdb_photometric_distort_u8"):          # null array -> MDB_EINVAL
        _lib.call("mdb_photometric_distort_u8", p, p, p, None, p, p, 1)
    for B in (0, -1, 65536):                                                      # batch size outside 1..65535 -> MDB_EINVAL
        with pytest.raises(RuntimeError, match="mdb_photometric_distort_u8"):
            _lib.call("mdb_photometric_distort_u8", p, p, p, p, p, p, B)
