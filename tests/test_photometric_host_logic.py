"""CPU: the host side of ImageBatchPreprocessor(..., distort=...) -- record validation and packing, the one metadata upload, the
distorted-image scratch buffer the warp reads, launch counts -- driven through stand-ins for mdb_photometric_distort_u8 and
mdb_warp_affine_normalize_u8 that compute with oracle/photometric.py and oracle/preprocess.py on host memory."""
import ctypes

import numpy as np
import pytest
import torch

import fake_device_lib          # tests/fake_device_lib.py (pytest puts this directory on sys.path)
from fake_device_lib import FakeLib
from monodetr_b200 import _lib
from monodetr_b200 import preprocess as pp
from oracle import photometric as ph
from oracle import preprocess as op


def _arr(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(int(ptr)))


def _image(ptr, W, H, pitch):
    raw = _arr(ptr, ctypes.c_uint8, (H - 1) * pitch + 3 * W)
    return np.lib.stride_tricks.as_strided(raw, (H, W, 3), (pitch, 3, 1))


class PhotometricFakeLib(FakeLib):
    def mdb_photometric_distort_u8(self, src, wh, pitch, params, dst, dpitch, B, stream):
        s, d = _arr(src, ctypes.c_int64, B), _arr(dst, ctypes.c_int64, B)
        p, dp = _arr(pitch, ctypes.c_int64, B), _arr(dpitch, ctypes.c_int64, B)
        sizes = _arr(wh, ctypes.c_int32, 2 * B).reshape(B, 2)
        recs = _arr(params, ctypes.c_uint8, 24 * B).view(pp._RECORD_DTYPE)
        self.distort_calls.append(dict(src=s.copy(), dst=d.copy(), pitch=p.copy(), dpitch=dp.copy(), wh=sizes.copy(), recs=recs.copy()))
        for b in range(B):
            W, H = (int(v) for v in sizes[b])
            r = recs[b]
            out = ph.distort(_image(s[b], W, H, p[b]), ph.Params(*(float(r[k]) for k in range(4)), int(r[4]), int(r[5])))
            _image(d[b], W, H, dp[b])[:] = out
        return 0

    def mdb_warp_affine_normalize_u8(self, src, wh, pitch, trans_inv, flip, B, W, H, mean3, std3, out, stream):
        s, p = _arr(src, ctypes.c_int64, B), _arr(pitch, ctypes.c_int64, B)
        sizes = _arr(wh, ctypes.c_int32, 2 * B).reshape(B, 2)
        tinv = _arr(trans_inv, ctypes.c_double, 6 * B).reshape(B, 6)
        fl = _arr(flip, ctypes.c_uint8, B) if flip else np.zeros(B, np.uint8)
        self.warp_calls.append(dict(src=s.copy(), pitch=p.copy()))
        o = fake_device_lib.f32(out, B, 3, H, W)
        for b in range(B):
            img = _image(s[b], int(sizes[b, 0]), int(sizes[b, 1]), p[b]).copy()
            o[b].copy_(torch.from_numpy(op.preprocess(img, tinv[b], (W, H), bool(fl[b]))))
        return 0


@pytest.fixture
def fake(monkeypatch):
    fake_device_lib.install(monkeypatch)
    lib = PhotometricFakeLib(1)
    lib.distort_calls, lib.warp_calls = [], []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(pp, "_require_cuda", lambda device: None)
    monkeypatch.setattr(torch.Tensor, "pin_memory", lambda self: self)
    return lib


SIZES = [(21, 9), (16, 7), (13, 11)]


def _batch(seed=3):
    imgs = op.synthetic_images(seed, SIZES)
    tinv = np.stack([pp.get_affine_transform(np.array([W, H]) / 2, np.array([W, H], np.float64), 0, np.array([24, 10]), inv=1)[1]
                     for W, H in SIZES])
    np.random.seed(7)
    recs = [pp.PhotometricDistort().sample() for _ in SIZES]
    recs[0] = recs[0]._replace(contrast=1.3, saturation=1.4, perm=3)      # drives values outside [0, 256)
    return imgs, tinv, recs


def test_records_are_packed_into_the_metadata_and_the_warp_reads_the_distorted_images(fake):
    imgs, tinv, recs = _batch()
    srcs = [torch.from_numpy(im.copy()) for im in imgs]
    pre = pp.ImageBatchPreprocessor(resolution=(24, 10), device="cpu")
    out = pre(srcs, tinv, [False, True, False], distort=recs)
    (d,) = fake.distort_calls
    np.testing.assert_array_equal(d["src"], [t.data_ptr() for t in srcs])
    np.testing.assert_array_equal(d["wh"], SIZES)
    np.testing.assert_array_equal(d["pitch"], [3 * W for W, _ in SIZES])
    np.testing.assert_array_equal(d["dpitch"], [3 * W for W, _ in SIZES])
    # one flat scratch buffer, images back to back
    np.testing.assert_array_equal(np.diff(d["dst"]), [3 * W * H for W, H in SIZES[:-1]])
    for b, r in enumerate(recs):
        got = d["recs"][b]
        assert tuple(got)[:4] == tuple(np.float32(v) for v in r[:4]) and (got[4], got[5]) == (r.contrast_last, r.perm)
    (w,) = fake.warp_calls
    np.testing.assert_array_equal(w["src"], d["dst"])
    np.testing.assert_array_equal(w["pitch"], d["dpitch"])
    for b, (im, r) in enumerate(zip(imgs, recs)):
        want = op.preprocess(ph.distort(im, ph.Params(*r)), tinv[b].reshape(-1), (24, 10), b == 1)
        assert np.array_equal(out[b].numpy(), want), b


def test_launch_counts_and_unchanged_inputs(fake):
    imgs, tinv, recs = _batch()
    srcs = [torch.from_numpy(im.copy()) for im in imgs]
    pre = pp.ImageBatchPreprocessor(resolution=(24, 10), device="cpu")
    n0 = _lib.launch_count()
    with_pd = pre(srcs, tinv, None, distort=recs)
    assert _lib.launch_count() - n0 == 2
    n0 = _lib.launch_count()
    without = pre(srcs, tinv, None)
    assert _lib.launch_count() - n0 == 1 and len(fake.distort_calls) == 1
    assert fake.warp_calls[1]["src"].tolist() == [t.data_ptr() for t in srcs]
    for t, im in zip(srcs, imgs):
        assert np.array_equal(t.numpy(), im)
    for b, im in enumerate(imgs):
        assert np.array_equal(without[b].numpy(), op.preprocess(im, tinv[b].reshape(-1), (24, 10)))
    assert not torch.equal(with_pd, without)


def test_distort_alone(fake):
    imgs, _, recs = _batch()
    pre = pp.ImageBatchPreprocessor(device="cpu")
    n0 = _lib.launch_count()
    outs = pre.distort([torch.from_numpy(im) for im in imgs], recs)
    assert _lib.launch_count() - n0 == 1
    for o, im, r in zip(outs, imgs, recs):
        assert np.array_equal(o.numpy(), ph.distort(im, ph.Params(*r)))


@pytest.mark.parametrize("bad", [
    (0.0, 1.0, 1.0, 0.0, 0, 6), (0.0, 1.0, 1.0, 0.0, 0, -1), (0.0, 1.0, 1.0, 0.0, 2, 0), (0.0, 1.0, 1.0, 0.0, 0, 1.5),
    (float("nan"), 1.0, 1.0, 0.0, 0, 0), (0.0, float("inf"), 1.0, 0.0, 0, 0), (0.0, 1.0, 1e39, 0.0, 0, 0),
    (0.0, 1.0, 1.0, 0.0, 0), None, "abcdef"])
def test_malformed_records_raise_before_any_launch(fake, bad):
    imgs, tinv, recs = _batch()
    pre = pp.ImageBatchPreprocessor(resolution=(24, 10), device="cpu")
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        pre([torch.from_numpy(im) for im in imgs], tinv, None, distort=recs[:2] + [bad])
    with pytest.raises(ValueError):
        pre.distort([torch.from_numpy(im) for im in imgs], recs[:2] + [bad])
    assert _lib.launch_count() == n0 and not fake.distort_calls and not fake.warp_calls


def test_record_count_must_match_the_batch(fake):
    imgs, tinv, recs = _batch()
    with pytest.raises(ValueError):
        pp.ImageBatchPreprocessor(resolution=(24, 10), device="cpu")([torch.from_numpy(im) for im in imgs], tinv, None, distort=recs[:2])


def test_record_layout_matches_the_header():
    assert pp._RECORD_DTYPE.itemsize == 24
    assert [pp._RECORD_DTYPE.fields[n][1] for n in pp.PhotometricParams._fields] == [0, 4, 8, 12, 16, 20]
