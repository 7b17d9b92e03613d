"""oracle/photometric.py and PhotometricDistort.sample() against the reference's photometric distortion (pd.py + cv2 + numpy):
the fixture tests/golden/photometric.npz (tools/gen_golden_photometric.py) and, with the reference tree present, the live code."""
import importlib.util
import os

import numpy as np
import pytest

from oracle import photometric as ph
from oracle import preprocess as op

GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "photometric.npz"))
N_CASES = len(GOLD["sizes"])


def case_image(i):
    return op.synthetic_images(int(GOLD["img_seed"]) + i, [tuple(int(v) for v in GOLD["sizes"][i])])[0]


def case_params(i):
    r = GOLD[f"{i}.record"]
    return ph.Params(*r[:4], int(r[4]), int(r[5]))


def test_oracle_is_bit_identical_to_the_fixture():
    for i in range(N_CASES):
        assert np.array_equal(ph.distort(case_image(i), case_params(i)), GOLD[f"{i}.u8"]), i


def test_fixture_covers_orders_steps_permutations_and_tails():
    recs = np.stack([GOLD[f"{i}.record"] for i in range(N_CASES)])
    assert set(recs[:, 4]) == {0, 1} and set(recs[:, 5]) == set(range(6))
    for col, neutral in ((0, 0.0), (1, 1.0), (2, 1.0), (3, 0.0)):
        assert (recs[:, col] == neutral).any() and (recs[:, col] != neutral).any(), col
    assert {int(w) % ph.SIMD_WIDTH for w in GOLD["sizes"][:, 0]} == set(range(ph.SIMD_WIDTH))


def test_sample_reproduces_the_reference_draws_and_stream():
    from monodetr_b200.preprocess import PhotometricDistort
    pd = PhotometricDistort()
    for i in range(N_CASES):
        np.random.seed(int(GOLD["seeds"][i]))
        rec = pd.sample()
        assert tuple(rec) == tuple(case_params(i)), i
        assert ph.state_matches(GOLD, f"{i}."), i


def test_getitem_end_to_end_on_the_cpu():
    """Distortion -> flip -> PIL warp as KITTI_Dataset.__getitem__ does, replayed from the seed, equals the dataset's output."""
    from monodetr_b200.preprocess import PhotometricDistort, get_affine_transform
    src = op.synthetic_images(int(GOLD["e2e.img_seed"]), [tuple(int(v) for v in GOLD["e2e.size"])])[0]
    flips = []
    for k in range(len(GOLD["e2e.seeds"])):
        rec, flip, tinv = ph.replay_getitem(GOLD, k, PhotometricDistort().sample, get_affine_transform)
        assert ph.state_matches(GOLD, f"e2e.{k}.")
        assert flip == bool(GOLD[f"e2e.{k}.flip"])
        img = ph.distort(src, ph.Params(*rec))
        if flip:
            img = img[:, ::-1]
        u8 = op.warp_affine_bilinear(img, tinv.reshape(-1), tuple(int(v) for v in GOLD["e2e.res"]))
        assert np.array_equal(u8, GOLD[f"e2e.{k}.u8"]), k
        flips.append(flip)
    assert set(flips) == {False, True}


# ---- live reference ------------------------------------------------------------------------------------------------------------

def _reference_pd():
    pytest.importorskip("cv2")
    from ref_shims import REF_ROOT
    spec = importlib.util.spec_from_file_location("ref_pd", os.path.join(REF_ROOT, "lib", "datasets", "kitti", "pd.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.PhotometricDistort()


@pytest.mark.reference
def test_oracle_matches_live_reference_on_random_images_and_draws():
    """Widths 1..40 and 1224..1242 (every row-tail residue), full-range pixels (the uint8 wrap); float output compared bitwise."""
    ref = _reference_pd()
    g = np.random.default_rng(5)
    n_wrap = 0
    for W in list(range(1, 41)) + list(range(1224, 1243)):
        H = 3 if W > 100 else 5
        for rep in range(3):
            img = g.integers(0, 256, (H, W, 3), dtype=np.uint8)
            np.random.seed(W * 10 + rep)
            st = np.random.get_state()
            p = ph.sample()
            np.random.set_state(st)
            want = ref(img.astype(np.float32))
            got = ph.distort_float(img, p)
            assert np.array_equal(got.view(np.int32), np.ascontiguousarray(want).view(np.int32)), (W, rep, p)
            assert np.array_equal(ph.to_u8(got), want.astype(np.uint8)), (W, rep, p)
            n_wrap += int(((want < 0) | (want >= 256)).sum())
    assert n_wrap > 0


@pytest.mark.reference
def test_sample_leaves_the_same_stream_as_the_reference_call():
    from monodetr_b200.preprocess import PhotometricDistort
    ref, pd = _reference_pd(), PhotometricDistort()
    img = np.zeros((2, 2, 3), np.float32)
    for seed in range(200):
        np.random.seed(seed)
        pd.sample()
        mine = np.random.get_state()
        np.random.seed(seed)
        ref(img.copy())
        theirs = np.random.get_state()
        assert mine[2:] == theirs[2:] and np.array_equal(mine[1], theirs[1]), seed
