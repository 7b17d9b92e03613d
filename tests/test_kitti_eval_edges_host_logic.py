"""CPU: oracle/kitti_eval.py against the reference where overlaps meet the thresholds (tests/golden/kitti_eval_edges.npz,
tools/gen_golden_kitti_eval_edges.py), bit for bit, and proof that the fixture catches one-ulp errors: overlaps moved across
a threshold, a rotated intersection with contracted multiply-adds, and cos / sin one float32 ulp off all change its results."""
import math
import os

import numpy as np
import pytest

from monodetr_b200 import kitti_eval as ke
from oracle import kitti_eval as ok

CASES = ("e1", "e2", "e3", "e4", "e5")
TIE_CASES = ("e1", "e2", "e3")
F32 = np.float32
MO = ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_eval_edges.npz")))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


def same_bits(a, b):
    """Bit-identical float64 arrays (any NaN matches any NaN: the reference's 0 / 0 and the device's differ in payload)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(((a.view(np.int64) == b.view(np.int64)) | (np.isnan(a) & np.isnan(b))).all())


def base(metric, t):
    """The largest value of the metric's type that does not pass `overlap > t`."""
    if metric == 0:
        return np.float64(t)
    b = F32(t)
    return b if float(b) <= t else np.nextafter(b, F32(-1))


def value_at(metric, t, k):
    b = base(metric, t)
    if metric == 0:
        return np.array(int(b.view(np.int64)) + k, np.int64).view(np.float64)[()]
    return np.float64(np.array(int(b.view(np.int32)) + k, np.int32).view(np.float32)[()])


def labels(golden, case):
    return zip(golden[f"{case}__label_metric"], golden[f"{case}__label_t"], golden[f"{case}__label_k"])


def ap_arrays(golden, case, key):
    return [golden[f"{case}__{key}{i}"] if golden[f"{case}__{key}{i}"].size else None for i in range(8)]


def ap_equal(got, ref):
    return all((g is None and r is None) or (g is not None and r is not None and np.array_equal(g, r)) for g, r in zip(got, ref))


class CachedOverlaps:
    """oracle.kitti_eval.image_overlaps served from a cache keyed by image (so that a mutant run costs only the statistics),
    with an optional change to one image's block."""

    def __init__(self, gt, dt):
        self.blocks = {id(g): ok.image_overlaps(g, d) for g, d in zip(gt, dt)}
        self.change = None

    def __call__(self, g, d):
        blocks = [b.copy() for b in self.blocks[id(g)]]
        if self.change is not None and self.change[0] == id(g):
            _, m, value = self.change
            blocks[m][0, 0] = value
        return tuple(blocks)


# ---------------------------------------------------------------------------------------------------------------- parity
@pytest.mark.parametrize("case", CASES)
def test_overlaps_match_reference_bit_for_bit(golden, case):
    gt, dt = annos(golden, case)
    blocks = [ok.image_overlaps(g, d) for g, d in zip(gt, dt)]
    for m in range(3):
        got = np.concatenate([b[m].reshape(-1) for b in blocks])
        assert same_bits(got, golden[f"{case}__ov{m}"]), f"metric {m}"


@pytest.mark.parametrize("case", CASES)
def test_ap_arrays_match_reference(golden, case):
    gt, dt = annos(golden, case)
    aos = bool(golden[f"{case}__compute_aos"])
    for key, mo in (("do_eval", MO), ("do_eval_edge", golden["mo_edge"])):
        got = ok.do_eval(gt, dt, [0, 1, 2], mo, aos)
        for g, r in zip(got, ap_arrays(golden, case, key)):
            if r is None:
                assert g is None
            else:
                np.testing.assert_array_equal(g, r)


@pytest.mark.parametrize("case", CASES)
def test_result_strings_match_reference(golden, case, monkeypatch):
    import fake_device_lib
    import torch
    from monodetr_b200 import _lib
    from test_kitti_eval_host_logic import KittiFakeLib
    fake_device_lib.install(monkeypatch)
    lib = KittiFakeLib(1)
    lib.evals = []
    monkeypatch.setattr(_lib, "_lib", lib)
    monkeypatch.setattr(ke, "_device", lambda: torch.device("cpu"))
    gt, dt = annos(golden, case)
    for c in range(3):
        assert ke.get_official_eval_result(gt, dt, c)[0] == str(golden[f"{case}__result{c}"])


# ---------------------------------------------------------------------------------------------------------------- labels
@pytest.mark.parametrize("case", TIE_CASES)
def test_labels_are_true(golden, case):
    """Each image of e1-e3 holds one pair whose overlap of the labelled metric is exactly base(t) stepped k values (0 for the
    touching boxes of e1)."""
    for b, (m, t, k) in enumerate(labels(golden, case)):
        v = golden[f"{case}__ov{m}"][b]
        want = 0.0 if t == 0.0 else value_at(int(m), float(t), int(k))
        assert same_bits(v, want), (case, b, m, t, k, v, want)
        if t:
            assert (v > t) == (k >= 1)


def test_every_threshold_and_step_is_covered(golden):
    counts = {}
    for case in TIE_CASES:
        for m, t, k in labels(golden, case):
            if t:
                counts[(int(m), float(t), int(k))] = counts.get((int(m), float(t), int(k)), 0) + 1
    for m in range(3):
        for t in (0.25, 0.5, 0.7):
            for k in golden["steps"]:
                assert counts.get((m, t, int(k)), 0) >= 3, (m, t, k)
    print("tie cases per (metric, threshold):", {(m, t): sum(v for (mm, tt, _), v in counts.items() if (mm, tt) == (m, t))
                                                  for m in range(3) for t in (0.25, 0.5, 0.7)})
    assert golden["e1__label_grid"].all() and golden["e2__label_grid"].any() and golden["e3__label_grid"].any()


def candidates(g, d):
    """How many points the reference's quadrilateral_intersection (rotate_iou.py:180-201) writes for gt g and detection d:
    corners of each box inside the other, then edge crossings."""
    def rb(a):
        return np.array([a["location"][0, 0], a["location"][0, 2], a["dimensions"][0, 0], a["dimensions"][0, 2],
                         a["rotation_y"][0]], F32)
    c1, c2 = ok._corners(rb(g)), ok._corners(rb(d))
    n = sum(int(ok._in_quad(c1[2 * i], c1[2 * i + 1], c2)) + int(ok._in_quad(c2[2 * i], c2[2 * i + 1], c1)) for i in range(4))
    return n + sum(ok._segment(c1, c2, i, j) is not None for i in range(4) for j in range(4))


def test_candidate_count_of_identical_boxes_is_eight():
    box = {"location": np.array([[1.0, 1.5, 20.0]]), "dimensions": np.array([[4.0, 1.5, 2.0]]), "rotation_y": np.array([0.0])}
    assert candidates(box, box) == 8


def test_e4_pairs_stay_within_eight_points(golden):
    """Every e4 pair went through the reference, whose point array holds 8 points."""
    gt, dt = annos(golden, "e4")
    counts = [candidates(g, d) for g, d in zip(gt, dt)]
    assert max(counts) <= 8 and len(golden["e4__kind"]) == len(gt)


def test_more_than_eight_candidates_are_recorded(golden):
    """e4o: the same box with its heading flipped between float32(+-pi / 2) or float32(+-pi) gives 9 candidates (two
    parallel edges cross by a rounding error); the reference's simulator run raises there.  The oracle keeps the first 8."""
    gt, dt = annos(golden, "e4o")
    assert len(gt) >= 6
    for b, (g, d) in enumerate(zip(gt, dt)):
        assert candidates(g, d) == golden["e4o__n"][b] > 8
        assert str(golden["e4o__reference_error"][b]).startswith("IndexError"), golden["e4o__reference_error"][b]
        assert np.isfinite(np.concatenate([o.reshape(-1) for o in ok.image_overlaps(g, d)])).all()
    headings = {(float(g["rotation_y"][0]), float(d["rotation_y"][0])) for g, d in zip(gt, dt)}
    pi2, pi = float(F32(math.pi / 2)), float(F32(math.pi))
    assert (pi2, -pi2) in headings and (-pi2, pi2) in headings and (pi, -pi) in headings


def rank_tie(n, G, ranks):
    """Whether one comparison (r - c) < (c - l) of get_thresholds along its run is an exact tie: c = j / 40 after j
    thresholds, l = (i + 1) / G, r = (i + 2) / G, so j G = 20 (2 i + 3)."""
    taken, j = set(int(x) for x in ranks), 0
    for i in range(n - 1):
        if j * G == 20 * (2 * i + 3):
            return True
        j += i in taken
    return False


def test_e6_ranks_match_reference(golden):
    counts, ranks = golden["e6__count"], golden["e6__rank"]
    off = np.concatenate([[0], np.cumsum(counts)])
    p = 0
    for G in range(1, 301):
        for n in range(1, G + 1):
            thr = ok.get_thresholds(np.arange(n, 0, -1).astype(np.float64), G)
            assert [n - int(s) for s in thr] == ranks[off[p]:off[p + 1]].tolist(), (n, G)
            assert bool(golden["e6__tie"][p]) == rank_tie(n, G, ranks[off[p]:off[p + 1]]), (n, G)
            p += 1
    assert p == len(counts) and counts.max() <= ke.NUM_THRESH
    assert 0 < golden["e6__tie"].sum() < p


# ---------------------------------------------------------------------------------------------------------------- mutants
@pytest.mark.parametrize("case", TIE_CASES)
def test_one_ulp_across_the_threshold_changes_do_eval(golden, case, monkeypatch):
    """Every overlap at k = 0 moved one value up, and every one at k = 1 one value down, changes some do_eval array."""
    gt, dt = annos(golden, case)
    cache = CachedOverlaps(gt, dt)
    monkeypatch.setattr(ok, "image_overlaps", cache)
    aos = bool(golden[f"{case}__compute_aos"])
    ref = ap_arrays(golden, case, "do_eval_edge")
    assert ap_equal(ok.do_eval(gt, dt, [0, 1, 2], golden["mo_edge"], aos), ref)
    n = 0
    for b, (m, t, k) in enumerate(labels(golden, case)):
        if not t or k not in (0, 1):
            continue
        cache.change = (id(gt[b]), int(m), value_at(int(m), float(t), 1 - int(k)))
        assert not ap_equal(ok.do_eval(gt, dt, [0, 1, 2], golden["mo_edge"], aos), ref), (case, b, m, t, k)
        n += 1
    assert n >= 18


def fma32(a, b, c):
    """float32 fma(a, b, c), exact: a * b is exact in float64; the float64 sum is rounded to odd before the float32 rounding."""
    p, c = float(a) * float(b), float(c)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    if e != 0.0 and not (np.float64(s).view(np.int64) & 1):
        s = float(np.nextafter(s, math.inf if e > 0 else -math.inf))
    return F32(s)


def contracted_corners(rb):
    a_cos, a_sin = F32(math.cos(float(rb[4]))), F32(math.sin(float(rb[4])))
    hx, hy = -rb[2] / F32(2), -rb[3] / F32(2)
    c = []
    for x, y in zip((hx, hx, -hx, -hx), (hy, -hy, -hy, hy)):
        c.append(fma32(a_cos, x, a_sin * y) + rb[0])
        c.append(fma32(-a_sin, x, a_cos * y) + rb[1])
    return c


def contracted_in_quad(px, py, c):
    ab0, ab1, ad0, ad1 = c[2] - c[0], c[3] - c[1], c[6] - c[0], c[7] - c[1]
    ap0, ap1 = px - c[0], py - c[1]
    abab, abap = fma32(ab0, ab0, ab1 * ab1), fma32(ab0, ap0, ab1 * ap1)
    adad, adap = fma32(ad0, ad0, ad1 * ad1), fma32(ad0, ap0, ad1 * ap1)
    return abab >= abap and abap >= 0 and adad >= adap and adap >= 0


def contracted_segment(p1, p2, i, j):
    A0, A1 = p1[2 * i], p1[2 * i + 1]
    B0, B1 = p1[2 * ((i + 1) % 4)], p1[2 * ((i + 1) % 4) + 1]
    C0, C1 = p2[2 * j], p2[2 * j + 1]
    D0, D1 = p2[2 * ((j + 1) % 4)], p2[2 * ((j + 1) % 4) + 1]
    BA0, BA1, DA0, CA0, DA1, CA1 = B0 - A0, B1 - A1, D0 - A0, C0 - A0, D1 - A1, C1 - A1
    if (fma32(DA1, CA0, -(CA1 * DA0)) > 0) == (fma32(D1 - B1, C0 - B0, -((C1 - B1) * (D0 - B0))) > 0):
        return None
    if (fma32(CA1, BA0, -(BA1 * CA0)) > 0) == (fma32(DA1, BA0, -(BA1 * DA0)) > 0):
        return None
    DC0, DC1 = D0 - C0, D1 - C1
    ABBA, CDDC = fma32(A0, B1, -(B0 * A1)), fma32(C0, D1, -(D0 * C1))
    DH = fma32(BA1, DC0, -(BA0 * DC1))
    with np.errstate(divide="ignore", invalid="ignore"):
        return fma32(ABBA, DC0, -(BA0 * CDDC)) / DH, fma32(ABBA, DC1, -(BA1 * CDDC)) / DH


def contracted_triangle(a, b, c):
    return fma32(a[0] - c[0], b[1] - c[1], -((a[1] - c[1]) * (b[0] - c[0]))) / F32(2)


def test_contracted_intersection_changes_e2_ap(golden, monkeypatch):
    """The rotated intersection with the multiply-adds an optimising compiler would fuse (corner map, cross products,
    triangle area) gives different AP arrays on e2: the fixture catches a kernel built with contraction."""
    gt, dt = annos(golden, "e2")
    for name, f in (("_corners", contracted_corners), ("_in_quad", contracted_in_quad), ("_segment", contracted_segment),
                    ("_triangle_area", contracted_triangle)):
        monkeypatch.setattr(ok, name, f)
    blocks = [ok.image_overlaps(g, d) for g, d in zip(gt, dt)]
    moved = sum(not same_bits(b[1], golden["e2__ov1"][i]) for i, b in enumerate(blocks))
    got = ok.do_eval(gt, dt, [0, 1, 2], golden["mo_edge"], bool(golden["e2__compute_aos"]))
    assert not ap_equal(got, ap_arrays(golden, "e2", "do_eval_edge"))
    print(f"contracted intersection: {moved} of {len(blocks)} e2 BEV overlaps differ")


@pytest.mark.parametrize("which", ("cos", "sin"))
def test_cos_sin_one_ulp_off_changes_e2_overlaps(golden, monkeypatch, which):
    gt, dt = annos(golden, "e2")

    def off_by_one(rb):
        """oracle.kitti_eval._corners with the rounded cos or sin one float32 ulp up."""
        a_cos, a_sin = F32(math.cos(float(rb[4]))), F32(math.sin(float(rb[4])))
        if which == "cos":
            a_cos = np.nextafter(a_cos, F32(2))
        else:
            a_sin = np.nextafter(a_sin, F32(2))
        hx, hy = -rb[2] / F32(2), -rb[3] / F32(2)
        c = []
        for x, y in zip((hx, hx, -hx, -hx), (hy, -hy, -hy, hy)):
            c.append(a_cos * x + a_sin * y + rb[0])
            c.append(-a_sin * x + a_cos * y + rb[1])
        return c
    monkeypatch.setattr(ok, "_corners", off_by_one)
    blocks = [ok.image_overlaps(g, d) for g, d in zip(gt, dt)]
    moved = sum(not same_bits(b[1], golden["e2__ov1"][i]) for i, b in enumerate(blocks))
    assert moved >= 1
    print(f"{which} one ulp off: {moved} of {len(blocks)} e2 BEV overlaps differ")
