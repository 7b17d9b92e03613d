"""GPU: the device KITTI evaluation (csrc/kitti_eval.cu via monodetr_b200/kitti_eval.py) where overlaps meet the thresholds,
against the reference's golden vectors (tests/golden/kitti_eval_edges.npz, tools/gen_golden_kitti_eval_edges.py) and the
oracle: overlaps bit for bit, AP arrays and result strings equal, in default and in reproducible mode."""
import math
import os

import numpy as np
import pytest

from monodetr_b200 import _lib
from monodetr_b200 import kitti_eval as ke
from oracle import kitti_eval as ok

pytestmark = pytest.mark.gpu
CASES = ("e1", "e2", "e3", "e4", "e5")
MO = ke.OFFICIAL_MIN_OVERLAPS[:, :, [0, 1, 2]]
F32 = np.float32


@pytest.fixture(scope="module")
def golden(golden_dir):
    return dict(np.load(os.path.join(golden_dir, "kitti_eval_edges.npz")))


@pytest.fixture(params=("default", "reproducible"))
def mode(request):
    was = _lib.deterministic()
    _lib.lib().mdb_set_deterministic(int(request.param == "reproducible"))
    yield request.param
    _lib.lib().mdb_set_deterministic(int(was))


def annos(golden, case):
    return ok.fixture_annos(golden, f"{case}__gt_"), ok.fixture_annos(golden, f"{case}__dt_")


def bit_diff(a, b):
    """Indices where two float64 arrays differ in their bits (any NaN matches any NaN)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape
    return np.flatnonzero((a.view(np.int64) != b.view(np.int64)) & ~(np.isnan(a) & np.isnan(b)))


def check_ap(got, ref):
    for i, (g, r) in enumerate(zip(got, ref)):
        if r is None:
            assert g is None
        elif i in (3, 7):                                       # AOS: device cos against libm
            np.testing.assert_allclose(g, r, rtol=0, atol=1e-10)
        else:
            np.testing.assert_array_equal(g, r)


def ap_arrays(golden, case, key):
    return [golden[f"{case}__{key}{i}"] if golden[f"{case}__{key}{i}"].size else None for i in range(8)]


def box(name, bbox, loc, lhw, ry, alpha=0.0, score=0.0, occluded=0, truncated=0.0):
    return dict(name=name, bbox=bbox, loc=loc, lhw=lhw, ry=ry, alpha=alpha, score=score, occluded=occluded, truncated=truncated)


def anno(objs):
    n = len(objs)
    return {"name": np.array([o["name"] for o in objs]), "truncated": np.array([o["truncated"] for o in objs], np.float64),
            "occluded": np.array([o["occluded"] for o in objs], np.int64), "alpha": np.array([o["alpha"] for o in objs], np.float64),
            "bbox": np.array([o["bbox"] for o in objs], np.float64).reshape(n, 4),
            "dimensions": np.array([o["lhw"] for o in objs], np.float64).reshape(n, 3),
            "location": np.array([o["loc"] for o in objs], np.float64).reshape(n, 3),
            "rotation_y": np.array([o["ry"] for o in objs], np.float64), "score": np.array([o["score"] for o in objs], np.float64)}


# ---------------------------------------------------------------------------------------------------------------- golden
@pytest.mark.parametrize("case", CASES)
def test_overlaps_bit_identical_to_reference(golden, case, mode):
    gt, dt = annos(golden, case)
    blocks = ke.image_overlaps(gt, dt)
    for m in range(3):
        got = np.concatenate([b.reshape(-1) for b in blocks[m]])
        ref = golden[f"{case}__ov{m}"]
        bad = bit_diff(got, ref)
        assert bad.size == 0, f"{case} metric {m}: {bad.size} overlaps differ, first {[(got[i], ref[i]) for i in bad[:4]]}"


@pytest.mark.parametrize("case", CASES)
def test_ap_and_strings_match_reference(golden, case, mode):
    gt, dt = annos(golden, case)
    aos = bool(golden[f"{case}__compute_aos"])
    check_ap(ke.do_eval(gt, dt, [0, 1, 2], MO, aos), ap_arrays(golden, case, "do_eval"))
    check_ap(ke.do_eval(gt, dt, [0, 1, 2], golden["mo_edge"], aos), ap_arrays(golden, case, "do_eval_edge"))
    for c in range(3):
        assert ke.get_official_eval_result(gt, dt, c)[0] == str(golden[f"{case}__result{c}"])
    if f"{case}__do_eval_dist0" in golden:
        check_ap(ke.do_eval(gt, dt, [0, 1, 2], MO, aos, DIForDIS=False), ap_arrays(golden, case, "do_eval_dist"))
        for c in range(3):
            assert ke.get_distance_eval_result(gt, dt, c)[0] == str(golden[f"{case}__dist_result{c}"])


def test_more_than_eight_candidates_keep_the_first_eight(golden, mode):
    """e4o: pairs whose intersection has more than 8 candidate points, where the reference's 16-float point array overflows
    (its simulator run raises).  The device keeps the first 8 candidates, as the oracle does: bit for bit."""
    gt, dt = annos(golden, "e4o")
    assert len(gt) >= 1
    blocks = ke.image_overlaps(gt, dt)
    for b, (g, d) in enumerate(zip(gt, dt)):
        ref = ok.image_overlaps(g, d)
        for m in range(3):
            assert bit_diff(blocks[m][b], ref[m]).size == 0, (str(golden["e4o__kind"][b]), m, blocks[m][b], ref[m])


# ---------------------------------------------------------------------------------------------------------------- ranks
def rank_sets(golden):
    counts = golden["e6__count"]
    off = np.concatenate([[0], np.cumsum(counts)])
    out, p = {}, 0
    for G in range(1, 301):
        for n in range(1, G + 1):
            out[(n, G)] = golden["e6__rank"][off[p]:off[p + 1]]
            p += 1
    return out


def rank_image(name, Gs, chains):
    """One class's image for three rank pairs per metric.  Gs = (G_easy, G_moderate, G_hard): the first G_easy gts are valid
    at every difficulty (occlusion 0), the next G_moderate - G_easy at moderate and hard (occlusion 1), the rest at hard only
    (occlusion 2).  chains[metric] = (n_easy, n_moderate, n_hard): the detections of the first n_easy easy gts, of the first
    n_moderate - n_easy occlusion-1 gts and of the first n_hard - n_moderate occlusion-2 gts match their gt in that metric
    (3-d matches need BEV matches: chains[2] <= chains[1]); every other detection meets nothing.  Gts sit 10 m and 100 px
    apart, and scores fall with the index, so each configuration's TP scores are distinct."""
    G = Gs[2]
    level = np.searchsorted(np.array(Gs), np.arange(G), side="right")          # 0 easy, 1 moderate-only, 2 hard-only
    start = np.array([0, Gs[0], Gs[1]])
    rank_in_level = np.arange(G) - start[level]

    def matched(chain):
        lo = np.array([0, chain[0], chain[1]])
        return rank_in_level < np.array(chain)[level] - lo[level]
    m2d, mbev, m3d = matched(chains[0]), matched(chains[1]), matched(chains[2])
    assert not (m3d & ~mbev).any()
    i = np.arange(G, dtype=np.float64)
    x = 10.0 * i - 1500.0
    gbox = np.stack([100.0 * i, np.full(G, 100.0), 100.0 * i + 60.0, np.full(G, 160.0)], 1)
    dbox = gbox + np.where(m2d, 0.0, 500.0)[:, None] * np.array([0.0, 1.0, 0.0, 1.0])
    gloc = np.stack([x, np.full(G, 1.5), np.full(G, 30.0)], 1)
    dloc = np.stack([np.where(mbev, x, x + 5.0), np.where(m3d | ~mbev, 1.5, 2.9), np.full(G, 30.0)], 1)
    dims = np.tile([4.0, 1.5, 1.6], (G, 1))
    common = {"name": np.array([name] * G), "truncated": np.zeros(G), "alpha": np.zeros(G), "dimensions": dims}
    gt = dict(common, occluded=level.astype(np.int64), bbox=gbox, location=gloc, rotation_y=np.zeros(G), score=np.zeros(G))
    dt = dict(common, occluded=np.zeros(G, np.int64), bbox=dbox, location=dloc, rotation_y=np.full(G, 0.02),
              score=0.9 - 0.001 * i)
    return gt, dt


def rank_slots():
    """Every (n, G) with 1 <= n <= G <= 300, as slots (Gs, chains) of rank_image.  G comes in groups (a, a + 1, a + 2), one
    per difficulty; the chains (n, n, n) for n <= a, (a, a + 1, a + 1) and (a, a + 1, a + 2) cover every n of the group, and
    three of them (componentwise ordered, so that 3-d <= BEV) fill one slot."""
    slots = []
    for a in range(1, 301, 3):
        chains = [(n, n, n) for n in range(1, a + 1)] + [(a, a + 1, a + 1), (a, a + 1, a + 2)]
        for j in range(0, len(chains), 3):
            part = (chains[j:j + 3] + [chains[-1]] * 2)[:3]
            slots.append(((a, a + 1, a + 2), (part[0], part[2], part[1])))         # (2-d, BEV, 3-d)
    return slots


def test_rank_selection_through_whole_evaluations(golden, mode):
    """get_thresholds' ranks (e6) for every (TP count n, valid-gt count G <= 300), through whole evaluations.  One call
    evaluates 6 classes x 3 metrics x 3 difficulties = 54 pairs; the TP count at threshold j is rank j + 1.  The pairs on
    which one of get_thresholds' comparisons is an exact tie (e6__tie) are among them."""
    ranks = rank_sets(golden)
    slots = rank_slots()
    names = [ke.CLASS_TO_NAME[c] for c in range(6)]
    seen = set()
    for s0 in range(0, len(slots), 6):
        call = (slots[s0:s0 + 6] + slots[:6])[:6]
        imgs = [rank_image(names[c], Gs, (ch[0], ch[1], ch[2])) for c, (Gs, ch) in enumerate(call)]
        table = ke.eval_counts([g for g, _ in imgs], [d for _, d in imgs], list(range(6)), ke.OFFICIAL_MIN_OVERLAPS, False)
        table = table.reshape(3, 6, 3, 2, 1 + 4 * ke.NUM_THRESH)
        for c, (Gs, chains) in enumerate(call):
            for metric in range(3):
                for l in range(3):
                    n, G = chains[metric][l], Gs[l]
                    want = ranks[(n, G)]
                    for k in range(2):
                        row = table[metric, c, l, k]
                        assert int(row[0]) == len(want), (n, G, metric, l, k)
                        np.testing.assert_array_equal(row[1::4][:len(want)], want + 1.0, err_msg=f"n={n} G={G}")
                    seen.add((n, G))
    assert seen == set(ranks)
    ties = [key for key, tie in zip(ranks, golden["e6__tie"]) if tie]
    assert ties and set(ties) <= seen
    print(f"rank selection: {len(seen)} (n, G) pairs ({len(ties)} with an exact tie) in {-(-len(slots) // 6)} evaluations")


# ---------------------------------------------------------------------------------------------------------------- headings
def test_every_two_decimal_heading(mode):
    """The BEV overlap of a box rotated to every 2-decimal ry in [-3.15, 3.15] (and float32(+-pi/2), float32(pi)) with one
    fixed box, bit-identical to the oracle: the corner step's cos / sin in isolation."""
    rys = [k / 100 for k in range(-315, 316)] + [float(F32(math.pi / 2)), float(F32(-math.pi / 2)), float(F32(math.pi))]
    g = anno([box("Car", [100.0, 100.0, 300.0, 200.0], [0.37, 1.5, 20.11], [4.13, 1.5, 1.71], 0.0)])
    d = anno([box("Car", [110.0, 100.0, 290.0, 200.0], [0.81, 1.52, 19.64], [3.87, 1.48, 1.63], ry, score=0.5) for ry in rys])
    got = ke.image_overlaps([g], [d])
    ref = ok.image_overlaps(g, d)
    for m in (1, 2):
        bad = bit_diff(got[m][0][:, 0], ref[m][:, 0])
        assert bad.size == 0, f"metric {m}: {[(rys[i], got[m][0][i, 0], ref[m][i, 0]) for i in bad[:6]]}"


# ---------------------------------------------------------------------------------------------------------------- live set
def tie_dense_set(rng, n_img):
    """Integer-pixel 2-d boxes and 0.5 m BEV steps at ry in {0, 1.57, 3.14}, detections jittered from the gts on the same
    steps: exact rational IoUs (0.25, 0.5, ...) are common."""
    names = np.array(["Car", "Pedestrian", "Cyclist", "Van", "DontCare"])
    gts, dts = [], []
    for _ in range(n_img):
        ng, nfp = int(rng.integers(0, 7)), int(rng.integers(0, 3))
        x0, y0 = rng.integers(0, 60, ng) * 10.0, rng.integers(0, 10, ng) * 10.0 + 100.0
        w, h = rng.integers(2, 12, ng) * 10.0, rng.choice([30.0, 40.0, 50.0, 60.0, 80.0], ng)
        g = {"name": rng.choice(names, ng), "truncated": rng.choice([0.0, 0.2, 0.4], ng), "occluded": rng.integers(0, 3, ng),
             "alpha": np.round(rng.uniform(-3, 3, ng), 2), "bbox": np.stack([x0, y0, x0 + w, y0 + h], 1),
             "dimensions": np.stack([rng.choice([2.0, 3.0, 4.0], ng), rng.choice([1.5, 2.0], ng), rng.choice([1.0, 2.0], ng)], 1),
             "location": np.stack([rng.integers(-8, 9, ng) * 2.0, rng.choice([1.5, 2.0], ng), rng.integers(10, 30, ng) * 2.0], 1),
             "rotation_y": rng.choice([0.0, 1.57, 3.14], ng), "score": np.zeros(ng)}
        keep = np.flatnonzero(g["name"] != "DontCare")
        src = np.concatenate([keep, rng.integers(0, max(ng, 1), nfp if ng else 0)]).astype(np.int64)
        nd = len(src)
        bb = g["bbox"][src] + rng.integers(-2, 3, (nd, 4)) * 10.0
        bb[:, 2:] = np.maximum(bb[:, 2:], bb[:, :2] + 10.0)
        d = {"name": np.where(g["name"][src] == "DontCare", "Car", g["name"][src]) if nd else np.zeros(0, "<U3"),
             "truncated": np.zeros(nd), "occluded": np.zeros(nd, np.int64), "alpha": np.round(rng.uniform(-3, 3, nd), 2),
             "bbox": bb, "dimensions": np.stack([rng.choice([2.0, 3.0, 4.0], nd), g["dimensions"][src, 1],
                                                 rng.choice([1.0, 2.0], nd)], 1).reshape(nd, 3),
             "location": g["location"][src] + np.stack([rng.integers(-2, 3, nd) * 0.5, rng.choice([0.0, 0.5], nd),
                                                        rng.integers(-2, 3, nd) * 0.5], 1).reshape(nd, 3),
             "rotation_y": g["rotation_y"][src], "score": np.round(rng.uniform(0, 1, nd), 2)}
        gts.append(g)
        dts.append(d)
    return gts, dts


def test_tie_dense_random_set_matches_oracle(mode):
    rng = np.random.default_rng(20261018)
    gt, dt = tie_dense_set(rng, 80)
    blocks = ke.image_overlaps(gt, dt)
    ties = np.zeros(3, np.int64)
    for b, (g, d) in enumerate(zip(gt, dt)):
        ref = ok.image_overlaps(g, d)
        for m in range(3):
            bad = bit_diff(blocks[m][b], ref[m])
            assert bad.size == 0, f"image {b} metric {m}: {blocks[m][b].reshape(-1)[bad[:4]]} vs {ref[m].reshape(-1)[bad[:4]]}"
            ties[m] += sum(int((ref[m] == t).sum()) for t in (0.25, 0.5, F32(0.25), F32(0.5)))
    assert (ties > 0).all()
    check_ap(ke.do_eval(gt, dt, [0, 1, 2], MO, True), ok.do_eval(gt, dt, [0, 1, 2], MO, True))
    print(f"tie-dense set: overlaps exactly 0.25 / 0.5 per metric {ties.tolist()}")
