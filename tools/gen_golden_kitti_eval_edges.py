"""Generate tests/golden/kitti_eval_edges.npz: the reference KITTI evaluation where overlaps meet the thresholds (CPU only).

    NUMBA_ENABLE_CUDASIM=1 python tools/gen_golden_kitti_eval_edges.py      (the variable is set here if absent)

The UNMODIFIED reference is imported in place as tools/gen_golden_kitti_eval.py does it (numba's CUDA simulator for
rotate_iou.py, an in-memory stand-in for `skimage.io`).  Candidate cases are searched with oracle/kitti_eval.py (fast); every
stored overlap block, AP array and result string comes from the reference itself, and the generator stops if the reference
disagrees with a case's label.  Annotations are built in memory (no text round trip), so that a value one ulp off the 0.01
grid survives.

A label (metric m, threshold t, step k) says that the reference's overlap of the pair is the k-th representable value above
base(t), where base(t) is the largest value of the metric's type that does not pass `overlap > t` (t as a float64, the type
min_overlaps has): fp64(t) for the 2-d overlap, the largest float32 <= fp64(t) for BEV and 3-d, which are float32 values
widened to float64.  So k <= 0 fails the threshold and k >= 1 passes it; k = 0 / 1 are the two values a one-ulp error flips.

Cases (one image per pair in e1-e4; gt and detection of the class whose min_overlap is t):
  e1  2-d ties, t in (0.25, 0.5, 0.7), k in -2..2: boxes on the 0.01 grid first (nested and partly overlapping boxes whose
      exact IoU is t), float64 ulp steps of one coordinate for the bins the grid does not fill; plus touching boxes (iw == 0)
  e2  BEV ties, k in -2..2, ry in {0, +-1.57, +-3.14, float32(+-pi/2), float32(pi)} and random 2-decimal angles: nested
      rotated footprints whose exact area ratio is t, 2-decimal dimensions / locations first, float32 ulp steps after
  e3  3-d ties, the same search on the 3-d overlap (fp64 height overlap times the fp32 intersection, stored through fp32)
  e4  degenerate rotated geometry: identical and concentric boxes (collinear and coincident edges) at every multiple of
      pi/2, boxes inside others with one or two shared edges, corners on edges, boxes meeting at one corner, zero-length /
      zero-width detections, and repeated intersection vertices (the 0 / 0 of the reference's vertex sort).  A gt and a
      detection that both have zero volume are left out: the reference's d3_box_overlap_kernel raises ZeroDivisionError
  e5  whole-evaluation images where every match decision sits on a tie: all three classes and difficulties, an ignored
      detection on a tie, two detections with bit-identical overlaps to one gt (the lower index wins), a valid and an
      ignored detection at equal overlap, DontCare regions whose criterion-0 overlap is at the threshold; also evaluated by
      distance bin
  e4o pairs with more than 8 candidate intersection points (a box and the same box with the heading flipped between
      float32(pi / 2) and float32(-pi / 2), or float32(pi) and float32(-pi)), with the error the reference raises there
  e6  get_thresholds' 41-point rank selection for every (TP count n, valid-gt count G), 1 <= n <= G <= 300, and whether
      one of its comparisons is an exact tie along the way (e6__tie)

Stored per case e1-e5: the annotations (flattened as in kitti_eval.npz; oracle.kitti_eval.fixture_annos reads them back),
the per-image overlap blocks of the 3 metrics, the 8 do_eval arrays for classes (0, 1, 2) under the official min_overlaps and
under MO_EDGE (the official ones with 0.25 as the 2-d overlap of the second set, so that every e1 threshold decides a match),
and each class's get_official_eval_result output; e5 also get_distance_eval_result.  Deterministic: a second run writes the
same file.
"""
import math
import os
import sys

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")

import numpy as np  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gen_golden_kitti_eval as gk  # noqa: E402
from oracle import kitti_eval as ok  # noqa: E402  (gk put the repository root on sys.path)

OUT = os.path.join(gk.ROOT, "tests", "golden", "kitti_eval_edges.npz")
F32 = np.float32
THRESHOLDS = (0.25, 0.5, 0.7)
STEPS = (-2, -1, 0, 1, 2)
PER_BIN = 3                                   # cases per (threshold, step) in e1-e3
MO_OFFICIAL = np.stack([np.array([[0.7, 0.5, 0.5]] * 3),
                        np.array([[0.7, 0.5, 0.5], [0.5, 0.25, 0.25], [0.5, 0.25, 0.25]])])
MO_EDGE = MO_OFFICIAL.copy()
MO_EDGE[1, 0, :] = 0.25
# the class whose first or second min_overlap of the metric is t (MO_EDGE for the 2-d metric)
CLASS_2D = {0.7: "Car", 0.5: "Pedestrian", 0.25: "Cyclist"}
CLASS_3D = {0.7: "Car", 0.5: "Cyclist", 0.25: "Pedestrian"}
ANGLES = (0.0, 1.57, -1.57, 3.14, -3.14, float(F32(math.pi / 2)), float(F32(-math.pi / 2)), float(F32(math.pi)))
MAX_RANK_GT = 300


# ------------------------------------------------------------------------------------------------------------ labels
def grid(k):
    """The float64 that float('%d.%02d') parses for k hundredths, as a label or result file gives it."""
    s = "-" if k < 0 else ""
    k = abs(int(k))
    return float(f"{s}{k // 100}.{k % 100:02d}")


def base(metric, t):
    if metric == 0:
        return np.float64(t)
    b = F32(t)
    return b if float(b) <= t else np.nextafter(b, F32(-1))


def step_of(metric, t, v):
    """k such that v is k representable values above base(t) (None for NaN / non-positive v)."""
    if not (v > 0):
        return None
    if metric == 0:
        return int(np.float64(v).view(np.int64)) - int(base(0, t).view(np.int64))
    v32 = F32(v)
    if float(v32) != float(v):
        return None
    return int(v32.view(np.int32)) - int(base(metric, t).view(np.int32))


def value_at(metric, t, k):
    """base(t) stepped k representable values up, as a float64."""
    b = base(metric, t)
    if metric == 0:
        return float(np.array(int(b.view(np.int64)) + k, np.int64).view(np.float64))
    return float(np.array(int(b.view(np.int32)) + k, np.int32).view(np.float32))


# ------------------------------------------------------------------------------------------------------------ objects
def obj(name, bbox, loc, hwl, ry, alpha=0.0, occluded=0, truncated=0.0, score=0.0, **extra):
    return dict(name=name, bbox=[float(v) for v in bbox], loc=[float(v) for v in loc], hwl=[float(v) for v in hwl],
                ry=float(ry), alpha=float(alpha), occluded=int(occluded), truncated=float(truncated), score=float(score), **extra)


def anno(objs, det=False):
    """In-memory annotations as get_label_anno returns them (dimensions l, h, w)."""
    import gen_golden_kitti_distance as gd
    return gd.anno(objs, det)


def far_3d(k):
    """A 3-d box that meets nothing: gt and detection of 2-d pairs sit 20 m apart."""
    return [grid(-3000 + 40 * k), grid(150), grid(4000)], [grid(-3000 + 40 * k), grid(150), grid(6000)]


def overlaps_of(g, d):
    """Oracle overlaps (2-d, BEV, 3-d) of one gt / detection pair."""
    o = ok.image_overlaps(anno([g]), anno([d], det=True))
    return [float(x[0, 0]) for x in o]


class Bins:
    """Up to PER_BIN cases per (threshold, step)."""

    def __init__(self, metric):
        self.metric, self.cases = metric, {(t, k): [] for t in THRESHOLDS for k in STEPS}

    def offer(self, t, v, case):
        k = step_of(self.metric, t, v)
        if k in STEPS and len(self.cases[(t, k)]) < PER_BIN:
            self.cases[(t, k)].append(case)
            return True
        return False

    def missing(self):
        return [key for key, c in self.cases.items() if len(c) < PER_BIN]

    def full(self):
        return not self.missing()


# ------------------------------------------------------------------------------------------------------------ e1
RATIOS_2D = {0.25: [(1, 4), (1, 2, 1, 2)], 0.5: [(1, 2), (5, 8, 4, 5)], 0.7: [(7, 10), (7, 8, 4, 5)]}


def draw_2d(rng, t, idx, score):
    """A gt / detection pair whose exact (decimal) IoU is t: nested boxes or two equal-height boxes overlapping in x."""
    x0, y0 = int(rng.integers(0, 100000)), int(rng.integers(0, 20000))
    kind = rng.integers(3)
    if kind < 2:                                                    # nested: area ratio t
        r = RATIOS_2D[t][kind]
        if len(r) == 2:
            (p, q), (pp, qq) = r, (1, 1)
        else:
            p, q, pp, qq = r
        u, v = int(rng.integers(60, 3000)), int(rng.integers(1000, 3000))
        W, w, H, h = q * u, p * u, qq * v, pp * v
        if H < 4000 or h < 4000:
            H, h = H * 3, h * 3
        sx, sy = int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1))
        gb = [x0, y0, x0 + W, y0 + H]
        db = [x0 + sx, y0 + sy, x0 + sx + w, y0 + sy + h]
    else:                                                           # equal heights, overlap o of widths W1, W2: o / (W1 + W2 - o) = t
        p, q = {0.25: (1, 4), 0.5: (1, 2), 0.7: (7, 10)}[t]
        o = int(rng.integers(20, 800)) * p
        tot = o * q // p                                            # W1 + W2 - o
        W1 = int(rng.integers(o, tot + 1))
        W2 = tot + o - W1
        H = int(rng.integers(4000, 20000))
        gb = [x0, y0, x0 + W1, y0 + H]
        db = [x0 + W1 - o, y0, x0 + W1 - o + W2, y0 + H]
    if rng.random() < 0.5:
        gb, db = db, gb
    gl, dl = far_3d(idx)
    g = obj(CLASS_2D[t], [grid(v) for v in gb], gl, [1.5, 1.6, 4.0], 0.0, alpha=0.3)
    d = obj(CLASS_2D[t], [grid(v) for v in db], dl, [1.5, 1.6, 4.0], 0.0, alpha=0.2, score=score)
    return g, d


def ulp_walk(rng, metric, t, k_want, g, d, fields, steps, bins):
    """float ulp steps of the detection's `fields` (list of (key, index, dtype)) until the pair lands in bin (t, k_want)."""
    for _ in range(steps):
        d2 = {key: (list(val) if isinstance(val, list) else val) for key, val in d.items()}
        for key, i, dt in fields:
            n = int(rng.integers(-24, 25))
            cur = d2[key][i] if i is not None else d2[key]
            x = dt(cur)
            for _ in range(abs(n)):
                x = np.nextafter(x, dt(np.inf) if n > 0 else dt(-np.inf))
            if i is None:
                d2[key] = float(x)
            else:
                d2[key][i] = float(x)
        v = overlaps_of(g, d2)[metric]
        if step_of(metric, t, v) == k_want:
            bins.offer(t, v, (g, d2, "ulp"))
            return True
    return False


def e1_cases(rng):
    bins = Bins(0)
    n = 0
    while not bins.full() and n < 20000:
        t = THRESHOLDS[n % 3]
        g, d = draw_2d(rng, t, n % 50, gk.r2(rng.uniform(0.1, 1.0)))
        bins.offer(t, overlaps_of(g, d)[0], (g, d, "grid"))
        n += 1
    for (t, k) in bins.missing():
        while len(bins.cases[(t, k)]) < PER_BIN:
            g, d = draw_2d(rng, t, 7, gk.r2(rng.uniform(0.1, 1.0)))
            ulp_walk(rng, 0, t, k, g, d, [("bbox", 2, np.float64)], 400, bins)
    images, labels = [], []
    for (t, k), cases in sorted(bins.cases.items()):
        for g, d, how in cases:
            images.append(([g], [d]))
            labels.append((0, t, k, how == "grid"))
    # touching boxes: iw == 0 (shared vertical edge), ih == 0 (shared horizontal edge), a shared corner
    for j, (gb, db) in enumerate((([100.1, 120.2, 300.3, 200.4], [300.3, 120.2, 420.5, 200.4]),
                                  ([100.1, 120.2, 300.3, 200.4], [150.7, 200.4, 260.1, 280.9]),
                                  ([100.1, 120.2, 300.3, 200.4], [300.3, 200.4, 400.0, 290.0]))):
        gl, dl = far_3d(60 + j)
        images.append(([obj("Car", gb, gl, [1.5, 1.6, 4.0], 0.0)], [obj("Car", db, dl, [1.5, 1.6, 4.0], 0.0, score=0.5)]))
        labels.append((0, 0.0, 0, True))
    return images, labels


# ------------------------------------------------------------------------------------------------------------ e2 / e3
# (length ratio, width ratio, height ratio) of a detection nested in its gt; the product is t
RATIOS_3D = {0.25: [(5, 16, 4, 5, 1, 1), (5, 8, 1, 2, 4, 5), (1, 2, 5, 8, 4, 5)],
             0.5: [(5, 8, 4, 5, 1, 1), (4, 5, 5, 8, 1, 1), (5, 6, 3, 4, 4, 5)],
             0.7: [(7, 8, 4, 5, 1, 1), (4, 5, 7, 8, 1, 1), (7, 8, 9, 10, 8, 9)]}


def draw_3d(rng, t, angle_idx, score, name):
    """A gt and a nested detection with the same heading: exact footprint-area x height ratio t."""
    lp, lq, wp, wq, hp, hq = RATIOS_3D[t][rng.integers(3)]
    ry = ANGLES[angle_idx] if angle_idx < len(ANGLES) else grid(int(rng.integers(-314, 315)))
    m = int(rng.integers(2, 12))
    L, l = lq * m * 20, lp * m * 20                             # hundredths; l / L = lp / lq
    W, w = wq * 30, wp * 30
    H, h = hq * 25, hp * 25
    x, z, y = int(rng.integers(-1500, 1500)), int(rng.integers(500, 6000)), int(rng.integers(100, 200))
    sl = (L - l) // 2 - 5
    s = int(rng.integers(-sl, sl + 1)) if (sl > 0 and angle_idx < 5 and angle_idx % 2 == 0) else 0   # along x when ry ~ 0 / pi
    sh = int(rng.integers(0, H - h + 1))
    gl, dl = [x, y, z], [x + s, y - sh, z]
    g = obj(name, [100.0, 100.0, 300.0, 200.0], [grid(v) for v in gl], [grid(H), grid(W), grid(L)], ry, alpha=0.1)
    d = obj(name, [110.0, 105.0, 290.0, 195.0], [grid(v) for v in dl], [grid(h), grid(w), grid(l)], ry, alpha=0.4, score=score)
    if rng.random() < 0.3:
        g, d = dict(d, score=0.0, alpha=0.1), dict(g, score=score, alpha=0.4)
    return g, d


def e23_cases(rng):
    bins = {1: Bins(1), 2: Bins(2)}
    n = 0
    while not (bins[1].full() and bins[2].full()) and n < 60000:
        t = THRESHOLDS[n % 3]
        g, d = draw_3d(rng, t, int(rng.integers(0, len(ANGLES) + 4)), gk.r2(rng.uniform(0.1, 1.0)), CLASS_3D[t])
        v = overlaps_of(g, d)
        for m in (1, 2):
            bins[m].offer(t, v[m], (g, d, "grid"))
        n += 1
    print(f"[gen_golden_kitti_eval_edges] e2/e3: {n} grid draws, missing BEV {bins[1].missing()}, 3d {bins[2].missing()}",
          flush=True)
    for m in (1, 2):
        for (t, k) in bins[m].missing():
            while len(bins[m].cases[(t, k)]) < PER_BIN:
                g, d = draw_3d(rng, t, int(rng.integers(0, len(ANGLES) + 4)), gk.r2(rng.uniform(0.1, 1.0)), CLASS_3D[t])
                ulp_walk(rng, m, t, k, g, d, [("hwl", 2, F32), ("loc", 0, F32)], 400, bins[m])
    out = {}
    for m in (1, 2):
        images, labels = [], []
        for (t, k), cases in sorted(bins[m].cases.items()):
            for g, d, how in cases:
                images.append(([g], [d]))
                labels.append((m, t, k, how == "grid"))
        out[m] = (images, labels)
    return out


# ------------------------------------------------------------------------------------------------------------ e4
def n_candidates(g, d):
    """How many points the reference's quadrilateral_intersection would write for the pair (gt = query box)."""
    a = anno([g])
    b = anno([d], det=True)
    r1 = np.array([*a["location"][0, [0, 2]], a["dimensions"][0, 0], a["dimensions"][0, 2], a["rotation_y"][0]], F32)
    r2 = np.array([*b["location"][0, [0, 2]], b["dimensions"][0, 0], b["dimensions"][0, 2], b["rotation_y"][0]], F32)
    c1, c2 = ok._corners(r1), ok._corners(r2)
    n = sum(int(ok._in_quad(c1[2 * i], c1[2 * i + 1], c2)) + int(ok._in_quad(c2[2 * i], c2[2 * i + 1], c1)) for i in range(4))
    return n + sum(ok._segment(c1, c2, i, j) is not None for i in range(4) for j in range(4))


def e4_cases():
    """Crafted degenerate pairs, each at every heading of `angles`; pairs with more than 8 candidate points are returned apart."""
    angles = (0.0, float(F32(math.pi / 2)), float(F32(-math.pi / 2)), float(F32(math.pi)), float(F32(-math.pi)), 1.57, 3.14,
              float(F32(math.pi / 4)), 0.5)
    # (gt (x, z, l, w), detection (x, z, l, w)) in the box's own frame at ry = 0; the pair is rotated about the gt centre
    shapes = [("identical", (0.0, 0.0, 4.0, 2.0), (0.0, 0.0, 4.0, 2.0)),
              ("concentric, equal width", (0.0, 0.0, 4.0, 2.0), (0.0, 0.0, 2.8, 2.0)),
              ("concentric, equal length", (0.0, 0.0, 4.0, 2.0), (0.0, 0.0, 4.0, 1.0)),
              ("inside, one shared edge", (0.0, 0.0, 4.0, 2.0), (1.0, 0.0, 2.0, 1.2)),
              ("inside, two shared edges", (0.0, 0.0, 4.0, 2.0), (1.0, 0.5, 2.0, 1.0)),
              ("collinear edge, half outside", (0.0, 0.0, 4.0, 2.0), (2.0, 0.0, 4.0, 2.0)),
              ("corner on an edge", (0.0, 0.0, 4.0, 2.0), (2.0, 0.5, 2.0, 1.0)),
              ("edge to edge", (0.0, 0.0, 4.0, 2.0), (4.0, 0.0, 4.0, 2.0)),
              ("corner to corner", (0.0, 0.0, 4.0, 2.0), (4.0, 2.0, 4.0, 2.0)),
              ("zero length", (0.0, 0.0, 4.0, 2.0), (0.0, 0.0, 0.0, 1.0)),
              ("zero width", (0.0, 0.0, 4.0, 2.0), (0.0, 0.0, 2.0, 0.0)),
              ("cross", (0.0, 0.0, 4.0, 2.0), (0.0, 0.0, 2.0, 4.0))]
    images, kinds, over = [], [], []
    for ai, ry in enumerate(angles):
        c, s = math.cos(ry), math.sin(ry)
        for si, (kind, (gx, gz, gl_, gw), (dx, dz, dl_, dw)) in enumerate(shapes):
            X, Z = 2.0 + 12.0 * si, 20.0 + 3.0 * ai
            # the reference's corner map: x' = cos * x + sin * z, z' = -sin * x + cos * z (rotate_iou.py:225-228)
            def place(px, pz):
                return round(X + c * px + s * pz, 6), round(Z - s * px + c * pz, 6)
            g_xz, d_xz = place(gx, gz), place(dx, dz)
            if ai < 7:                                  # the multiples of pi/2 (and 1.57 / 3.14): exact 0.01-grid offsets
                g_xz = (X + (gx if ai in (0, 6) else 0.0), Z)
                d_xz = {0: (X + dx, Z + dz), 6: (X - dx, Z - dz), 1: (X + dz, Z - dx), 5: (X + dz, Z - dx),
                        2: (X - dz, Z + dx), 3: (X - dx, Z - dz), 4: (X - dx, Z - dz)}[ai]
            g = obj("Car", [100.0, 100.0, 300.0, 200.0], [g_xz[0], 1.5, g_xz[1]], [1.5, gw, gl_], ry, alpha=0.1)
            d = obj("Car", [120.0, 100.0, 320.0, 200.0], [d_xz[0], 1.5, d_xz[1]], [1.5, dw, dl_], ry, alpha=0.3, score=0.5)
            n = n_candidates(g, d)
            if n > 8:                                   # the reference's int_pts holds 8 points
                over.append((kind, ry, n, g, d))
                continue
            images.append(([g], [d]))
            kinds.append(f"{kind} @ ry={ry!r}")
    return images, kinds, over



FLIP_HEADINGS = (0.0, 1.57, -1.57, 3.14, -3.14, float(F32(math.pi / 2)), float(F32(-math.pi / 2)), float(F32(math.pi)),
                 float(F32(-math.pi)))


def overflow_cases(rng, per_pair=3, draws=40000):
    """Pairs whose intersection has more than 8 candidate points: one box on the 0.01 grid and the same box with another
    heading of FLIP_HEADINGS (float32(pi / 2) against float32(-pi / 2) and float32(pi) against float32(-pi) give them:
    parallel edges that cross by a rounding error).  At most `per_pair` cases per (gt heading, detection heading)."""
    found, per = [], {}
    for _ in range(draws):
        a, b = FLIP_HEADINGS[rng.integers(len(FLIP_HEADINGS))], FLIP_HEADINGS[rng.integers(len(FLIP_HEADINGS))]
        x, z = grid(int(rng.integers(-1500, 1500))), grid(int(rng.integers(500, 6000)))
        l, w, h = grid(int(rng.integers(100, 500))), grid(int(rng.integers(50, 250))), grid(int(rng.integers(140, 200)))
        if a == b or per.get((a, b), 0) >= per_pair:
            continue
        g = obj("Car", [100.0, 100.0, 300.0, 200.0], [x, 1.5, z], [h, w, l], a, alpha=0.1)
        d = obj("Car", [120.0, 100.0, 320.0, 200.0], [x, 1.5, z], [h, w, l], b, alpha=0.3, score=0.5)
        n = n_candidates(g, d)
        if n > 8:
            per[(a, b)] = per.get((a, b), 0) + 1
            found.append((f"same box, ry {a!r} / {b!r}", n, g, d))
    return found


# ------------------------------------------------------------------------------------------------------------ e5
DIFFICULTY = (dict(occluded=0, truncated=0.0), dict(occluded=1, truncated=0.2), dict(occluded=2, truncated=0.4))


def _quiet(objs_g, objs_d):
    """True if no two pairs of the image meet: every overlap off the pairs' own (gt i, detection i) is 0 in all 3 metrics."""
    ov = ok.image_overlaps(anno(objs_g), anno(objs_d, det=True))
    for j in range(len(objs_d)):
        for i in range(len(objs_g)):
            if objs_d[j].get("pair", j) != objs_g[i].get("pair", i) and any(o[j, i] != 0 for o in ov):
                return False
    return True


def _strip(objs):
    return [{k: v for k, v in o.items() if k != "pair"} for o in objs]


def _slot(g, d, m, j):
    """Moves a pair to slot j of an image without touching the metric that carries its tie: a 2-d pair gets its 3-d boxes
    placed for the slot, a BEV / 3-d pair its 2-d boxes (which overlap well: IoU ~0.9)."""
    g, d = dict(g), dict(d)
    if m == 0:
        x = grid(-2500 + 1000 * j)
        g["loc"], d["loc"] = [x, grid(150), grid(6500)], [x, grid(150), grid(4500)]
        g["ry"] = d["ry"] = 0.0
        g["hwl"] = d["hwl"] = [1.5, 1.6, 4.0]
    else:
        x = float(1500 + 250 * j)
        g["bbox"], d["bbox"] = [x, 100.0, x + 150.0, 160.0], [x + 5.0, 103.0, x + 150.0, 160.0]
    return g, d


def dontcare_pair(rng, t, k):
    """A DontCare region and a detection of another place whose criterion-0 overlap (the share of the detection's area inside
    the region, eval.py:336-344) is the label's value: grid first, float64 ulp steps of the detection's right edge after."""
    for it in range(200000):
        W, w = int(rng.integers(2000, 20000)), int(rng.integers(1000, 10000))
        p, q = {0.25: (1, 4), 0.5: (1, 2), 0.7: (7, 10)}[t]
        w = (w // q) * q
        a = w * p // q
        x0, y0, H = int(rng.integers(0, 50000)), int(rng.integers(0, 20000)), int(rng.integers(5000, 15000))
        dc = [grid(x0), grid(y0), grid(x0 + W), grid(y0 + H)]
        db = [grid(x0 + W - a), grid(y0), grid(x0 + W - a + w), grid(y0 + H)]
        if it > 1000:
            n = int(rng.integers(-24, 25))
            v = np.float64(db[2])
            for _ in range(abs(n)):
                v = np.nextafter(v, np.inf if n > 0 else -np.inf)
            db[2] = float(v)
        if step_of(0, t, ok.image_box_overlap(np.array([db]), np.array([dc]), 0)[0, 0]) == k:
            return dc, db
    raise RuntimeError("no DontCare pair found")


def e5_images(e1, e23):
    """Whole-evaluation images whose match decisions sit on ties, from the e1-e3 pairs with k = 0 (just fails) and k = 1
    (just passes).  Classes, difficulties and metrics rotate over the slots; a slot is kept only if it meets no other pair."""
    rng = np.random.default_rng(20261018)
    pool = {}
    for m, (images, labels) in ((0, e1), (1, e23[1]), (2, e23[2])):
        for (gts, dts), (_, t, k, _) in zip(images, labels):
            if k in (0, 1):
                pool.setdefault((m, t), []).append((gts[0], dts[0]))
    images = []
    for b in range(18):
        gts, dts = [], []
        for j in range(6):
            for _ in range(50):
                m, t = int(rng.integers(3)), THRESHOLDS[int(rng.integers(3))]
                g, d = pool[(m, t)][int(rng.integers(len(pool[(m, t)])))]
                g, d = _slot(g, d, m, j)
                g.update(DIFFICULTY[(b + j) % 3], alpha=gk.r2(rng.uniform(-3, 3)), pair=j)
                d.update(alpha=gk.r2(rng.uniform(-3, 3)), score=gk.r2(rng.uniform(0.2, 0.95)), pair=j)
                if _quiet(gts + [g], dts + [d]):
                    gts.append(g)
                    dts.append(d)
                    break
        # one anchor TP per class at a low score, so that a detection left unmatched by a tie is a false positive
        for c, name in enumerate(("Car", "Pedestrian", "Cyclist")):
            x = float(3500 + 200 * c)
            loc = [grid(-1200 + 1200 * c), grid(160), grid(1500 + 500 * (b % 4))]
            g = obj(name, [x, 100.0, x + 120.0, 170.0], loc, [1.6, 1.7, 3.9], 0.3, alpha=0.5, pair=10 + c)
            d = obj(name, [x + 4.0, 102.0, x + 120.0, 170.0], [loc[0] + 0.1, loc[1], loc[2] + 0.1], [1.6, 1.7, 3.8], 0.32,
                    alpha=0.4, score=0.05, pair=10 + c)
            if _quiet(gts + [g], dts + [d]):
                gts.append(g)
                dts.append(d)
        images.append((gts, dts))

    # crafted images; each keeps its anchors
    def crafted(extra_g, extra_d):
        gts, dts = list(images[0][0][-3:]), list(images[0][1][-3:])
        assert _quiet(gts + extra_g, dts + extra_d), "crafted e5 image must keep its pairs apart"
        images.append((gts + extra_g, dts + extra_d))

    for t in (0.25, 0.5, 0.7):
        g, d = pool[(1, t)][0] if step_of(1, t, overlaps_of(*pool[(1, t)][0])[1]) == 1 else \
            next(p for p in pool[(1, t)] if step_of(1, t, overlaps_of(*p)[1]) == 1)
        g, d = _slot(g, d, 1, 0)
        g.update(pair=0)
        # an ignored detection on a tie: 2-d height 30 < 40 (easy), valid at moderate / hard
        d_ign = dict(d, bbox=[d["bbox"][0], 130.0, d["bbox"][2], 160.0], pair=0, score=0.7)
        crafted([g], [d_ign])
        # two detections with bit-identical overlaps: the lower index has the lower score and another alpha
        crafted([g], [dict(d, score=0.6, alpha=1.0, pair=0), dict(d, score=0.8, alpha=-1.0, pair=0)])
        # a valid and an ignored detection at equal overlap (same 3-d box; 2-d heights 57 and 30)
        crafted([g], [dict(d_ign, score=0.9, alpha=2.0), dict(d, score=0.6, alpha=-2.0, pair=0)])
    for t in (0.25, 0.5, 0.7):
        g, d = next(p for p in pool[(0, t)] if step_of(0, t, overlaps_of(*p)[0]) == 1)
        g, d = _slot(g, d, 0, 0)
        g.update(pair=0)
        crafted([g], [dict(d, score=0.6, alpha=1.0, pair=0), dict(d, score=0.8, alpha=-1.0, pair=0)])
    # DontCare regions at the criterion-0 threshold of each class (k = 0 keeps the false positive, k = 1 absorbs it)
    for t, name in ((0.7, "Car"), (0.5, "Pedestrian"), (0.25, "Cyclist")):
        for k in (0, 1):
            dc, db = dontcare_pair(rng, t, k)
            g = obj("DontCare", dc, [-1000.0, -1000.0, -1000.0], [-1.0, -1.0, -1.0], -10.0, alpha=-10.0, pair=20)
            d = obj(name, db, [grid(2000), grid(150), grid(6800)], [1.5, 1.6, 4.0], 0.0, alpha=0.1, score=0.5, pair=20)
            crafted([g], [d])
    return [(_strip(g), _strip(d)) for g, d in images]


# ------------------------------------------------------------------------------------------------------------ e6
def rank_tie(n, G, ranks):
    """Whether one of get_thresholds' comparisons (r - c) < (c - l) along the reference's run is a tie in exact arithmetic:
    at step i < n - 1, with j thresholds taken so far, c = j / 40, l = (i + 1) / G, r = (i + 2) / G, and r - c = c - l
    <=> j * G = 20 * (2 i + 3).  There the float64 drift of c (j additions of 1 / 40.0) decides."""
    taken = set(int(x) for x in ranks)
    j = 0
    for i in range(n - 1):
        if j * G == 20 * (2 * i + 3):
            return True
        j += i in taken
    return False


def e6_ranks(ev):
    counts, ranks, tie = [], [], []
    for G in range(1, MAX_RANK_GT + 1):
        for n in range(1, G + 1):
            scores = np.arange(n, 0, -1).astype(np.float64)
            thr = ev.get_thresholds(scores, G)
            r = [n - int(s) for s in thr]
            counts.append(len(r))
            ranks.extend(r)
            tie.append(rank_tie(n, G, r))
    return np.array(counts, np.int16), np.array(ranks, np.int16), np.array(tie)


# ------------------------------------------------------------------------------------------------------------ reference runs
def run_case(ev, name, images, store, distance=False):
    gt, dt = [anno(g) for g, _ in images], [anno(d, det=True) for _, d in images]
    gk.run_case(ev, name, gt, dt, store)
    compute_aos = bool(store[f"{name}__compute_aos"])
    for i, r in enumerate(ev.do_eval(gt, dt, [0, 1, 2], MO_EDGE, compute_aos)):
        store[f"{name}__do_eval_edge{i}"] = np.zeros(0) if r is None else r
    if distance:
        for i, r in enumerate(ev.do_eval(gt, dt, [0, 1, 2], MO_OFFICIAL, compute_aos, DIForDIS=False)):
            store[f"{name}__do_eval_dist{i}"] = np.zeros(0) if r is None else r
        for c in range(3):
            store[f"{name}__dist_result{c}"] = np.array(ev.get_distance_eval_result(gt, dt, c)[0])
    # the oracle must reproduce every reference overlap bit for bit (else the search above labelled the wrong values)
    blocks = [ok.image_overlaps(g, d) for g, d in zip(gt, dt)]
    for m in range(3):
        got = np.concatenate([b[m].reshape(-1) for b in blocks]) if blocks else np.zeros(0)
        ref = store[f"{name}__ov{m}"]
        same = (got.view(np.int64) == ref.view(np.int64)) | (np.isnan(got) & np.isnan(ref))
        assert same.all(), f"{name}: oracle and reference differ on metric {m} at {np.flatnonzero(~same)[:5]}"
    return gt, dt


def store_labels(ev, name, labels, store):
    """Labels of one-pair images, checked against the reference's own overlaps."""
    lab = np.array([(m, t, k, grid_) for m, t, k, grid_ in labels], np.float64).reshape(-1, 4)
    store[f"{name}__label_metric"] = lab[:, 0].astype(np.int64)
    store[f"{name}__label_t"] = lab[:, 1]
    store[f"{name}__label_k"] = lab[:, 2].astype(np.int64)
    store[f"{name}__label_grid"] = lab[:, 3].astype(bool)
    for b, (m, t, k, _) in enumerate(labels):
        v = store[f"{name}__ov{m}"][b]                 # one gt and one detection per image: block b is entry b
        want = 0.0 if t == 0.0 else value_at(m, t, k)
        assert v.view(np.int64) == np.float64(want).view(np.int64), f"{name} image {b}: reference {v!r}, label {want!r}"


def main():
    ev, _ = gk.reference()
    rng = np.random.default_rng(20261018)
    store = {"steps": np.array(STEPS), "thresholds": np.array(THRESHOLDS), "mo_edge": MO_EDGE}

    e1, e1_labels = e1_cases(rng)
    e23 = e23_cases(rng)
    e4, e4_kinds, e4_over = e4_cases()
    for name, images, labels in (("e1", e1, e1_labels), ("e2", *e23[1]), ("e3", *e23[2])):
        run_case(ev, name, images, store)
        store_labels(ev, name, labels, store)
    run_case(ev, "e4", e4, store)
    store["e4__kind"] = np.array(e4_kinds)
    assert not e4_over, "a same-heading e4 pair has more than 8 candidate points"
    # more than 8 candidate points: the reference's 16-float int_pts overflows (its simulator run raises, its GPU run writes
    # past a local array); stored with the error the reference raises, for the oracle's and the device's 8-point clamp
    over = overflow_cases(np.random.default_rng(20261019))
    gk.flatten("e4o__gt_", [anno([g]) for _, _, g, _ in over], store)
    gk.flatten("e4o__dt_", [anno([d], det=True) for _, _, _, d in over], store)
    store["e4o__kind"] = np.array([k for k, _, _, _ in over])
    store["e4o__n"] = np.array([n for _, n, _, _ in over], np.int64)
    errors = []
    for _, _, g, d in over:
        try:
            ev.calculate_iou_partly([anno([d], det=True)], [anno([g])], 1, 1)
            errors.append("no error")
        except Exception as e:                         # noqa: BLE001 -- recorded, not handled
            errors.append(f"{type(e).__name__}: {e}")
    store["e4o__reference_error"] = np.array(errors)
    print(f"[gen_golden_kitti_eval_edges] e4o: {len(over)} pairs with > 8 candidate points, reference: {sorted(set(errors))}",
          flush=True)
    e5 = e5_images((e1, e1_labels), e23)
    run_case(ev, "e5", e5, store, distance=True)
    print("[gen_golden_kitti_eval_edges] e6: get_thresholds ranks", flush=True)
    store["e6__count"], store["e6__rank"], store["e6__tie"] = e6_ranks(ev)
    np.savez_compressed(OUT, **store)
    print(f"[gen_golden_kitti_eval_edges] wrote {OUT} ({os.path.getsize(OUT)} bytes)")


if __name__ == "__main__":
    main()
