"""numpy restatement of the label half of the reference dataset's __getitem__ (lib/datasets/kitti/kitti_dataset.py:173-330,
with Object3d / Calibration.rect_to_img / ry2alpha of kitti_utils.py:13-51,180-189,286-294 and angle2class of
lib/datasets/utils.py:8-16), written from the reference's observable behaviour.  Test and benchmark infrastructure only.

Every step is evaluated at the precision numpy 2 gives it in the reference:
  - fp64: the flip of box2d and ry, the affine map of the box corners and of the projected 3-d centre, the projection itself,
    the normalisations by `resolution` and l / r / t / b, depth scaling, the level test and the size encoding;
  - fp32: the 2-d centre, w / h, and all of ry2alpha + angle2class (the Python floats there are weak scalars: rounded to
    float32 first, numpy's float `%` semantics);
each result rounded to float32 where the reference stores it into a float32 array.  Sums run left to right without FMA.  The one
step numpy does not round correctly, float32 arctan2, is taken here as atan2 in fp64 rounded to float32.

A label line is one row of the record layout below (float32 fields hold float32 values).
"""
import numpy as np

F32 = np.float32
WIDTH = 16
CLS, TRUNC, OCC, ALPHA, X1, Y1, X2, Y2, H, W, L, PX, PY, PZ, RY = range(15)
CLASS_NAMES = ("Pedestrian", "Car", "Cyclist")          # class code = index; any other type is -1
MAX_OBJS = 50
NUM_HEADING_BIN = 12
DEPTH_SCALES = ("normal", "inverse", "none")
KEYS = ("calibs", "indices", "labels", "boxes", "boxes_3d", "depth", "size_2d", "size_3d", "src_size_3d", "heading_bin",
        "heading_res", "mask_2d")
CLS_MEAN_SIZE = np.array([[1.76255119, 0.66068622, 0.84422524],
                          [1.52563191462, 1.62856739989, 3.88311640418],
                          [1.73698127, 0.59706367, 1.76282397]])


def records(cls_names, f64, box2d, pos):
    """Record rows from parsed Object3d fields: class names, (n, 7) fp64 (trunc, occ, alpha, h, w, l, ry), box2d / pos float32."""
    recs = np.zeros((len(cls_names), WIDTH))
    recs[:, CLS] = [CLASS_NAMES.index(c) if c in CLASS_NAMES else -1 for c in cls_names]
    recs[:, [TRUNC, OCC, ALPHA, H, W, L, RY]] = np.asarray(f64, np.float64).reshape(-1, 7)
    recs[:, X1:Y2 + 1] = np.asarray(box2d, np.float32).reshape(-1, 4)
    recs[:, PX:PZ + 1] = np.asarray(pos, np.float32).reshape(-1, 3)
    return recs


def gold_bank(gold):
    """(offsets, records, P2s) of the fixture's parsed label lines."""
    offsets = np.concatenate([[0], np.cumsum(gold["parsed.count"])]).astype(np.int64)
    return offsets, records([str(c) for c in gold["parsed.cls"]], gold["parsed.f64"], gold["parsed.box2d"], gold["parsed.pos"]), \
        gold["parsed.P2"]


def gold_config(gold, name):
    """The encoder settings of fixture variant `name` (its json overrides on top of configs/monodetr.yaml's)."""
    import json
    over = json.loads(str(gold[f"{name}.cfg"]))
    return dict(class_mask=sum(1 << CLASS_NAMES.index(c) for c in over.get("writelist", ["Car"])),
                clip_2d=bool(over.get("clip_2d", False)), depth_scale=over.get("depth_scale", "normal"),
                mean_size=CLS_MEAN_SIZE if over.get("meanshape", False) else None,
                resolution=tuple(int(v) for v in gold[f"{name}.resolution"]))


def empty_targets(B, max_objs=MAX_OBJS):
    return {"calibs": np.zeros((B, max_objs, 3, 4), np.float32), "indices": np.zeros((B, max_objs), np.int64),
            "labels": np.zeros((B, max_objs), np.int8), "boxes": np.zeros((B, max_objs, 4), np.float32),
            "boxes_3d": np.zeros((B, max_objs, 6), np.float32), "depth": np.zeros((B, max_objs, 1), np.float32),
            "size_2d": np.zeros((B, max_objs, 2), np.float32), "size_3d": np.zeros((B, max_objs, 3), np.float32),
            "src_size_3d": np.zeros((B, max_objs, 3), np.float32), "heading_bin": np.zeros((B, max_objs, 1), np.int64),
            "heading_res": np.zeros((B, max_objs, 1), np.float32), "mask_2d": np.zeros((B, max_objs), bool)}


def level_unknown(box, trunc, occ):
    """Object3d.get_obj_level() == 4 ('UnKnown'); the height comes from the float32 box in fp64."""
    height = float(box[3]) - float(box[1]) + 1
    if trunc == -1:
        return False
    if height >= 40 and trunc <= 0.15 and occ <= 0:
        return False
    if height >= 25 and trunc <= 0.3 and occ <= 1:
        return False
    return not (height >= 25 and trunc <= 0.5 and occ <= 2)


def _affine(t, x, y):
    """affine_transform(): the point goes through a float32 array, the product is fp64."""
    x, y = float(F32(x)), float(F32(y))
    return t[0, 0] * x + t[0, 1] * y + t[0, 2], t[1, 0] * x + t[1, 1] * y + t[1, 2]


def _mod32(a, b):
    """numpy's float32 `%`: fmod, then moved into the divisor's sign."""
    m = F32(np.fmod(F32(a), F32(b)))
    if m != 0 and (m < 0) != (F32(b) < 0):
        m = F32(m + F32(b))
    return m


def angle2class(angle):
    """lib/datasets/utils.py:8-16 with a float32 angle."""
    two_pi = F32(2 * np.pi)
    apc = 2 * np.pi / float(NUM_HEADING_BIN)
    a = _mod32(angle, two_pi)
    shifted = _mod32(F32(a + F32(apc / 2)), two_pi)
    cid = int(F32(shifted / F32(apc)))
    return cid, F32(shifted - F32(cid * apc + apc / 2)), shifted


def ry2alpha(ry, u, P2):
    """Calibration.ry2alpha for a fp64 ry and a float32 u: float32 throughout."""
    at = F32(np.arctan2(float(F32(u - P2[0, 2])), float(P2[0, 0])))
    alpha = F32(F32(ry) - at)
    pi, two_pi = F32(np.pi), F32(2 * np.pi)
    for _ in range(2):                        # ry2alpha's range check, then kitti_dataset.py:296-297 again
        if alpha > pi:
            alpha = F32(alpha - two_pi)
        if alpha < -pi:
            alpha = F32(alpha + two_pi)
    return alpha


def encode_image(objs, P2, img_size, flip, crop_scale, trans, *, class_mask=0b010, clip_2d=False, depth_scale="normal",
                 mean_size=None, resolution=(1280, 384), max_objs=MAX_OBJS, out=None, b=0, margins=None):
    """Targets of one image into out[key][b] (a fresh batch of one if `out` is None).  objs (n, WIDTH) records, P2 (3, 4) float32,
    img_size (W, H) ints, trans (2, 3) fp64.  class_mask bit c keeps class code c (the writelist).  `margins`, if a list, receives
    (what, signed distance from the threshold) for every decision taken on a kept object."""
    if out is None:
        out = empty_targets(1, max_objs)
    ms = np.zeros((3, 3)) if mean_size is None else np.asarray(mean_size, np.float64)
    P2 = np.asarray(P2, np.float32)
    trans = np.asarray(trans, np.float64)
    resw, resh = float(resolution[0]), float(resolution[1])
    W_img = float(img_size[0])
    mrg = margins.append if margins is not None else (lambda m: None)
    for i in range(min(len(objs), max_objs)):
        o = objs[i]
        c = int(o[CLS])
        if c < 0 or not (class_mask >> c) & 1:
            continue
        box = o[X1:Y2 + 1].astype(np.float32)
        if level_unknown(box, o[TRUNC], o[OCC]) or F32(o[PZ]) < 2 or F32(o[PZ]) > 65:
            continue
        mrg(("z", float(o[PZ]) - 2)); mrg(("z", 65 - float(o[PZ])))
        ry = float(o[RY])
        if flip:
            box = np.array([W_img - float(box[2]), box[1], W_img - float(box[0]), box[3]], np.float32)
            ry = np.pi - ry
            if ry > np.pi:
                ry -= 2 * np.pi
            if ry < -np.pi:
                ry += 2 * np.pi
        b0, b1 = (F32(v) for v in _affine(trans, box[0], box[1]))
        b2, b3 = (F32(v) for v in _affine(trans, box[2], box[3]))
        c2x, c2y = F32(F32(b0 + b2) / F32(2)), F32(F32(b1 + b3) / F32(2))
        # projected 3-d centre: (pos + [0, -h/2, 0]) in fp64, [x y z 1] . P2 rows, / z
        X, Y, Z = float(F32(o[PX])), float(F32(o[PY])) + (-float(o[H]) / 2), float(F32(o[PZ]))
        p = P2.astype(np.float64)
        u = (((p[0, 0] * X + p[0, 1] * Y) + p[0, 2] * Z) + p[0, 3] * 1.0) / Z
        v = (((p[1, 0] * X + p[1, 1] * Y) + p[1, 2] * Z) + p[1, 3] * 1.0) / Z
        if flip:
            u = W_img - u
        c3x, c3y = _affine(trans, u, v)
        mrg(("proj", c3x)); mrg(("proj", resw - c3x)); mrg(("proj", c3y)); mrg(("proj", resh - c3y))
        if c3x < 0 or c3x >= resw or c3y < 0 or c3y >= resh:
            continue
        out["labels"][b, i] = c
        w2, h2 = F32(b2 - b0), F32(b3 - b1)
        out["size_2d"][b, i] = w2, h2
        cn = [F32(float(b0) / resw), F32(float(b1) / resh), F32(float(b2) / resw), F32(float(b3) / resh)]
        c3nx, c3ny = c3x / resw, c3y / resh
        ltrb = [c3nx - float(cn[0]), float(cn[2]) - c3nx, c3ny - float(cn[1]), float(cn[3]) - c3ny]
        for s in ltrb:
            mrg(("ltrb", s))
        if min(ltrb) < 0:
            if not clip_2d:
                continue
            ltrb = [min(max(s, 0.0), 1.0) for s in ltrb]
        out["boxes"][b, i] = float(c2x) / resw, float(c2y) / resh, float(w2) / resw, float(h2) / resh
        out["boxes_3d"][b, i] = [c3nx, c3ny] + ltrb
        z = F32(o[PZ])
        out["depth"][b, i] = {"normal": float(z) * crop_scale, "inverse": float(z) / crop_scale, "none": z}[depth_scale]
        alpha = ry2alpha(ry, F32(F32(box[0] + box[2]) / F32(2)), P2)
        cid, res, shifted = angle2class(alpha)
        apc = 2 * np.pi / NUM_HEADING_BIN
        mrg(("bin", float(shifted) - cid * apc)); mrg(("bin", (cid + 1) * apc - float(shifted)))
        out["heading_bin"][b, i] = cid
        out["heading_res"][b, i] = res
        src = np.array([o[H], o[W], o[L]], np.float32)
        out["src_size_3d"][b, i] = src
        out["size_3d"][b, i] = src.astype(np.float64) - ms[c]
        if o[TRUNC] <= 0.5 and o[OCC] <= 2:
            out["mask_2d"][b, i] = True
        out["calibs"][b, i] = P2
    return out


def encode_batch(offsets, objects, P2s, bank_idx, img_sizes, flips, crop_scales, trans, **cfg):
    """The encoder over a batch: image b reads objects[offsets[k]:offsets[k+1]] and P2s[k], k = bank_idx[b]."""
    out = empty_targets(len(bank_idx), cfg.get("max_objs", MAX_OBJS))
    for b, k in enumerate(bank_idx):
        encode_image(objects[offsets[k]:offsets[k + 1]], P2s[k], img_sizes[b], bool(flips[b]), float(crop_scales[b]), trans[b],
                     out=out, b=b, **cfg)
    return out


EXACT = ("labels", "mask_2d", "indices", "calibs", "depth", "size_3d", "src_size_3d", "heading_bin")


def assert_targets_match(got, want, what=""):
    """The encoder's agreement with the reference's targets (numpy arrays of equal shapes):
      - exact: the slot pattern (labels, mask_2d, and every zero slot of every key), indices, calibs, depth, size_3d, src_size_3d,
        heading_bin -- no step on their path is evaluated differently;
      - boxes, boxes_3d, size_2d within 1 float32 ulp: they come from fp64 dot products (the affine map, the projection) that
        numpy hands to BLAS, which may contract them to FMA; the value stored is the fp64 result rounded once, so expected exact;
      - heading_res within 1e-6 (absolute): numpy's float32 arctan2 is not correctly rounded (up to 3 ulp on AVX-512 hosts), the
        encoder's is."""
    for k in EXACT:
        np.testing.assert_array_equal(np.asarray(got[k]), np.asarray(want[k]), err_msg=f"{what} {k}")
    for k in ("boxes", "boxes_3d", "size_2d", "heading_res"):
        g, w = np.asarray(got[k], np.float32), np.asarray(want[k], np.float32)
        np.testing.assert_array_equal(g == 0, w == 0, err_msg=f"{what} {k}: slot pattern")
        if k == "heading_res":
            np.testing.assert_allclose(g, w, rtol=0, atol=1e-6, err_msg=f"{what} {k}")
        else:
            ulps = np.abs(g.view(np.int32).astype(np.int64) - w.view(np.int32).astype(np.int64))
            assert ulps.max(initial=0) <= 1, f"{what} {k}: {ulps.max()} ulp"
