"""Device target encoder (csrc/labels.cu through monodetr_b200.labels) against the reference's own __getitem__ targets
(tests/golden/labels.npz, tools/gen_golden_labels.py) and the numpy restatement (oracle/labels.py), with the tolerances stated in
oracle.labels.assert_targets_match; the batch builder end to end; SetCriterion on the device-built targets."""
import os

import numpy as np
import pytest
import torch

from oracle import labels as ol

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(os.path.dirname(__file__), "golden", "labels.npz"))
VARIANTS = ["shipped", "all3", "clip2d", "inverse", "none", "meanshape", "val", "e2e"]
SHIPPED = {"aug_pd": True, "aug_crop": True, "random_flip": 0.5, "random_crop": 0.5, "scale": 0.05, "shift": 0.05,
           "writelist": ["Car"], "clip_2d": False, "depth_scale": "normal", "meanshape": False}


CRIT_CFG = {"num_classes": 3, "cls_loss_coef": 2, "focal_alpha": 0.25, "bbox_loss_coef": 5, "giou_loss_coef": 2,
            "3dcenter_loss_coef": 10, "dim_loss_coef": 1, "angle_loss_coef": 1, "depth_loss_coef": 1, "depth_map_loss_coef": 1,
            "set_cost_class": 2, "set_cost_bbox": 5, "set_cost_giou": 2, "set_cost_3dcenter": 10, "aux_loss": True, "dec_layers": 3}


def _cfg(name):
    import json
    return dict(SHIPPED, **json.loads(str(GOLD[f"{name}.cfg"])))


def _bank():
    from monodetr_b200 import labels as lb
    offsets, recs, P2s = ol.gold_bank(GOLD)
    return lb.LabelBank(offsets, recs, P2s, GOLD["img_ids"])


def _encoder(name):
    from monodetr_b200 import labels as lb
    c = _cfg(name)
    return lb.TargetEncoder(c["writelist"], c["clip_2d"], c["depth_scale"], c["meanshape"],
                            tuple(int(v) for v in GOLD[f"{name}.resolution"]))


def _host(t):
    return {k: v.cpu().numpy() for k, v in t.items()}


@pytest.mark.parametrize("name", VARIANTS)
def test_encoder_matches_the_reference(name):
    """Each variant's images in a batch of 16 (the fixture's images repeated in a shuffled order, ragged line counts 8..55)."""
    from monodetr_b200 import labels as lb
    n = len(GOLD[f"{name}.seeds"])
    order = np.random.default_rng(1).permutation(np.arange(16) % n)
    recs = [lb.AugRecord(tuple(GOLD["sizes"][i]), bool(GOLD[f"{name}.flip"][i]), float(GOLD[f"{name}.crop_scale"][i]),
                         GOLD[f"{name}.center"][i], GOLD[f"{name}.trans"][i], GOLD[f"{name}.trans_inv"][i]) for i in order]
    got = _host(_encoder(name)(_bank(), order.tolist(), recs))
    ol.assert_targets_match(got, {k: GOLD[f"{name}.{k}"][order] for k in ol.KEYS}, name)
    for k in ol.KEYS:
        assert got[k].dtype == GOLD[f"{name}.{k}"].dtype, k


def _synthetic_bank(seed, n_img):
    """KITTI-like random lines (every class code, out-of-range depths, boxes anywhere) with ragged counts 0..60."""
    g = np.random.default_rng(seed)
    counts = g.integers(0, 61, n_img)
    counts[0] = 0
    M = int(counts.sum())
    recs = np.zeros((M, ol.WIDTH))
    recs[:, ol.CLS] = g.integers(-1, 3, M)
    recs[:, ol.TRUNC] = g.choice([-1, 0, 0, 0.1, 0.3, 0.45, 0.6], M)
    recs[:, ol.OCC] = g.integers(0, 4, M)
    x1, y1 = g.uniform(-20, 1200, M), g.uniform(100, 300, M)
    recs[:, ol.X1:ol.Y2 + 1] = np.stack([x1, y1, x1 + g.uniform(5, 300, M), y1 + g.uniform(10, 150, M)], 1).astype(np.float32)
    recs[:, ol.H:ol.L + 1] = np.round(g.uniform(0.5, 4, (M, 3)), 2)
    z = g.uniform(0.5, 75, M)
    recs[:, ol.PX:ol.PZ + 1] = np.stack([g.uniform(-0.5, 0.5, M) * z, g.uniform(1, 2.2, M), z], 1).astype(np.float32)
    recs[:, ol.RY] = np.round(g.uniform(-np.pi, np.pi, M), 2)
    P2 = np.tile(GOLD["parsed.P2"][:2], (n_img // 2 + 1, 1, 1))[:n_img]
    P2[:, 0, 2] += g.uniform(-20, 20, n_img).astype(np.float32)
    return counts, recs, P2


@pytest.mark.parametrize("B", [1, 8, 16])
def test_ragged_random_batch_matches_the_oracle(B):
    from monodetr_b200 import labels as lb
    counts, recs, P2 = _synthetic_bank(B, 40)
    bank = lb.LabelBank.from_arrays(counts, recs, P2)
    g = np.random.default_rng(100 + B)
    idx = g.integers(0, 40, B)
    idx[0] = 0                                                            # an image without lines
    sizes = [(1242, 375), (1224, 370), (1238, 374), (1241, 376)]
    np.random.seed(B)
    for writelist, depth_scale, clip in ((["Car"], "normal", False), (list(ol.CLASS_NAMES), "inverse", True)):
        s = lb.AugmentationSampler("train", True, True, 0.5, 0.8, 0.4, 0.1)
        recs_b = [s.sample(sizes[b % 4]) for b in range(B)]
        enc = lb.TargetEncoder(writelist, clip, depth_scale, meanshape=True)
        got = _host(enc(bank, idx.tolist(), recs_b))
        want = ol.encode_batch(bank.host_offsets, bank.host_objects, P2, idx, [r.img_size for r in recs_b], [r.flip for r in recs_b],
                               [r.crop_scale for r in recs_b], [r.trans for r in recs_b], class_mask=lb.class_mask(writelist),
                               clip_2d=clip, depth_scale=depth_scale, mean_size=ol.CLS_MEAN_SIZE)
        ol.assert_targets_match(got, want, f"B={B} {writelist}")
        assert want["mask_2d"].sum() > 0 or B == 1


def test_batch_builder_end_to_end():
    """The fixture's reference batch: same seeds -> sampler -> KittiBatchBuilder.  `inputs` bit-identical to the reference's
    normalised images; targets within the stated tolerances; P2 and info as the reference's collate."""
    from monodetr_b200 import labels as lb
    from oracle.preprocess import normalize, synthetic_images
    res = tuple(int(v) for v in GOLD["e2e.resolution"])
    n = len(GOLD["e2e.seeds"])
    builder = lb.KittiBatchBuilder(SHIPPED, "train", _bank(), resolution=res)
    imgs = synthetic_images(int(GOLD["img_seed"]), [tuple(s) for s in GOLD["sizes"]])[:n]
    recs = []
    for i, seed in enumerate(GOLD["e2e.seeds"]):
        np.random.seed(int(seed))
        recs.append(builder.sampler.sample(GOLD["sizes"][i]))
    assert [r.flip for r in recs] == GOLD["e2e.flip"].tolist() and any(r.flip for r in recs)
    assert [r.crop_scale for r in recs] == GOLD["e2e.crop_scale"].tolist()
    # get_affine_transform solves cv2.getAffineTransform's system with numpy: its trans_inv can differ from cv2's in the last bits
    # (here by up to 3e-14), which moves a rare PIL sample point across a pixel boundary.  With cv2's matrices (stored in the
    # fixture) the images are bit-identical; with the sampler's own, all but a handful of pixels are.
    cv2_recs = [r._replace(trans=GOLD["e2e.trans"][i], trans_inv=GOLD["e2e.trans_inv"][i]) for i, r in enumerate(recs)]
    dev_imgs = [torch.from_numpy(im) for im in imgs]
    inputs, P2, targets, info = builder(dev_imgs, list(range(n)), cv2_recs)
    own = builder(dev_imgs, list(range(n)), recs)
    torch.cuda.synchronize()
    for i in range(n):
        want = normalize(GOLD["e2e.u8"][i])
        assert np.array_equal(inputs[i].cpu().numpy(), want), i
        assert (own[0][i].cpu().numpy() != want).any(0).mean() < 1e-3, i
    ol.assert_targets_match(_host({k: own[2][k] for k in ol.KEYS}), {k: GOLD[f"e2e.{k}"] for k in ol.KEYS}, "e2e, own trans")
    ol.assert_targets_match(_host({k: targets[k] for k in ol.KEYS}), {k: GOLD[f"e2e.{k}"] for k in ol.KEYS}, "e2e")
    np.testing.assert_array_equal(P2.cpu().numpy(), GOLD["e2e.P2"])
    np.testing.assert_array_equal(targets["img_size"].cpu().numpy(), GOLD["sizes"][:n])
    np.testing.assert_array_equal(info["img_id"].numpy(), GOLD["e2e.info_img_id"])
    np.testing.assert_array_equal(info["img_size"].numpy(), GOLD["e2e.info_img_size"])
    np.testing.assert_array_equal(info["bbox_downsample_ratio"].numpy(), GOLD["e2e.info_ratio"])


def test_criterion_on_device_targets_matches_the_reference_targets():
    """SetCriterion fed the device-built targets and fed the reference's collated targets: same losses and gradients within
    tests/test_criterion_gpu.py's tolerances (the inputs differ only in heading_res, by at most 1e-6)."""
    from monodetr_b200 import labels as lb
    from monodetr_b200.criterion import build_criterion
    from oracle import criterion as oc
    name = "all3"
    n = len(GOLD[f"{name}.seeds"])
    recs = [lb.AugRecord(tuple(GOLD["sizes"][i]), bool(GOLD[f"{name}.flip"][i]), float(GOLD[f"{name}.crop_scale"][i]),
                         GOLD[f"{name}.center"][i], GOLD[f"{name}.trans"][i], GOLD[f"{name}.trans_inv"][i]) for i in range(n)]
    dev_t = _encoder(name)(_bank(), list(range(n)), recs)
    ref_t = {k: torch.from_numpy(GOLD[f"{name}.{k}"]).cuda() for k in ol.KEYS}
    out, _ = oc.synthetic_case(11, n, 66)
    results = []
    for tg in (ref_t, dev_t):
        crit = build_criterion(CRIT_CFG).cuda().train(True)
        o = {k: v.cuda().requires_grad_(True) for k, v in out.items() if torch.is_tensor(v)}
        o["aux_outputs"] = [{k: v.cuda().requires_grad_(True) for k, v in a.items()} for a in out["aux_outputs"]]
        losses = crit(o, tg)
        total = sum(losses[k] * crit.weight_dict[k] for k in losses if k in crit.weight_dict)
        total.backward()
        torch.cuda.synchronize()
        grads = {k: v.grad.cpu().numpy() for k, v in o.items() if torch.is_tensor(v) and v.grad is not None}
        grads.update({f"aux{i}.{k}": v.grad.cpu().numpy() for i, a in enumerate(o["aux_outputs"]) for k, v in a.items()
                      if v.grad is not None})
        results.append(({k: float(v) for k, v in losses.items()}, float(total), grads))
    (lr, tr, gr), (ld, td, gd) = results
    assert sorted(lr) == sorted(ld) and sorted(gr) == sorted(gd) and gr
    for k in lr:
        np.testing.assert_allclose(ld[k], lr[k], rtol=2e-5, atol=1e-6, err_msg=k)
    np.testing.assert_allclose(td, tr, rtol=2e-5)
    for k in gr:
        np.testing.assert_allclose(gd[k], gr[k], rtol=2e-4, atol=1e-9 + 2e-5 * np.abs(gr[k]).max(), err_msg=k)


@pytest.mark.parametrize("case", ["index", "empty", "nan_scale"])
def test_out_of_range_inputs_are_rejected_before_launch(case):
    from monodetr_b200 import _lib
    from monodetr_b200 import labels as lb
    bank = _bank()
    recs = [lb.AugRecord(tuple(GOLD["sizes"][i]), False, 1.0, None, GOLD["val.trans"][i], GOLD["val.trans_inv"][i]) for i in range(3)]
    idx = [0, 1, 2]
    if case == "index":
        idx = [0, 1, len(bank)]
    elif case == "empty":
        idx, recs = [], []
    else:
        recs[2] = recs[2]._replace(crop_scale=float("inf"))
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        lb.TargetEncoder()(bank, idx, recs)
    assert _lib.launch_count() == n0
