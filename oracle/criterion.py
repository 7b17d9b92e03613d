"""CPU restatement (PyTorch autograd + scipy) of the reference's training criterion -- TEST INFRASTRUCTURE ONLY (imported by
tests/ and tools/gen_golden_criterion.py; the product path is monodetr_b200/csrc/criterion.cu behind monodetr_b200/criterion.py).

  prepare_targets   lib/helpers/trainer_helper.py:175-186
  hungarian_match   lib/models/monodetr/matcher.py:36-104          (scipy.optimize.linear_sum_assignment per image and group)
  set_criterion     lib/models/monodetr/monodetr.py:297-532        (loss_labels/cardinality/3dcenter/boxes/depths/dims/angles/depth_map,
                                                                    forward incl. the aux-output loop)
  ddn_loss          depth_predictor/ddn_loss/ddn_loss.py:43-127, balancer.py:21-81, focalloss.py:52-125
  sigmoid_focal_loss  lib/models/monodetr/dn_components.py:16-41;  box helpers utils/box_ops.py:20-72;  accuracy utils/misc.py:436-451

Pinned against the unmodified reference classes (HungarianMatcher + SetCriterion run on CPU through in-memory shims) by
tests/golden/criterion.npz -- tools/gen_golden_criterion.py, tests/test_oracle_criterion.py.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

KEYS = ("labels", "boxes", "depth", "size_3d", "heading_bin", "heading_res", "boxes_3d")
COST = dict(set_cost_class=2.0, set_cost_bbox=5.0, set_cost_giou=2.0, set_cost_3dcenter=10.0)     # configs/monodetr.yaml:86-89


def prepare_targets(padded):
    mask = padded["mask_2d"].bool()
    return [{k: padded[k][b][mask[b]] for k in KEYS} for b in range(mask.shape[0])]


def cxcylrtb_to_xyxy(x):
    cx, cy, l, r, t, b = x.unbind(-1)
    return torch.stack([cx - l, cy - t, cx + r, cy + b], -1)


def cxcywh_to_xyxy(x):
    cx, cy, w, h = x.unbind(-1)
    return torch.stack([cx - 0.5 * w, cy - 0.5 * h, cx + 0.5 * w, cy + 0.5 * h], -1)


def generalized_box_iou(a, b):
    area1 = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
    area2 = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    lt, rb = torch.max(a[:, None, :2], b[:, :2]), torch.min(a[:, None, 2:], b[:, 2:])
    wh = (rb - lt).clamp(min=0)
    inter = wh[..., 0] * wh[..., 1]
    union = area1[:, None] + area2 - inter
    iou = inter / union
    lt, rb = torch.min(a[:, None, :2], b[:, :2]), torch.max(a[:, None, 2:], b[:, 2:])
    wh = (rb - lt).clamp(min=0)
    area = wh[..., 0] * wh[..., 1]
    return iou - (area - union) / area


@torch.no_grad()
def cost_matrix(out, targets, cost=COST):
    bs, nq = out["pred_boxes"].shape[:2]
    prob = out["pred_logits"].flatten(0, 1).sigmoid()
    tgt_ids = torch.cat([t["labels"] for t in targets]).long()
    neg = 0.75 * (prob ** 2.0) * (-(1 - prob + 1e-8).log())
    pos = 0.25 * ((1 - prob) ** 2.0) * (-(prob + 1e-8).log())
    c_class = pos[:, tgt_ids] - neg[:, tgt_ids]
    ob = out["pred_boxes"].flatten(0, 1)
    tb = torch.cat([t["boxes_3d"] for t in targets])
    c_center = torch.cdist(ob[:, 0:2], tb[:, 0:2], p=1)
    c_bbox = torch.cdist(ob[:, 2:6], tb[:, 2:6], p=1)
    c_giou = -generalized_box_iou(cxcylrtb_to_xyxy(ob), cxcylrtb_to_xyxy(tb))
    C = cost["set_cost_bbox"] * c_bbox + cost["set_cost_3dcenter"] * c_center + cost["set_cost_class"] * c_class + cost["set_cost_giou"] * c_giou
    return C.view(bs, nq, -1)


@torch.no_grad()
def hungarian_match(out, targets, group_num, cost=COST):
    C = cost_matrix(out, targets, cost)
    nq = C.shape[1]
    sizes = [len(t["boxes"]) for t in targets]
    g = nq // group_num
    indices = None
    for gi, Cg in enumerate(C.split(g, dim=1)):
        ind = [linear_sum_assignment(c[i]) for i, c in enumerate(Cg.split(sizes, -1))]
        if gi == 0:
            indices = ind
        else:
            indices = [(np.concatenate([a[0], b[0] + g * gi]), np.concatenate([a[1], b[1]])) for a, b in zip(indices, ind)]
    return [(torch.as_tensor(i, dtype=torch.int64), torch.as_tensor(j, dtype=torch.int64)) for i, j in indices]


def sigmoid_focal_loss(inputs, targets, num_boxes, alpha=0.25, gamma=2):
    prob = inputs.sigmoid()
    ce = F.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
    p_t = prob * targets + (1 - prob) * (1 - targets)
    loss = ce * ((1 - p_t) ** gamma)
    loss = (alpha * targets + (1 - alpha) * (1 - targets)) * loss
    return loss.mean(1).sum() / num_boxes


def ddn_target(gt_boxes2d, num_gt_per_img, gt_center_depth, B, H, W, depth_min=1e-3, depth_max=60, num_bins=80):
    """(B, H, W) LID bin of every pixel and its foreground mask, formed in the dtype of the boxes and depths."""
    depth_maps = torch.zeros((B, H, W), dtype=gt_center_depth.dtype)
    gt_boxes2d = gt_boxes2d.clone()
    gt_boxes2d[:, :2] = torch.floor(gt_boxes2d[:, :2])
    gt_boxes2d[:, 2:] = torch.ceil(gt_boxes2d[:, 2:])
    boxes = gt_boxes2d.long().split(num_gt_per_img, dim=0)
    depths = gt_center_depth.split(num_gt_per_img, dim=0)
    fg = torch.zeros((B, H, W), dtype=torch.bool)
    for b in range(B):
        d, order = torch.sort(depths[b], dim=0, descending=True)
        bb = boxes[b][order]
        for n in range(bb.shape[0]):
            u1, v1, u2, v2 = bb[n]
            depth_maps[b, v1:v2, u1:u2] = d[n]
            fg[b, v1:v2, u1:u2] = True
    bin_size = 2 * (depth_max - depth_min) / (num_bins * (1 + num_bins))
    idx = -0.5 + 0.5 * torch.sqrt(1 + 8 * (depth_maps - depth_min) / bin_size)
    bad = (idx < 0) | (idx > num_bins) | (~torch.isfinite(idx))
    idx[bad] = num_bins
    return idx.type(torch.int64), fg


def ddn_loss(depth_logits, gt_boxes2d, num_gt_per_img, gt_center_depth, alpha=0.25, gamma=2.0, fg_weight=13, bg_weight=1,
             depth_min=1e-3, depth_max=60, num_bins=80, per_pixel=False):
    """The depth-map loss; with per_pixel, also the (B, H, W) weighted loss of every pixel.  The target bins are formed in the
    dtype of the boxes and depths (ddn_target), the focal loss in that of the logits."""
    B, _, H, W = depth_logits.shape
    target, fg = ddn_target(gt_boxes2d, num_gt_per_img, gt_center_depth, B, H, W, depth_min, depth_max, num_bins)
    soft, logsoft = F.softmax(depth_logits, dim=1), F.log_softmax(depth_logits, dim=1)
    onehot = torch.zeros_like(depth_logits).scatter_(1, target.unsqueeze(1), 1.0) + 1e-6
    focal = -alpha * torch.pow(-soft + 1.0, gamma) * logsoft
    loss = torch.einsum("bc...,bc...->b...", (onehot, focal))
    weights = fg_weight * fg + bg_weight * (~fg)
    loss = loss * weights
    npix = fg.sum() + (~fg).sum()
    total = loss[fg].sum() / npix + loss[~fg].sum() / npix
    return (total, loss) if per_pixel else total


def _src_idx(indices):
    return (torch.cat([torch.full_like(s, i) for i, (s, _) in enumerate(indices)]), torch.cat([s for s, _ in indices]))


def layer_losses(out, targets, indices, num_boxes, num_classes=3, focal_alpha=0.25, log=True, depth_map=True, map_scale=(80, 24),
                 corner_dtype=None):
    """corner_dtype: round the predicted box corners to this dtype (keeping their gradient), as a kernel in that precision
    forms them, so that GIoU's max / min and clamp take the same branches in a higher-precision run."""
    L = {}
    idx = _src_idx(indices)
    logits = out["pred_logits"]
    tco = torch.cat([t["labels"][J] for t, (_, J) in zip(targets, indices)])
    tc = torch.full(logits.shape[:2], num_classes, dtype=torch.int64)
    tc[idx] = tco.long()
    onehot = torch.zeros(logits.shape[0], logits.shape[1], logits.shape[2] + 1, dtype=logits.dtype).scatter_(2, tc.unsqueeze(-1), 1)[:, :, :-1]
    L["loss_ce"] = sigmoid_focal_loss(logits, onehot, num_boxes, alpha=focal_alpha, gamma=2) * logits.shape[1]
    if log:
        if tco.numel() == 0:
            L["class_error"] = torch.tensor(100.0)
        else:
            pred = logits[idx].argmax(-1)
            L["class_error"] = 100 - (pred == tco.long()).float().sum() * (100.0 / tco.numel())
    tb = torch.cat([t["boxes_3d"][i] for t, (_, i) in zip(targets, indices)], dim=0)
    sb = out["pred_boxes"][idx]
    L["loss_bbox"] = F.l1_loss(sb[:, 2:6], tb[:, 2:6], reduction="none").sum() / num_boxes
    sxy = cxcylrtb_to_xyxy(sb)
    if corner_dtype is not None:
        sxy = sxy + (sxy.to(corner_dtype).to(sxy.dtype) - sxy).detach()
    L["loss_giou"] = (1 - torch.diag(generalized_box_iou(sxy, cxcylrtb_to_xyxy(tb)))).sum() / num_boxes
    lens = torch.as_tensor([len(t["labels"]) for t in targets])
    card = (logits.argmax(-1) != logits.shape[-1] - 1).sum(1)
    L["cardinality_error"] = F.l1_loss(card.float(), lens.float())
    sd = out["pred_depth"][idx]
    td = torch.cat([t["depth"][i] for t, (_, i) in zip(targets, indices)], dim=0).reshape(-1)
    L["loss_depth"] = (1.4142 * torch.exp(-sd[:, 1]) * torch.abs(sd[:, 0] - td) + sd[:, 1]).sum() / num_boxes
    s3 = out["pred_3d_dim"][idx]
    t3 = torch.cat([t["size_3d"][i] for t, (_, i) in zip(targets, indices)], dim=0)
    dim_loss = torch.abs(s3 - t3) / t3.clone().detach()
    with torch.no_grad():
        comp = F.l1_loss(s3, t3) / dim_loss.mean()
    L["loss_dim"] = (dim_loss * comp).sum() / num_boxes
    ha = out["pred_angle"][idx].view(-1, 24)
    hb = torch.cat([t["heading_bin"][i] for t, (_, i) in zip(targets, indices)], dim=0).view(-1).long()
    hr = torch.cat([t["heading_res"][i] for t, (_, i) in zip(targets, indices)], dim=0).view(-1)
    cls_loss = F.cross_entropy(ha[:, 0:12], hb, reduction="none")
    oh = torch.zeros(hb.shape[0], 12, dtype=ha.dtype).scatter_(dim=1, index=hb.view(-1, 1), value=1)
    reg_loss = F.l1_loss(torch.sum(ha[:, 12:24] * oh, 1), hr, reduction="none")
    L["loss_angle"] = (cls_loss + reg_loss).sum() / num_boxes
    L["loss_center"] = F.l1_loss(sb[:, 0:2], tb[:, 0:2], reduction="none").sum() / num_boxes
    if depth_map:
        n = [len(t["boxes"]) for t in targets]
        sx, sy = map_scale
        b2 = torch.cat([t["boxes"] for t in targets], dim=0)
        boxes2d = cxcywh_to_xyxy(b2 * torch.tensor([sx, sy, sx, sy], dtype=b2.dtype))
        L["loss_depth_map"] = ddn_loss(out["pred_depth_map_logits"], boxes2d, n, torch.cat([t["depth"] for t in targets], dim=0).squeeze(dim=1))
    return L


def set_criterion(outputs, padded, training=True, group_num=11, world_size=1, cost=COST, **kw):
    """Returns (losses dict as SetCriterion.forward, list of matcher indices per decoder layer)."""
    targets = prepare_targets(padded)
    g = group_num if training else 1
    main = {k: v for k, v in outputs.items() if k != "aux_outputs"}
    indices = hungarian_match(main, targets, g, cost)
    num_boxes = max(float(sum(len(t["labels"]) for t in targets) * g) / world_size, 1.0)
    losses = layer_losses(main, targets, indices, num_boxes, **kw)
    all_idx = [indices]
    for i, aux in enumerate(outputs.get("aux_outputs", [])):
        ind = hungarian_match(aux, targets, g, cost)
        all_idx.append(ind)
        for k, v in layer_losses(aux, targets, ind, num_boxes, log=False, depth_map=False, **kw).items():
            losses[f"{k}_{i}"] = v
    return losses, all_idx


WEIGHTS = {"loss_ce": 2.0, "loss_bbox": 5.0, "loss_giou": 2.0, "loss_dim": 1.0, "loss_angle": 1.0, "loss_depth": 1.0, "loss_center": 10.0,
           "loss_depth_map": 1.0}                                                       # configs/monodetr.yaml:74-83


def weight_dict(dec_layers=3):
    w = dict(WEIGHTS)
    for i in range(dec_layers - 1):
        w.update({f"{k}_{i}": v for k, v in WEIGHTS.items()})
    return w


def synthetic_case(seed, B, Q, C=3, Gmax=50, H=24, W=80, n_aux=2, max_gt=12, empty_image=True):
    """Seeded head outputs with MonoDETR.forward's shapes and loader-style padded targets (kitti_dataset.py:166-330)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.rand(*s, generator=g)  # noqa: E731
    n = lambda *s: torch.randn(*s, generator=g)  # noqa: E731

    def heads():
        return {"pred_logits": n(B, Q, C) * 2 - 2, "pred_boxes": torch.cat([0.1 + 0.8 * r(B, Q, 2), 0.01 + 0.2 * r(B, Q, 4)], -1),
                "pred_3d_dim": 1.5 + 0.5 * n(B, Q, 3), "pred_depth": torch.stack([3 + 50 * r(B, Q), n(B, Q)], -1), "pred_angle": n(B, Q, 24)}
    out = heads()
    out["pred_depth_map_logits"] = n(B, 81, H, W)
    out["aux_outputs"] = [heads() for _ in range(n_aux)]
    counts = torch.randint(1, max_gt + 1, (B,), generator=g)
    if empty_image and B > 1:
        counts[1] = 0
    mask = torch.zeros(B, Gmax, dtype=torch.bool)
    for b in range(B):
        sel = torch.randperm(Gmax, generator=g)[:counts[b]]          # valid rows are NOT a prefix (the loader filters objects)
        mask[b, sel] = True
    ctr = 0.05 + 0.9 * r(B, Gmax, 2)
    lrtb = 0.01 + 0.25 * r(B, Gmax, 4)
    boxes3d = torch.cat([ctr, lrtb], -1)
    x0, y0, x1, y1 = ctr[..., 0] - lrtb[..., 0], ctr[..., 1] - lrtb[..., 2], ctr[..., 0] + lrtb[..., 1], ctr[..., 1] + lrtb[..., 3]
    boxes = torch.stack([(x0 + x1) / 2, (y0 + y1) / 2, x1 - x0, y1 - y0], -1)            # may leave [0, 1]: exercises the slice wrap
    padded = {"mask_2d": mask, "labels": torch.randint(0, C, (B, Gmax), generator=g).to(torch.int8), "boxes": boxes, "boxes_3d": boxes3d,
              "depth": 2 + 60 * r(B, Gmax, 1), "size_3d": 0.5 + 3 * r(B, Gmax, 3),
              "heading_bin": torch.randint(0, 12, (B, Gmax, 1), generator=g), "heading_res": (r(B, Gmax, 1) - 0.5) * (math.pi / 6)}
    return out, padded


# ---- golden-vector storage of the criterion's gradients (tests/golden/criterion.npz) ----------------------------------
GOLDEN_GRAD_MAX_ELEMS = 16384


def store_golden_grad(out, key, g):
    """A gradient of at most GOLDEN_GRAD_MAX_ELEMS elements is stored whole under `key`; a larger one (the depth-map logits)
    as its max |g| (`key.absmax`) and the values (`key.val`) at a fixed, seeded sample of flat positions (`key.idx`)."""
    if g.size <= GOLDEN_GRAD_MAX_ELEMS:
        out[key] = g
        return
    rng = np.random.default_rng(sum(key.encode()))
    idx = np.sort(rng.choice(g.size, GOLDEN_GRAD_MAX_ELEMS, replace=False)).astype(np.int64)
    out[key + ".idx"] = idx
    out[key + ".val"] = g.reshape(-1)[idx].astype(np.float32)
    out[key + ".absmax"] = np.asarray(np.abs(g).max(), np.float64)


def golden_grad(gold, key, got):
    """(computed, golden, max |golden|) for a gradient stored by store_golden_grad; `got` is the full computed array."""
    if key in gold.files:
        g = gold[key]
        return got, g, float(np.abs(g).max())
    idx = gold[key + ".idx"]
    return got.reshape(-1)[idx], gold[key + ".val"], float(gold[key + ".absmax"])
