"""The device criterion (csrc/criterion.cu) at its edges, against scipy and a float64 run of oracle/criterion.py.

  matcher     inputs that tie exactly by construction (duplicated queries, duplicated targets, costs on a dyadic grid with the
              class and GIoU weights at zero, so every cost is exact in fp32): scipy's assignment, square and transposed
  depth map   boxes on pixel boundaries (column / row 0, the right / bottom edges, one ulp either side of an integer, negative
              starts, boxes outside the map, overlaps of equal depth) and depths on LID bin boundaries: every pixel's
              foreground mask and bin exactly, its loss and logit gradients within the float64 bounds
  losses      saturated class logits, boxes equal / sharing edges / touching / nested / disjoint, exact-equal centres,
              depths, dimensions and heading residuals, log-variance +-30, peaked and flat softmax logits: every loss and
              gradient element within the bounds of tests/criterion_error_model.py, with the device's matching fed to the
              reference; eval, training and the reproducible mode
"""
import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

import criterion_error_model as em
from oracle import criterion as oc

pytestmark = pytest.mark.gpu
F64 = torch.float64
CFG = {"num_classes": 3, "cls_loss_coef": 2, "focal_alpha": 0.25, "bbox_loss_coef": 5, "giou_loss_coef": 2, "3dcenter_loss_coef": 10,
       "dim_loss_coef": 1, "angle_loss_coef": 1, "depth_loss_coef": 1, "depth_map_loss_coef": 1, "set_cost_class": 2, "set_cost_bbox": 5,
       "set_cost_giou": 2, "set_cost_3dcenter": 10, "aux_loss": True, "dec_layers": 3, "num_queries": 300}
WORST = {}


def _record(name, ratio):
    WORST[name] = max(WORST.get(name, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    print("criterion error model, worst ratios (|got - ref64| / (u * mag)):")
    for k, v in sorted(WORST.items()):
        print(f"  {k}: {v:.3f}")


def _prepare(mask):
    from monodetr_b200 import _lib
    B, G = mask.shape
    tlist, count = torch.empty(B, G, dtype=torch.int32, device="cuda"), torch.empty(B, dtype=torch.int32, device="cuda")
    total = torch.empty(1, dtype=torch.float32, device="cuda")
    _lib.call("mdb_criterion_prepare", mask.to(torch.uint8).cuda().contiguous(), B, G, tlist, count, total)
    return tlist, count, total


# ---- matcher: scipy's assignment under exact ties ----------------------------------------------------------------------------
def _tie_case(seed, L, B, Q, C, group, G, counts, dup_q, dup_t):
    g = np.random.default_rng(seed)
    ctr = g.choice([0.25, 0.375, 0.5, 0.625], (L, B, Q, 2))
    lrtb = g.choice([0.0625, 0.125, 0.25], (L, B, Q, 4))
    boxes = np.concatenate([ctr, lrtb], -1).astype(np.float32)
    if dup_q:                                          # duplicated query rows: identical boxes and logits
        src = g.integers(0, Q, Q // 2)
        boxes[:, :, g.integers(0, Q, Q // 2)] = boxes[:, :, src]
    logits = g.standard_normal((L, B, Q, C)).astype(np.float32)
    tb = np.concatenate([g.choice([0.25, 0.5, 0.75], (B, G, 2)), g.choice([0.0625, 0.125, 0.25], (B, G, 4))], -1).astype(np.float32)
    if dup_t:                                          # duplicated target rows
        src = g.integers(0, G, G // 2)
        tb[:, g.integers(0, G, G // 2)] = tb[:, src]
    labels = g.integers(0, C, (B, G)).astype(np.int32)
    mask = np.zeros((B, G), bool)
    for b, n in enumerate(counts):
        mask[b, np.sort(g.choice(G, n, replace=False))] = True
    return logits, boxes, tb, labels, mask


def _scipy_tie_match(boxes, tb, labels, mask, group, C):
    """(L, B, group, G) expected match and (L, B, Q) expected target class, with costs 5 * L1(lrtb) + 10 * L1(centre)."""
    L, B, Q, _ = boxes.shape
    G = mask.shape[1]
    nq = Q // group
    match = np.full((L, B, group, G), -1)
    tclass = np.full((L, B, Q), C)
    for l in range(L):
        for b in range(B):
            valid = np.nonzero(mask[b])[0]
            if not len(valid):
                continue
            for gi in range(group):
                q = boxes[l, b, gi * nq:(gi + 1) * nq].astype(np.float64)
                t = tb[b, valid].astype(np.float64)
                cost = 5 * np.abs(q[:, None, 2:] - t[None, :, 2:]).sum(-1) + 10 * np.abs(q[:, None, :2] - t[None, :, :2]).sum(-1)
                assert np.array_equal(cost.astype(np.float32).astype(np.float64), cost)      # exact in fp32: scipy sees the kernel's costs
                qi, tj = linear_sum_assignment(cost)
                match[l, b, gi, tj] = gi * nq + qi
                tclass[l, b, gi * nq + qi] = labels[b, valid[tj]]
    return match, tclass


@pytest.mark.parametrize("name,L,B,Q,group,G,counts,dup_q,dup_t", [
    ("eval_square_50", 2, 2, 50, 1, 64, [50, 50], True, True),
    ("square_64", 1, 2, 64, 1, 64, [64, 64], True, False),
    ("square_64_dup_targets", 1, 2, 64, 1, 64, [64, 64], False, True),
    ("train_more_targets", 2, 3, 55, 11, 16, [12, 7, 5], True, True),      # 5 queries per group: nt > nq
    ("train_groups", 2, 2, 550, 11, 32, [20, 50 // 2], True, True),
    ("queries_300_targets_64", 1, 2, 300, 1, 64, [64, 40], True, True),
])
def test_matcher_ties_match_scipy(name, L, B, Q, group, G, counts, dup_q, dup_t):
    from monodetr_b200 import _lib
    C = 3
    logits, boxes, tb, labels, mask = _tie_case(sum(map(ord, name)), L, B, Q, C, group, G, counts, dup_q, dup_t)
    tlist, count, _ = _prepare(torch.from_numpy(mask))
    match = torch.empty(L, B, group, G, dtype=torch.int32, device="cuda")
    tclass = torch.empty(L, B, Q, dtype=torch.int32, device="cuda")
    lg = [torch.from_numpy(logits[l]).cuda() for l in range(L)]
    bx = [torch.from_numpy(boxes[l]).cuda() for l in range(L)]
    _lib.call("mdb_criterion_match_f32", L, lg, bx, torch.from_numpy(labels).cuda(), torch.from_numpy(tb).cuda(), tlist, count, B, Q, C,
              group, G, 0.0, 10.0, 5.0, 0.0, match, tclass)
    torch.cuda.synchronize()
    want_m, want_c = _scipy_tie_match(boxes, tb, labels, mask, group, C)
    got_m = match.cpu().numpy()
    for b in range(B):                                 # both indexed by the position among the image's valid targets
        assert np.array_equal(got_m[:, b], want_m[:, b]), (name, b)
    assert np.array_equal(tclass.cpu().numpy(), want_c), name


# ---- depth map: edges on pixel boundaries, bins on their boundaries -----------------------------------------------------------
IMG_W, IMG_H, MAP_W, MAP_H, NB = 1280, 384, 80, 24, 80
DMIN, DMAX = 1e-3, 60.0


def _px_box(x0, y0, x1, y1):
    """Integer image-pixel corners -> normalised (cx, cy, w, h) formed in fp32 like the loader's."""
    f = np.float32
    return [f(f(f(x0) + f(x1)) / f(2)) / f(IMG_W), f(f(f(y0) + f(y1)) / f(2)) / f(IMG_H), f(f(x1) - f(x0)) / f(IMG_W),
            f(f(y1) - f(y0)) / f(IMG_H)]


def _depth_map_case(seed):
    g = np.random.default_rng(seed)
    f = np.float32
    bin_size = 2 * (DMAX - DMIN) / (NB * (1 + NB))
    boxes = []
    for x0 in list(range(0, 1280, 97)) + [0] * 6:                     # column 0 and integer corners anywhere
        w = int(g.integers(1, min(320, 1280 - x0) + 1))
        y0 = int(g.choice([0, int(g.integers(0, 383))]))
        boxes.append(_px_box(x0, y0, x0 + w, y0 + int(g.integers(1, min(96, 384 - y0) + 1))))
    for y0 in [0] * 6 + list(range(0, 384, 53)):                      # row 0
        x0 = int(g.integers(0, 1279))
        boxes.append(_px_box(x0, y0, x0 + int(g.integers(1, min(320, 1280 - x0) + 1)), y0 + int(g.integers(1, min(96, 384 - y0) + 1))))
    for _ in range(8):                                                  # right / bottom edges
        x0, y0 = int(g.integers(960, 1279)), int(g.integers(288, 383))
        boxes.append(_px_box(x0, y0, 1280, 384))
    for k in range(16):                                                 # map-space edges one ulp either side of an integer
        wm, hm = f(2 ** int(g.integers(0, 4))), f(2 ** int(g.integers(0, 3)))
        cx, cy = f((f(int(g.integers(0, 70))) + wm / 2) / MAP_W), f((f(int(g.integers(0, 20))) + hm / 2) / MAP_H)
        d = np.inf if k % 2 else -np.inf
        for _ in range(int(g.integers(1, 3))):
            cx, cy = np.nextafter(cx, f(d)), np.nextafter(cy, f(-d))
        boxes.append([cx, cy, f(wm / MAP_W), f(hm / MAP_H)])
    boxes += [[f(0.02), f(0.5), f(0.2), f(0.3)], [f(0.5), f(-0.05), f(0.3), f(0.4)],     # negative starts: the slice wrap
              [f(-0.3), f(0.5), f(0.1), f(0.2)], [f(1.5), f(0.5), f(0.2), f(0.2)],        # entirely outside the map
              [f(0.5), f(1.4), f(0.2), f(0.3)], [f(-0.2), f(-0.2), f(0.1), f(0.1)]]
    n = len(boxes)
    ks = g.integers(0, NB + 1, n)
    depth = np.array([f(DMIN + bin_size * k * (k + 1) / 2) for k in ks], np.float32)          # on LID bin boundaries
    depth[::7] = f(DMAX)
    depth[3::7] = f(75.0)
    depth[5::7] = f(DMIN / 2)
    depth[6::11] = g.uniform(2, 59, len(depth[6::11]))
    boxes = np.array(boxes, np.float32)
    ov = g.choice(n, 6, replace=False)                                  # overlapping boxes of equal depth
    boxes[ov[3:]] = boxes[ov[:3]] + np.array([0.01, 0.02, 0.0, 0.0], np.float32)
    depth[ov[3:]] = depth[ov[:3]]
    return boxes, depth


def _depth_map_inputs(seed, B=16, G=24, logit_kind="mixed"):
    """Spread the case's boxes over B images of at most G targets; logits NCHW."""
    boxes, depth = _depth_map_case(seed)
    g = np.random.default_rng(seed + 1)
    perm = g.permutation(len(boxes))
    b2 = np.zeros((B, G, 4), np.float32)
    dd = np.ones((B, G), np.float32)
    mask = np.zeros((B, G), bool)
    for e, i in enumerate(perm):
        b, slot = e % B, e // B
        if slot >= G:
            break
        b2[b, slot], dd[b, slot], mask[b, slot] = boxes[i], depth[i], True
    mask[:, G - 1] = False                                              # an invalid row in every image
    c = torch.arange(NB + 1, dtype=torch.float32).view(1, -1, 1, 1)
    z = 0.05 * c + 0.01 * torch.rand(B, NB + 1, MAP_H, MAP_W, generator=torch.Generator().manual_seed(seed))
    if logit_kind == "mixed":                                           # peaked (+-50) and flat pixels too
        z[:, :, :, ::5] = 0.0
        z[:, 7, :, 1::5] = 50.0
        z[:, 11, :, 2::5] = -50.0
    return b2, dd, mask, z


def _run_depth_map(b2, dd, mask, z, gw=1.0):
    from monodetr_b200 import _lib
    B, G = mask.shape
    tlist, count, _ = _prepare(torch.from_numpy(mask))
    zc = z.contiguous().cuda()
    D, H, W = z.shape[1:]
    pix = torch.empty(B * H * W, dtype=torch.float32, device="cuda")
    dz = torch.empty_like(zc)
    args = (zc, D * H * W, 1, H * W, torch.from_numpy(b2).cuda(), torch.from_numpy(dd).cuda(), tlist, count, B, H, W, NB, G,
            float(MAP_W), float(MAP_H), DMIN, DMAX, 0.25, 13.0, 1.0)
    _lib.call("mdb_criterion_depth_map_f32", *args, pix, None, None)
    _lib.call("mdb_criterion_depth_map_f32", *args, None, torch.tensor([gw], device="cuda"), dz)
    torch.cuda.synchronize()
    return pix.view(B, H, W).cpu(), dz.cpu()


@pytest.mark.parametrize("seed,logit_kind", [(1, "mixed"), (2, "ramp"), (3, "mixed")])
def test_depth_map_edges(seed, logit_kind):
    b2, dd, mask, z = _depth_map_inputs(seed, logit_kind=logit_kind)
    B = mask.shape[0]
    gw = 0.75
    pix, dz = _run_depth_map(b2, dd, mask, z, gw)
    n = [int(m.sum()) for m in mask]
    boxes = torch.from_numpy(b2[mask])
    xyxy = oc.cxcywh_to_xyxy(boxes * torch.tensor([MAP_W, MAP_H, MAP_W, MAP_H], dtype=torch.float32))
    depth = torch.from_numpy(dd[mask])
    target, fg = oc.ddn_target(xyxy, n, depth, B, MAP_H, MAP_W)
    z64 = z.to(F64).requires_grad_(True)
    total, ref_pix = oc.ddn_loss(z64, xyxy, n, depth, per_pixel=True)
    (total * gw).backward()
    pix_mag, dz_mag, wgt = em.depth_map_mags(z64.detach(), target, fg)
    # mask and bin: the kernel's pixel loss must be nearest to the loss of the oracle's (foreground, bin), of all 2 x 81
    p = torch.softmax(z64.detach(), 1)
    fcls = -(1 - p) ** 2 * torch.log_softmax(z64.detach(), 1)              # per class, unweighted
    cand = 0.25 * (fcls + 1e-6 * fcls.sum(1, keepdim=True))                 # (B, 81, H, W): target bin = c
    cand = torch.cat([cand * 13.0, cand * 1.0], 1)                          # fg then bg
    got_key = (cand - pix.to(F64).unsqueeze(1)).abs().argmin(1)
    want_key = torch.where(fg, target, target + NB + 1)
    flat = z.amax(1) == z.amin(1)                                           # every bin has the same loss there: the mask only
    bad = torch.where(flat, (got_key <= NB) != fg, got_key != want_key).nonzero()
    assert not len(bad), f"{len(bad)} pixels with another mask / bin, first {bad[:5].tolist()}"
    assert int(fg.sum()) > 0 and int((~fg).sum()) > 0 and len(torch.unique(target[fg])) > 5
    _record("depth-map pixel", em.assert_rel("depth-map pixel loss", pix, ref_pix.detach(), pix_mag, em.C_PIX))
    scale = 0.25 * gw * wgt.unsqueeze(1) / pix.numel()
    _record("depth-map dlogits", em.assert_rel("depth-map dlogits", dz, z64.grad, scale * dz_mag, em.C_DMAP))


# ---- every loss and gradient against the float64 reference --------------------------------------------------------------------
def _edge_case(seed, B, Q, group, n_aux=2, G=16):
    out, padded = oc.synthetic_case(seed, B, Q, Gmax=G, n_aux=n_aux, max_gt=10)
    g = torch.Generator().manual_seed(seed + 7)
    nq = Q // group
    sat = torch.tensor([-100.0, -60.0, -20.0, 20.0, 60.0, 100.0])
    padded["boxes_3d"] = torch.round(padded["boxes_3d"] * 1024) / 1024        # dyadic: shared and touching edges are exact
    tb = padded["boxes_3d"]
    mask = padded["mask_2d"]
    for d in [out] + out["aux_outputs"]:
        lg, bx, dm, dp, an = d["pred_logits"], d["pred_boxes"], d["pred_3d_dim"], d["pred_depth"], d["pred_angle"]
        lg.view(-1)[::3] = sat[torch.randint(0, 6, (lg.numel() // 3 + 1,), generator=g)][:lg.view(-1)[::3].numel()]
        for b in range(B):
            valid = torch.nonzero(mask[b]).flatten()
            for gi in range(group):
                for j, t in enumerate(valid.tolist()):
                    q = gi * nq + j
                    if q >= (gi + 1) * nq:
                        break
                    T = tb[b, t].clone()
                    k = (j + gi) % 7
                    P = T.clone()
                    if k == 1:
                        P[3] = T[3] * 0.5                       # shares x0, y0, y1 (one side moved)
                    elif k == 2:
                        P[3], P[5] = T[3] * 0.5, T[5] * 0.5     # shares x0 and y0
                    elif k == 3:
                        P[0] = T[0] + T[3] + T[2]               # touching: its x0 == the target's x1 (iw == 0)
                    elif k == 4:
                        P[0] = T[0] + 0.5 + T[3] + T[2]         # disjoint
                    elif k == 5:
                        P[2:] = T[2:] * 0.5                     # nested
                    elif k == 6:
                        P[:2] = T[:2]
                        P[2:] = T[2:] * 1.5                     # same centre, larger
                    bx[b, q] = P
                    lg[b, q, int(padded["labels"][b, t])] = float(sat[3 + (j % 3)])
                    dp[b, q, 0] = padded["depth"][b, t, 0] if j % 2 == 0 else dp[b, q, 0]
                    dp[b, q, 1] = [30.0, -30.0, 0.5][j % 3]
                    if j % 3 == 0:
                        dm[b, q, 0] = padded["size_3d"][b, t, 0]
                    hb = int(padded["heading_bin"][b, t, 0])
                    if j % 2 == 0:
                        an[b, q, 12 + hb] = padded["heading_res"][b, t, 0]
                    if j % 4 == 1:
                        an[b, q, :12] = 0.0                     # flat
                    elif j % 4 == 2:
                        an[b, q, :12] = -50.0
                        an[b, q, hb] = 50.0                     # peaked at the bin
                    elif j % 4 == 3:
                        an[b, q, :12] = -50.0
                        an[b, q, (hb + 1) % 12] = 50.0          # peaked elsewhere
    dml = out["pred_depth_map_logits"]
    dml[:, :, :, ::4] = 0.0
    dml[:, 5, :, 1::4] = 50.0
    dml[:, 9, :, 2::4] = -50.0
    return out, padded


def _indices(m, mask, l):
    res = []
    for b in range(m.shape[1]):
        n = int(mask[b].sum())
        src, tgt = [], []
        for gi in range(m.shape[2]):
            for j in range(n):
                if m[l, b, gi, j] >= 0:
                    src.append(int(m[l, b, gi, j]))
                    tgt.append(j)
        res.append((torch.tensor(src, dtype=torch.int64), torch.tensor(tgt, dtype=torch.int64)))
    return res


def _check_against_f64(out, padded, training, tag):
    from monodetr_b200.criterion import build_criterion
    crit = build_criterion(CFG).cuda().train(training)
    keys = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle")
    o = {k: out[k].cuda().requires_grad_(True) for k in keys + ("pred_depth_map_logits",)}
    o["aux_outputs"] = [{k: a[k].cuda().requires_grad_(True) for k in keys} for a in out["aux_outputs"]]
    losses = crit(o, {k: v.cuda() for k, v in padded.items()})
    sum(losses[k] * crit.weight_dict[k] for k in losses if k in crit.weight_dict).backward()
    torch.cuda.synchronize()
    m = crit.last_indices.cpu().numpy()
    targets = oc.prepare_targets(padded)
    group = 11 if training else 1
    nb = max(float(sum(len(t["labels"]) for t in targets) * group), 1.0)
    w = oc.weight_dict()
    layers_dev = [o] + o["aux_outputs"]
    layers_src = [out] + out["aux_outputs"]
    for l, (dv, src) in enumerate(zip(layers_dev, layers_src)):
        suffix = "" if l == 0 else f"_{l - 1}"
        r = {k: src[k].to(F64).requires_grad_(True) for k in keys + (("pred_depth_map_logits",) if l == 0 else ())}
        ind = _indices(m, padded["mask_2d"], l)
        ref = oc.layer_losses(r, targets, ind, nb, log=l == 0, depth_map=l == 0, corner_dtype=torch.float32)
        sum(ref[k] * w[k + suffix] for k in ref if k + suffix in w).backward()
        # ---- loss scalars
        idx = oc._src_idx(ind)
        sb, tb = r["pred_boxes"].detach()[idx], torch.cat([t["boxes_3d"][j] for t, (_, j) in zip(targets, ind)]).to(F64)
        tc = torch.full(src["pred_logits"].shape[:2], 3, dtype=torch.int64)
        tc[idx] = torch.cat([t["labels"][j] for t, (_, j) in zip(targets, ind)]).long()
        onehot = torch.nn.functional.one_hot(tc, 4)[..., :3]
        fl_loss, fl_grad = em.focal_mags(src["pred_logits"], onehot)
        gi_loss, gi_grad = em.giou_mags(sb.float(), tb.float())
        sd = r["pred_depth"].detach()[idx]
        td = torch.cat([t["depth"][j] for t, (_, j) in zip(targets, ind)]).to(F64).reshape(-1)
        ev = 1.4142 * torch.exp(-sd[:, 1])
        s3 = r["pred_3d_dim"].detach()[idx]
        t3 = torch.cat([t["size_3d"][j] for t, (_, j) in zip(targets, ind)]).to(F64)
        ha = r["pred_angle"].detach()[idx]
        hb = torch.cat([t["heading_bin"][j] for t, (_, j) in zip(targets, ind)]).view(-1).long()
        hr = torch.cat([t["heading_res"][j] for t, (_, j) in zip(targets, ind)]).view(-1).to(F64)
        ce_mag, ce_grad = em.softmax_mags(ha[:, :12], hb)
        res = ha[:, 12:].gather(1, hb[:, None]).squeeze(1)
        mags = {"loss_ce": fl_loss.sum(), "loss_bbox": em.U32 * (sb[:, 2:] - tb[:, 2:]).abs().sum(),
                "loss_giou": gi_loss.sum(), "loss_depth": em.U32 * (ev * (sd[:, 0] - td).abs() + sd[:, 1].abs()).sum(),
                "loss_dim": em.U32 * (s3 - t3).abs().sum(), "loss_angle": (ce_mag + em.U32 * (res.abs() + hr.abs())).sum(),
                "loss_center": em.U32 * (sb[:, :2] - tb[:, :2]).abs().sum()}
        for k, mg in mags.items():
            _record("loss scalars", em.assert_rel(f"{tag} {k}{suffix}", losses[k + suffix].detach().cpu().reshape(1),
                                                  ref[k].detach().reshape(1), (mg / nb).reshape(1), em.C_LOSS))
        for k in ("cardinality_error", "class_error"):
            if k in ref:
                assert float(losses[k + suffix]) == pytest.approx(float(ref[k]), abs=1e-4), (tag, k, l)
        # ---- gradients
        W = lambda k: w[k + suffix] / nb  # noqa: E731
        g_log = fl_grad * W("loss_ce")
        g_box = torch.zeros(sb.shape[0], 6, dtype=F64)
        g_box[:, :2] += em.U32 * W("loss_center")
        g_box[:, 2:] += em.U32 * W("loss_bbox")
        g_box += gi_grad * W("loss_giou")
        g_dep = torch.stack([ev, 1 + ev * (sd[:, 0] - td).abs()], -1) * W("loss_depth") * em.U32
        with torch.no_grad():
            comp = float(torch.nn.functional.l1_loss(s3, t3) / ((s3 - t3).abs() / t3).mean()) if len(t3) else 0.0
        g_dim = comp / t3 * W("loss_dim") * em.U32
        g_ang = torch.cat([ce_grad, em.U32 * torch.nn.functional.one_hot(hb, 12).to(F64)], -1) * W("loss_angle")
        for k, gm, c in (("pred_boxes", g_box, em.C_BOX), ("pred_depth", g_dep, em.C_DEPTH), ("pred_3d_dim", g_dim, em.C_DIM),
                         ("pred_angle", g_ang, em.C_ANGLE)):
            full = torch.zeros(r[k].shape, dtype=F64)
            full[idx] = gm
            _record(k, em.assert_rel(f"{tag} d{k}{suffix}", dv[k].grad.cpu(), r[k].grad, full, c))
        _record("pred_logits", em.assert_rel(f"{tag} dpred_logits{suffix}", dv["pred_logits"].grad.cpu(), r["pred_logits"].grad, g_log,
                                             em.C_LOGITS))
        if l == 0:
            n = [len(t["boxes"]) for t in targets]
            b2 = torch.cat([t["boxes"] for t in targets])
            xyxy = oc.cxcywh_to_xyxy(b2 * torch.tensor([80, 24, 80, 24], dtype=torch.float32))
            depth = torch.cat([t["depth"] for t in targets]).squeeze(1)
            z = r["pred_depth_map_logits"]
            target, fg = oc.ddn_target(xyxy, n, depth, z.shape[0], z.shape[2], z.shape[3])
            pix_mag, dz_mag, wgt = em.depth_map_mags(z.detach(), target, fg)
            npix = fg.numel()
            _record("loss scalars", em.assert_rel(f"{tag} loss_depth_map", losses["loss_depth_map"].detach().cpu().reshape(1),
                                                  ref["loss_depth_map"].detach().reshape(1), (pix_mag.sum() / npix).reshape(1), em.C_LOSS))
            scale = 0.25 * w["loss_depth_map"] * wgt.unsqueeze(1) / npix
            _record("depth-map dlogits", em.assert_rel(f"{tag} dpred_depth_map_logits", dv["pred_depth_map_logits"].grad.cpu(), z.grad,
                                                       scale * dz_mag, em.C_DMAP))


@pytest.mark.parametrize("seed,B,Q,training", [(61, 3, 50, False), (62, 4, 550, True), (63, 2, 300, False)])
def test_losses_and_gradients_within_f64_bounds(seed, B, Q, training):
    out, padded = _edge_case(seed, B, Q, 11 if training else 1)
    _check_against_f64(out, padded, training, f"seed {seed}")


def test_reproducible_mode_within_f64_bounds():
    import monodetr_b200
    prev = monodetr_b200.set_deterministic(True)
    try:
        out, padded = _edge_case(64, 3, 550, 11)
        _check_against_f64(out, padded, True, "reproducible")
    finally:
        monodetr_b200.set_deterministic(prev)
