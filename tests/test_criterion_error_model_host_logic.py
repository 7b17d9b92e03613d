"""The bounds of tests/criterion_error_model.py are sharp: an fp32 emulation of the kernels' formulas (csrc/criterion.cu) fits
them, and a plausible slip in the same emulation exceeds them -- a dropped 1/2 on GIoU's max / min ties, an unstabilised
log(1 + e^-x), a missing (1 - p) factor in the focal gradient."""
import torch

import criterion_error_model as em
from oracle import criterion as oc

F64 = torch.float64


def _ratio(got, ref, mag):
    got = got.to(F64)
    if not bool(torch.isfinite(got).all()):
        return float("inf")
    err = (got - ref).abs()
    pos = mag > 0
    if not bool((err[~pos] == 0).all()):
        return float("inf")
    return float((err[pos] / mag[pos]).max())


def _focal_case():
    x = torch.tensor([-100.0, -60.0, -20.0, -3.0, -0.5, 0.0, 0.7, 2.5, 20.0, 60.0, 100.0])
    x = torch.cat([x, torch.randn(200, generator=torch.Generator().manual_seed(0)) * 4]).view(1, -1, 1).repeat(1, 1, 2)
    t = torch.zeros_like(x)
    t[..., 1] = 1.0
    return x.reshape(1, -1, 1), t.reshape(1, -1, 1)


def _focal_grad_fp32(x, t, alpha=0.25, stable=True, one_minus_p=True):
    """The kernel's focal gradient (crit_losses_bwd_kernel), in fp32, without g_ce / num_boxes."""
    prob = torch.sigmoid(x)
    bce = torch.clamp(x, min=0) - x * t + torch.log1p(torch.exp(-x.abs())) if stable else -x * t + torch.log(1 + torch.exp(x))
    pt = prob * t + (1 - prob) * (1 - t)
    at = alpha * t + (1 - alpha) * (1 - t)
    om = 1 - pt
    q = (1 - prob) if one_minus_p else torch.ones_like(prob)
    return at * (om * om * (prob - t) - 2 * bce * om * prob * q * (2 * t - 1))


def _focal_ref(x, t):
    x64 = x.to(F64).requires_grad_(True)
    (oc.sigmoid_focal_loss(x64, t.to(F64), 1.0) * x.shape[1]).backward()
    return x64.grad


def test_focal_gradient_bound_is_sharp():
    x, t = _focal_case()
    ref = _focal_ref(x, t)
    _, mag = em.focal_mags(x, t)
    assert _ratio(_focal_grad_fp32(x, t), ref, mag) <= em.C_LOGITS
    assert _ratio(_focal_grad_fp32(x, t, stable=False), ref, mag) > em.C_LOGITS             # log(1 + e^-x) overflows
    assert _ratio(_focal_grad_fp32(x, t, one_minus_p=False), ref, mag) > em.C_LOGITS


def _giou_grad_fp32(sb, tb, half=0.5):
    """d(1 - giou) / d(cx, cy, l, r, t, b) as the kernel forms it, in fp32."""
    x0, y0, x1, y1 = sb[:, 0] - sb[:, 2], sb[:, 1] - sb[:, 4], sb[:, 0] + sb[:, 3], sb[:, 1] + sb[:, 5]
    X0, Y0, X1, Y1 = tb[:, 0] - tb[:, 2], tb[:, 1] - tb[:, 4], tb[:, 0] + tb[:, 3], tb[:, 1] + tb[:, 5]
    w, h = x1 - x0, y1 - y0
    area1, area2 = w * h, (X1 - X0) * (Y1 - Y0)
    iwr, ihr = torch.minimum(x1, X1) - torch.maximum(x0, X0), torch.minimum(y1, Y1) - torch.maximum(y0, Y0)
    iw, ih = iwr.clamp(min=0), ihr.clamp(min=0)
    inter = iw * ih
    uni = area1 + area2 - inter
    cwr, chr_ = torch.maximum(x1, X1) - torch.minimum(x0, X0), torch.maximum(y1, Y1) - torch.minimum(y0, Y0)
    cw, ch = cwr.clamp(min=0), chr_.clamp(min=0)
    areac = cw * ch
    liv, lih, lcv, lch = ((v >= 0).float() for v in (iwr, ihr, cwr, chr_))

    def sel(gt, eq, val):
        return torch.where(gt, val, torch.where(eq, half * val, torch.zeros_like(val)))
    di = [-sel(x0 > X0, x0 == X0, ih * liv), -sel(y0 > Y0, y0 == Y0, iw * lih), sel(x1 < X1, x1 == X1, ih * liv),
          sel(y1 < Y1, y1 == Y1, iw * lih)]
    dc = [-sel(x0 < X0, x0 == X0, ch * lcv), -sel(y0 < Y0, y0 == Y0, cw * lch), sel(x1 > X1, x1 == X1, ch * lcv),
          sel(y1 > Y1, y1 == Y1, cw * lch)]
    da = [-h, -w, h, w]
    dx = []
    for k in range(4):
        du = da[k] - di[k]
        dx.append(-((di[k] * uni - inter * du) / (uni * uni) + (du * areac - uni * dc[k]) / (areac * areac)))
    return torch.stack([dx[0] + dx[2], dx[1] + dx[3], -dx[0], dx[2], -dx[1], dx[3]], -1)


def _giou_case():
    g = torch.Generator().manual_seed(1)
    tb = torch.round((torch.cat([0.2 + 0.6 * torch.rand(64, 2, generator=g), 0.02 + 0.2 * torch.rand(64, 4, generator=g)], -1)) * 1024) / 1024
    sb = tb.clone()
    sb[8:16, 3] *= 0.5                                  # shares three edges
    sb[16:24, 3:6:2] *= 0.5                             # shares x0 and y0
    sb[24:32, 0] = tb[24:32, 0] + tb[24:32, 3] + tb[24:32, 2]          # touching
    sb[32:40, 2:] *= 0.5                                # nested
    sb[40:48, 0] += 0.7                                 # disjoint
    sb[48:] = torch.round((sb[48:] + 0.05 * torch.randn(16, 6, generator=g)).abs() * 1024) / 1024 + 1 / 64
    return sb, tb


def test_giou_gradient_bound_is_sharp():
    sb, tb = _giou_case()
    s64 = sb.to(F64).requires_grad_(True)
    sxy = oc.cxcylrtb_to_xyxy(s64)
    sxy = sxy + (sxy.float().to(F64) - sxy).detach()
    (1 - torch.diag(oc.generalized_box_iou(sxy, oc.cxcylrtb_to_xyxy(tb.to(F64))))).sum().backward()
    _, mag = em.giou_mags(sb, tb)
    assert _ratio(_giou_grad_fp32(sb, tb), s64.grad, mag) <= em.C_BOX
    assert _ratio(_giou_grad_fp32(sb, tb, half=1.0), s64.grad, mag) > em.C_BOX               # ties not split
