"""Error model of the training criterion (csrc/criterion.cu), shared by the GPU tests that hold the kernels to it
(tests/test_criterion_edges_gpu.py) and by the CPU test that checks the bounds are sharp
(tests/test_criterion_error_model_host_logic.py).

The reference is oracle/criterion.py run in float64 from the kernels' fp32 inputs, with the device's matching, and with the
predicted box corners rounded to fp32 as the kernels form them (`corner_dtype`), so that GIoU's max / min ties and clamps take
the kernels' branches; every other decision (sign(0) of an fp32 difference, the depth map's edges and bins, argmax) is the
same in both precisions because it is formed from fp32 values or from an fp32 rounding that keeps the sign.  u = 2^-24.

Per element, |got - ref64| <= C * u * mag, where mag is the element's expression evaluated on absolute values (a difference
a - b counts as |a| + |b|, 1 - p as 1 + p, log p = z - max - log sum as |z| + |max| + |log sum|):

    focal dlogits    |g_ce| a_t ((1 + p_t)^2 (p + t) + 2 bce' (1 + p_t) p (1 + p)),  bce' = max(x, 0) + |x| t + log1p(e^-|x|)
    box gradients    L1: |g|;  GIoU: |g_giou| * sum over the corners it moves of
                     (|di| U + I (|da| + |di|)) / U^2 + ((|da| + |di|) A_c + U |dc|) / A_c^2
    depth            |g| e'  and  |g| (1 + e' |d|),  e' = 1.4142 e^-s1
    dimensions       |g| comp / t3
    heading          |g| (p_k (1 + |a_k - m| + sum_j p_j |a_j - m|) + [k == bin] + 2^-149 / u),  residual |g|
    depth-map pixel  a w sum_c t_c (1 + p_c)^2 lp'_c,  lp'_c = |z_c| + |m| + |log s|
    depth-map dz     |scale| (f'_k + p_k (1 + lp'_k) sum_c f'_c + 2^-149 / u),  f'_c = t_c (2 (1 + p_c) p_c lp'_c + (1 + p_c)^2)

and for each loss scalar, C_LOSS * u * sum |terms| / num_boxes over the terms it adds.  Cardinality and class error are
counts of argmax decisions: they must be equal.  The 2^-149 terms cover softmax probabilities below fp32's normal range
(e^-100 of a +-50 peak), which expf returns with an absolute, not a relative, error.
"""
import torch

from tc_error_model import assert_rel  # noqa: F401  (re-exported: |y - ref| <= c * mag per element)

F64 = torch.float64
U32 = 2.0 ** -24
SUB = 2.0 ** -149       # fp32's subnormal spacing: the absolute error of a softmax probability that underflows (e^-100)

# Twice the worst ratio measured on an H100 80GB HBM3 (700 W power limit) over every element of
# tests/test_criterion_edges_gpu.py (eval, training and reproducible mode).
C_LOSS = 3.5    # worst 1.75: loss scalars (loss_depth, log-variance -30)
C_LOGITS = 5.0  # worst 0.71; 2.39 on the CPU fp32 emulation of test_criterion_error_model_host_logic.py
C_BOX = 3.0     # worst 1.47: box gradients (L1 + GIoU)
C_DEPTH = 5.5   # worst 2.75: depth and log-variance gradients
C_DIM = 4.5     # worst 2.24: dimension gradients
C_ANGLE = 54.0  # worst 26.5: heading gradients (peaked logits)
C_PIX = 6.2     # worst 3.08: depth-map pixel loss
C_DMAP = 8.6    # worst 4.27: depth-map dlogits


def focal_mags(x, t, alpha=0.25):
    """Per element of the (B, Q, C) logits: (loss-term magnitude, gradient magnitude without g_ce / num_boxes)."""
    x, t = x.to(F64), t.to(F64)
    p = torch.sigmoid(x)
    pt = p * t + (1 - p) * (1 - t)
    at = alpha * t + (1 - alpha) * (1 - t)
    bce_m = x.clamp(min=0) + x.abs() * t + torch.log1p(torch.exp(-x.abs()))
    om_m = 1 + pt
    return U32 * at * bce_m * om_m ** 2, U32 * at * (om_m ** 2 * (p + t) + 2 * bce_m * om_m * p * (1 + p))


def corners(b):
    """(N, 6) fp32 (cx, cy, l, r, t, b) -> x0 y0 x1 y1 rounded as the kernels form them, in float64."""
    b = b.float()
    return [v.to(F64) for v in (b[:, 0] - b[:, 2], b[:, 1] - b[:, 4], b[:, 0] + b[:, 3], b[:, 1] + b[:, 5])]


def giou_mags(sb, tb):
    """Matched pairs (N, 6) predicted / target boxes: ((N,) magnitude of 1 - giou, (N, 6) magnitude of its gradient)."""
    x0, y0, x1, y1 = corners(sb)
    X0, Y0, X1, Y1 = corners(tb)
    w, h = x1 - x0, y1 - y0
    area1, area2 = w * h, (X1 - X0) * (Y1 - Y0)
    iwr, ihr = torch.minimum(x1, X1) - torch.maximum(x0, X0), torch.minimum(y1, Y1) - torch.maximum(y0, Y0)
    iw, ih = iwr.clamp(min=0), ihr.clamp(min=0)
    inter = iw * ih
    uni = area1 + area2 - inter
    cwr, chr_ = torch.maximum(x1, X1) - torch.minimum(x0, X0), torch.maximum(y1, Y1) - torch.minimum(y0, Y0)
    cw, ch = cwr.clamp(min=0), chr_.clamp(min=0)
    areac = cw * ch
    liv, lih, lcv, lch = ((v >= 0).to(F64) for v in (iwr, ihr, cwr, chr_))

    def split(lt, eq, val):             # 1 on a strict inequality, 1/2 on a tie
        return torch.where(lt, val, torch.where(eq, 0.5 * val, torch.zeros_like(val)))
    di = [split(x0 > X0, x0 == X0, ih * liv), split(y0 > Y0, y0 == Y0, iw * lih),
          split(x1 < X1, x1 == X1, ih * liv), split(y1 < Y1, y1 == Y1, iw * lih)]
    dc = [split(x0 < X0, x0 == X0, ch * lcv), split(y0 < Y0, y0 == Y0, cw * lch),
          split(x1 > X1, x1 == X1, ch * lcv), split(y1 > Y1, y1 == Y1, cw * lch)]
    da = [h.abs(), w.abs(), h.abs(), w.abs()]
    dx = []
    for k in range(4):
        du = da[k] + di[k]
        dx.append((di[k] * uni + inter * du) / uni ** 2 + (du * areac + uni * dc[k]) / areac ** 2)
    grad = torch.stack([dx[0] + dx[2], dx[1] + dx[3], dx[0], dx[2], dx[1], dx[3]], -1)
    return U32 * (1 + inter / uni + (areac + uni) / areac), U32 * grad


def softmax_mags(a, hb):
    """Heading logits (N, 12), bins (N,): ((N,) magnitude of the cross-entropy, (N, 12) magnitude of its gradient)."""
    a = a.to(F64)
    m = a.max(-1, keepdim=True).values
    p = torch.softmax(a, -1)
    dz = (a - m).abs()
    oh = torch.nn.functional.one_hot(hb, a.shape[-1]).to(F64)
    lse = torch.logsumexp(a, -1)
    ce_mag = m.squeeze(-1).abs() + (lse - m.squeeze(-1)).abs() + (a * oh).sum(-1).abs() + (p * dz).sum(-1)
    return U32 * ce_mag, U32 * (p * (1 + dz + (p * dz).sum(-1, keepdim=True)) + oh) + SUB


def depth_map_mags(z, target, fg, alpha=0.25, fg_w=13.0, bg_w=1.0):
    """Depth-map logits (B, D, H, W) (float64), target bins and foreground (B, H, W): ((B, H, W) magnitude of the pixel loss,
    (B, D, H, W) magnitude of d loss / d z without the scale alpha * weight * g / npix, and the weight per pixel)."""
    z = z.to(F64)
    m = z.max(1, keepdim=True).values
    logs = torch.logsumexp(z - m, 1, keepdim=True)
    p = torch.softmax(z, 1)
    lp_m = z.abs() + m.abs() + logs.abs()
    t = torch.zeros_like(z).scatter_(1, target.unsqueeze(1), 1.0) + 1e-6
    wgt = torch.where(fg, torch.full_like(fg, fg_w, dtype=F64), torch.full_like(fg, bg_w, dtype=F64))
    pix = alpha * wgt * (t * (1 + p) ** 2 * lp_m).sum(1)
    f_m = t * (2 * (1 + p) * p * lp_m + (1 + p) ** 2)
    dz = f_m + p * (1 + lp_m) * f_m.sum(1, keepdim=True)
    return U32 * pix, U32 * dz + SUB, wgt
