"""Error model of the fused head chains (csrc/heads.cu) and the elementwise helpers around the GEMMs (csrc/elementwise.cu),
shared by the GPU test that holds the kernels to it (tests/test_heads_edges_gpu.py) and by the CPU test that checks the
bounds are sharp (tests/test_heads_error_model_host_logic.py).

Every reference is float64, computed from the kernel's own fp32 inputs.  Where a kernel makes a discrete choice from fp32
arithmetic, the reference makes the kernel's choice: the bilinear cell of a centre and the resize source index are the
kernel's fp32 coordinate (emulated below, bit for bit); the depth-tail cell and fraction are read from the kernel's own
weighted-depth output; the mask of the query-depth height clamp is the kernel's fp32 height.  No element near a boundary
is excluded.  u = 2^-24.  Per element, |y - ref| <= C * u * mag (tc_error_model.assert_rel; zero magnitude: exact):

  box_refine fwd   sigmoid(tmp + inverse_sigmoid(ref))         mag = y(1-y)(|tmp| + |log max(x,eps)| + |log max(1-x,eps)| + 1) + y
  box_refine bwd   dtmp = dy y(1-y) from the kernel's y        mag = |dy| y(1-y)
                   dref = autograd of the reference in fp64     mag = |g| (sum of the 1/r, 1/(1-r) terms autograd includes)
                   (eps = fp32(1e-5) as torch compares it: the included set is autograd's; a term the kernel adds or drops
                   is an error of the term's size)
  head_depth fwd   (dr + geo + dm) / 3                          mag = (|dr| + 1 + |geo| + sum w|d|) / 3;  out[1] exact copy
  head_depth bwd   dhn (both of dcoord[4..5]), dsize3d[0]       mag = |ref|;  dcoord[0..3], dsize3d[1..2]: exact zeros
                   dreg[0] = -g s(1-s) / (s + 1e-6)^2           mag = |g| s (2 - s) / (s + 1e-6)^2   (s carries a relative
                   error of a few u, so 1 - s carries an absolute one);  dreg[1]: exact copy
                   map gradient sum_q w_q g_q                   mag = sum_q w_q |g_q|,  g = dout / 3
  depth_tail fwd   wd = sum p b                                 mag = sum p |b|
                   ip = e0 (1 - d) + e1 d                       mag = |e0| (1 - d) + |e1| d
  depth_tail bwd   dlogits = p_j (b_j - wd) dwd                 mag = (p_j + 2^-125)(|b_j| + sum p|b|)(dd_mag + |d_wd_ext|),
                                                                dd_mag = sum_ch |g| (|e0| + |e1|)
                   demb = sum_px g * weight                     mag = sum_px |g| * weight
  sum_mean_squares loss = sum_k mean(x_k^2)                     mag = the float64 loss;   grad 2 x / n dloss: mag = |ref|
  mean3, scale     torch fp32 (a + b + c) / 3;  dy * fp32(1/3)  bit-exact
  stem             relu(s conv(x, w) + b), relu on both sides   mag = |s| sum |w||x| + |b|
  max-pool 3x3/2   F.max_pool2d                                 bit-exact
  depth_sample     bilinear, zeros, align_corners=True          mag = sum w|d|;  backward sum_q w_q |g_q|
  resize           the kernel's source rule, fp64 weights       mag = sum w|x|;  backward sum w|dy|
  colsum           column sum (+ the prior when accumulating)   mag = sum |x| + |prior|
  relu_backward    where(y > 0, dy * scale, 0)                  bit-exact
  round_tf32       cvt.rna.tf32.f32: + 0x1000, clear 13 bits    bit-exact for finite and infinite inputs; what a NaN input
                                                                gives is not pinned

The depth-tail cell d = clamp(wd, 0, dmax) - floor(...) is the kernel's, read from its forward `wd` output, in the
forward and in both backward kernels.  The backward recomputes wd in three places (depth_tail_bwd_kernel<true>,
<false> and depth_tail_emb_grad_kernel); holding demb to sum |g| * weight with the forward's fraction is only possible
when each recomputation gives the forward's bits, and a different cell moves a whole row of the gradient.  wd, ip and
the rest are each held to their own bound.  The 2^-125 in the dlogits bound is the absolute error of an expf that
underflows into the denormals (logits 100 below the maximum): 2^-149 = u * 2^-125.

Compiled for sm_90a with the build's flags (cuobjdump -sass): up_src contracts to s = fma(o + 0.5, scale, -0.5) in both
resize kernels, and resize_src below emulates that; the backward's window bounds are a true division followed by a
FADD.  The bilinear centre (c - 0.5) * 2 + 1 contracts to one FFMA, which gives the same bits (the * 2 is exact).  The
depth-tail softmax sums are FMUL + FADD (no FFMA) in all four kernels.

Not covered, by design: NaN propagation.  fmaxf in the stem's ReLU and the max-pool drops a NaN where torch keeps it,
and relu_backward masks on y > 0; frozen weights and 8-bit images cannot produce one there.
"""
import torch

from tc_error_model import assert_rel  # noqa: F401  (re-exported: |y - ref| <= c * mag per element)

F64 = torch.float64
F32 = torch.float32
U32 = 2.0 ** -24
TINY = 2.0 ** -125          # expf underflow floor, in units of u (see above)

# Twice the worst ratio measured on an H100 80GB HBM3 (700 W power limit) over every element of tests/test_heads_edges_gpu.py,
# both modes (rounded up in the second digit).
C_BOX_FWD = 2.9       # worst 1.44: rd = 6, n = 4100
C_BOX_BWD = 6.9       # worst 3.45: dref, rd = 6, n = 4100
C_HD_FWD = 6.7        # worst 3.35: B = 1, N = 4096 on one 2x2 patch of 24 x 80
C_HD_BWD = 13.0       # worst 6.10: dcoord[4], B = 1, N = 4096 on one patch
C_HD_MAP = 4.7        # worst 2.31: B = 8, N = 300, 24 x 80
C_DT_WD = 16.0        # worst 7.69: npix = 15360, nb = 96, C = 132, bins outside [0, dmax]
C_DT_IP = 4.0         # worst 1.97: npix = 15360, nb = 33, C = 128, edge depths
C_DT_DLOGITS = 83.0   # worst 41.0: npix = 15360, nb = 96, C = 132, bins outside [0, dmax], d_wd only
C_DT_DEMB = 8.9       # worst 4.40: npix = 15360, nb = 81, C = 256, edge depths, d_ip only
C_SMS_FWD = 27.0      # worst 13.4: 32 tensors, n up to 1.2M, default mode (atomics: 10.4 in another run)
C_SMS_BWD = 3.0       # worst 1.48: n = 20 900 001
C_STEM = 13.0         # worst 6.05: B = 3, 384 x 1280
C_SAMPLE_FWD = 5.3    # worst 2.65: N = 4096 on one patch of 24 x 80
C_SAMPLE_BWD = 3.9    # worst 1.90: B = 2, N = 500, 24 x 80
C_RESIZE_FWD = 6.1    # worst 3.03: 12 x 40 -> 24 x 80, C = 256
C_RESIZE_BWD = 8.9    # worst 4.42: W 2 -> 30, C = 4
C_COLSUM = 62.0       # worst 30.9: M = 81600, N = 1025, accumulate

def f32c(v):
    """A Python float rounded to fp32, as a float64 (the constant an fp32 kernel or torch fp32 compares against)."""
    return float(torch.tensor(v, dtype=F32))


EPS_BOX = f32c(1e-5)
EPS_DEN = f32c(1e-6)


# ---- box refinement ---------------------------------------------------------------------------------------------------
def _inv_sigmoid64(r):
    x = r.clamp(min=0, max=1)
    return torch.log(x.clamp(min=EPS_BOX) / (1 - x).clamp(min=EPS_BOX))


def box_refine_fwd(tmp, ref):
    """tmp (n, 6), ref (n, rd) fp32 -> (y64, mag)."""
    rd = ref.shape[-1]
    t, r = tmp.to(F64), ref.to(F64)
    v = t.clone()
    v[:, :rd] = v[:, :rd] + _inv_sigmoid64(r)
    y = torch.sigmoid(v)
    x = r.clamp(0, 1)
    lg = torch.zeros_like(t)
    lg[:, :rd] = x.clamp(min=EPS_BOX).log().abs() + (1 - x).clamp(min=EPS_BOX).log().abs()
    return y, U32 * (y * (1 - y) * (t.abs() + lg + 1) + y)


def box_refine_bwd(dy, y, ref):
    """dy, y (the kernel's) (n, 6), ref (n, rd) -> (dtmp64, mag, dref64, mag)."""
    rd = ref.shape[-1]
    d, yy = dy.to(F64), y.to(F64)
    g = d * yy * (1 - yy)
    r = ref.to(F64).clone().requires_grad_()
    (dinv,) = torch.autograd.grad(_inv_sigmoid64(r), r, torch.ones_like(r))
    rr = ref.to(F64)
    inside = (rr >= 0) & (rr <= 1)
    terms = torch.where(inside & (rr >= EPS_BOX), 1 / rr, torch.zeros_like(rr)) + \
        torch.where(inside & (1 - rr >= EPS_BOX), 1 / (1 - rr), torch.zeros_like(rr))
    gr = g[:, :rd]
    return g, U32 * d.abs() * yy * (1 - yy), gr * dinv, U32 * gr.abs() * terms


# ---- bilinear sampling, align_corners=True (the heads' depth-map lookup) ----------------------------------------------------
def head_xy32(coord):
    """The kernel's fp32 map coordinates of head_depth: ((c - 0.5) * 2 + 1) * 0.5, before the * (W - 1)."""
    t = (coord.to(F32) - 0.5) * 2 + 1
    return t * 0.5


def grid_xy32(xy):
    """depth_sample: (xy + 1) * 0.5, before the * (W - 1)."""
    return (xy.to(F32) + 1) * 0.5


def corners(ux, uy, H, W):
    """ux, uy (..., ) fp32 as from head_xy32 / grid_xy32 -> x0, y0 (int64) and lx, ly (float64) of the kernel."""
    x = ux * float(W - 1)
    y = uy * float(H - 1)
    xf, yf = torch.floor(x), torch.floor(y)
    return xf.to(torch.int64), yf.to(torch.int64), (x - xf).to(F64), (y - yf).to(F64)


def _taps(x0, y0, lx, ly, H, W):
    """[(flat index or -1, weight)] for the four corners (out-of-map corners get index -1)."""
    out = []
    for dy_, dx_, w in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx), (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
        xx, yy = x0 + dx_, y0 + dy_
        ok = (xx >= 0) & (xx <= W - 1) & (yy >= 0) & (yy <= H - 1)
        out.append((torch.where(ok, yy * W + xx, torch.full_like(xx, -1)), w))
    return out


def bilinear_fwd(depth, x0, y0, lx, ly):
    """depth (B, H, W); corners (B, N) -> (value64, sum w|d|) per (b, n)."""
    B, H, W = depth.shape
    d = depth.to(F64).reshape(B, H * W)
    val = torch.zeros(x0.shape, dtype=F64, device=depth.device)
    mag = torch.zeros_like(val)
    for idx, w in _taps(x0, y0, lx, ly, H, W):
        v = torch.gather(d, 1, idx.clamp(min=0)) * (idx >= 0)
        val += w * v
        mag += w * v.abs()
    return val, mag


def bilinear_bwd(g, x0, y0, lx, ly, H, W):
    """g (B, N) -> (map gradient64, sum w|g|) (B, H, W)."""
    B = g.shape[0]
    g = g.to(F64)
    val = torch.zeros(B, H * W + 1, dtype=F64, device=g.device)
    mag = torch.zeros_like(val)
    for idx, w in _taps(x0, y0, lx, ly, H, W):
        i = torch.where(idx >= 0, idx, torch.full_like(idx, H * W))
        val.scatter_add_(1, i, w * g)
        mag.scatter_add_(1, i, w * g.abs())
    return val[:, :-1].reshape(B, H, W), mag[:, :-1].reshape(B, H, W)


# ---- depth of a query (monodetr.py:230-262) ---------------------------------------------------------------------------------
def head_depth_fwd(coord, size3d, reg, wdepth, calibs, img_sizes):
    """coord (B, N, 6), size3d (B, N, 3), reg (B, N, 2), wdepth (B, H, W), calibs (B, 3, 4), img_sizes (B, 2) ->
    (out0 64, mag) (B, N)."""
    B, N = coord.shape[:2]
    H, W = wdepth.shape[1:]
    c = coord.to(F64)
    ih, fu = img_sizes[:, 1].to(F64).view(B, 1), calibs[:, 0, 0].to(F64).view(B, 1)
    h = ((c[..., 4] + c[..., 5]) * ih).clamp(min=1)
    geo = size3d[..., 0].to(F64) / h * fu
    s = torch.sigmoid(reg[..., 0].to(F64))
    dr = 1 / (s + EPS_DEN) - 1
    u = head_xy32(coord[..., :2])
    x0, y0, lx, ly = corners(u[..., 0], u[..., 1], H, W)
    dm, dmag = bilinear_fwd(wdepth, x0, y0, lx, ly)
    return (dr + geo + dm) / 3, U32 * (dr.abs() + 1 + geo.abs() + dmag) / 3


def head_depth_bwd(dout, coord, size3d, reg, calibs, img_sizes, H, W):
    """-> dict name -> (ref64, mag) for dhn (dcoord[..., 4] == dcoord[..., 5]), dsize0, dreg0 and dmap."""
    B, N = coord.shape[:2]
    c = coord.to(F64)
    g = dout[..., 0].to(F64) / 3
    ih, fu = img_sizes[:, 1].to(F64).view(B, 1), calibs[:, 0, 0].to(F64).view(B, 1)
    hraw32 = (coord[..., 4].to(F32) + coord[..., 5].to(F32)) * img_sizes[:, 1].to(F32).view(B, 1)
    h = ((c[..., 4] + c[..., 5]) * ih).clamp(min=1)
    s0 = size3d[..., 0].to(F64)
    dhn = torch.where(hraw32 >= 1, -g * s0 * fu / (h * h) * ih, torch.zeros_like(h))
    ds0 = g * fu / h
    s = torch.sigmoid(reg[..., 0].to(F64))
    den = s + EPS_DEN
    dreg0 = -g * s * (1 - s) / (den * den)
    u = head_xy32(coord[..., :2])
    x0, y0, lx, ly = corners(u[..., 0], u[..., 1], H, W)
    dmap, mmag = bilinear_bwd(g, x0, y0, lx, ly, H, W)
    return {"dhn": (dhn, U32 * dhn.abs()), "dsize0": (ds0, U32 * ds0.abs()),
            "dreg0": (dreg0, U32 * g.abs() * s * (2 - s) / (den * den)), "dmap": (dmap, U32 * mmag)}


# ---- depth predictor tail (depth_predictor.py:74-104) -------------------------------------------------------------------------
def depth_tail_cell(wd_kernel, E, dmax):
    """The kernel's cell from its fp32 wd output: fi, ci (int64), d (float64) and x = clamp(wd, 0, dmax) (float32)."""
    x = wd_kernel.to(F32).clamp(min=0, max=float(torch.tensor(dmax, dtype=F32)))
    f = torch.floor(x)
    fi = f.to(torch.int64)
    return fi, (fi + 1).clamp(max=E - 1), (x - f).to(F64), x


def depth_tail_fwd(logits, bins, emb, wd_kernel, dmax):
    """logits (P, nb), bins (nb,), emb (E, C), the kernel's wd (P,) -> (wd64, mag), (ip64, mag)."""
    p = torch.softmax(logits.to(F64), -1)
    b = bins.to(F64)
    wd = (p * b).sum(-1)
    wdmag = (p * b.abs()).sum(-1)
    fi, ci, d, _ = depth_tail_cell(wd_kernel, emb.shape[0], dmax)
    e = emb.to(F64)
    e0, e1, dd = e[fi], e[ci], d.unsqueeze(-1)
    ip = e0 * (1 - dd) + e1 * dd
    return (wd, U32 * wdmag), (ip, U32 * (e0.abs() * (1 - dd) + e1.abs() * dd))


def depth_tail_bwd(logits, bins, emb, d_ip, d_wd_ext, wd_kernel, dmax):
    """-> (dlogits64, mag), (demb64, mag).  d_wd_ext may be None."""
    E, C = emb.shape
    p = torch.softmax(logits.to(F64), -1)
    b = bins.to(F64)
    wd = (p * b).sum(-1, keepdim=True)
    wdmag = (p * b.abs()).sum(-1, keepdim=True)
    fi, ci, d, _ = depth_tail_cell(wd_kernel, E, dmax)
    e = emb.to(F64)
    g = d_ip.to(F64)
    dd = (g * (e[ci] - e[fi])).sum(-1)
    ddmag = (g.abs() * (e[ci].abs() + e[fi].abs())).sum(-1)
    wk = wd_kernel.to(F32)
    inside = (wk >= 0) & (wk <= float(torch.tensor(dmax, dtype=F32)))
    dwd = torch.where(inside, dd, torch.zeros_like(dd))
    ext = torch.zeros_like(dd) if d_wd_ext is None else d_wd_ext.to(F64)
    dwd = dwd + ext
    dlog = p * (b - wd) * dwd.unsqueeze(-1)
    dmag = (p + TINY) * (b.abs() + wdmag) * (ddmag + ext.abs()).unsqueeze(-1)
    dl = d.unsqueeze(-1)
    demb = torch.zeros(E, C, dtype=F64, device=g.device)
    emag = torch.zeros_like(demb)
    for idx, w in ((fi, 1 - dl), (ci, dl)):
        demb.index_add_(0, idx, g * w)
        emag.index_add_(0, idx, g.abs() * w)
    return (dlog, U32 * dmag), (demb, U32 * emag)


# ---- sum_k mean(x_k^2) ------------------------------------------------------------------------------------------------------
def sum_mean_squares(xs, dloss):
    """-> (loss64, mag), [(grad64, mag)] for dloss (fp32 scalar)."""
    loss = sum((x.to(F64) ** 2).mean() for x in xs)
    dl = float(dloss)
    grads = [(2 * x.to(F64) / x.numel() * dl, U32 * (2 * x.to(F64) / x.numel() * dl).abs()) for x in xs]
    return (loss, U32 * loss), grads


# ---- stem ---------------------------------------------------------------------------------------------------------------------
def stem(x, w, scale, bias):
    """x (B, 3, H, W), w (64, 3, 7, 7) -> (relu(y64) NHWC, mag NHWC)."""
    import torch.nn.functional as F
    conv = F.conv2d(x.to(F64), w.to(F64), None, stride=2, padding=3)
    cabs = F.conv2d(x.to(F64).abs(), w.to(F64).abs(), None, stride=2, padding=3)
    s, b = scale.to(F64).view(1, -1, 1, 1), bias.to(F64).view(1, -1, 1, 1)
    y = torch.relu(conv * s + b)
    mag = U32 * (s.abs() * cabs + b.abs())
    return y.permute(0, 2, 3, 1), mag.permute(0, 2, 3, 1)


# ---- bilinear resize, align_corners=False ---------------------------------------------------------------------------------------
def resize_src(Hi, Ho, fma=True, clamp=True):
    """The kernel's up_src for every output row o < Ho: i0, i1 (int64), l0, l1 (float64 of the kernel's fp32 source index).
    fma: s = fp32(fma(o + 0.5, scale, -0.5)) as compiled (the product of two floats is exact in float64 and so is the sum
    at these sizes); otherwise a rounded product and a rounded difference."""
    scale = torch.tensor(float(Hi), dtype=F32) / torch.tensor(float(Ho), dtype=F32)
    o = torch.arange(Ho, dtype=F32) + 0.5
    if fma:
        s = (o.to(F64) * float(scale) - 0.5).to(F32)
    else:
        s = o * scale - 0.5
    if clamp:
        s = s.clamp(min=0)
    i0 = s.to(torch.int64)                                 # truncation, like (int)
    i1 = i0 + (i0 < Hi - 1).to(torch.int64)
    l1 = s.to(F64) - i0.to(F64)
    return i0, i1, 1 - l1, l1


def resize_matrix(Hi, Ho, **kw):
    """(Ho, Hi) float64 interpolation matrix of one axis."""
    i0, i1, l0, l1 = resize_src(Hi, Ho, **kw)
    A = torch.zeros(Ho, Hi, dtype=F64)
    r = torch.arange(Ho)
    A.index_put_((r, i0), l0, accumulate=True)
    A.index_put_((r, i1), l1, accumulate=True)
    return A


def resize_fwd(x, Ho, Wo, **kw):
    """x (B, Hi, Wi, C) -> (y64, mag)."""
    Ah = resize_matrix(x.shape[1], Ho, **kw).to(x.device)
    Aw = resize_matrix(x.shape[2], Wo, **kw).to(x.device)
    xx = x.to(F64)
    y = torch.einsum("oh,bhwc,pw->bopc", Ah, xx, Aw)
    mag = torch.einsum("oh,bhwc,pw->bopc", Ah.abs(), xx.abs(), Aw.abs())
    return y, U32 * mag


def resize_bwd(dy, Hi, Wi, **kw):
    """dy (B, Ho, Wo, C) -> (dx64, mag)."""
    Ah = resize_matrix(Hi, dy.shape[1], **kw).to(dy.device)
    Aw = resize_matrix(Wi, dy.shape[2], **kw).to(dy.device)
    g = dy.to(F64)
    dx = torch.einsum("oh,bopc,pw->bhwc", Ah, g, Aw)
    mag = torch.einsum("oh,bopc,pw->bhwc", Ah.abs(), g.abs(), Aw.abs())
    return dx, U32 * mag


def resize_window(h, scale, Ho):
    """The backward's fp32 window [ylo, yhi] of input row h (int64 tensors) for scale = fp32(Hi) / fp32(Ho)."""
    hf = h.to(F32)
    sc = torch.tensor(float(scale), dtype=F32)
    lo = torch.floor((hf - 0.5) / sc - 0.5).to(torch.int64) - 2
    lo = torch.where(h <= 1, torch.zeros_like(lo), lo.clamp(min=0))
    hi = (torch.ceil((hf + 1.5) / sc - 0.5).to(torch.int64) + 2).clamp(max=Ho - 1)
    return lo, hi


# ---- column sums ------------------------------------------------------------------------------------------------------------------
def colsum(x, prior=None):
    """x (M, N) -> (sum64 (+ prior), mag)."""
    xx = x.to(F64)
    s, mag = xx.sum(0), xx.abs().sum(0)
    if prior is not None:
        s, mag = s + prior.to(F64), mag + prior.to(F64).abs()
    return s, U32 * mag


# ---- exact operations ---------------------------------------------------------------------------------------------------------
def round_tf32(x):
    """cvt.rna.tf32.f32 in integers: round the low 13 bits to nearest, ties away from zero (add 0x1000 to the magnitude,
    clear the 13 bits); a carry moves into the exponent, and past the largest finite tf32 into infinity (no saturation).
    NaN inputs are out of its domain: the H100 does not return these bits for every NaN."""
    b = x.to(F32).view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x1000) & 0xFFFFE000
    return (r - ((r >> 31) << 32)).to(torch.int32).view(F32)


def relu_backward(dy, y, scale):
    s = torch.tensor(scale, dtype=F32, device=dy.device)
    return torch.where(y > 0, dy * s, torch.zeros_like(dy))


# ---- depth-tail edge inputs -----------------------------------------------------------------------------------------------------
def edge_logits(bins, dmax, steps=4):
    """fp32 logits (rows, nb) whose float64 weighted depth is exactly an integer k, for every k in (0, dmax] the bins allow,
    and the same rows with one logit stepped -steps..steps ulps; then all the mass on the last bin (the other logits at -100,
    then at -30).  The bin A just below k holds the maximum (e = 1); bins B and B + 32, one lane of the kernels' softmax,
    carry e_C = 0.3 and e_B solved in float64, so that lane adds an inexact product onto a non-zero partial sum -- where an
    FMA would round differently.  The other logits are -100."""
    b = bins.to(F64)
    nb, rows = b.numel(), []
    for k in range(1, int(dmax) + 1):
        a = int(torch.searchsorted(b, torch.tensor(float(k), dtype=F64))) - 1
        if a < 0 or float(b[a]) >= k:
            continue
        for j in range(nb - 32):
            if j % 32 == a % 32 or j == a or j + 32 == a:
                continue
            bB, bC, eC = float(b[j]), float(b[j + 32]), 0.3
            if bB == k:
                continue
            eB = (k * (1 + eC) - float(b[a]) - eC * bC) / (bB - k)
            if not 0.02 < eB < 0.98:
                continue
            base = torch.full((nb,), -100.0, dtype=F64)
            base[a], base[j], base[j + 32] = 0.0, float(torch.log(torch.tensor(eB, dtype=F64))), float(torch.log(torch.tensor(eC, dtype=F64)))
            l0 = base.to(F32)
            lo = hi = l0[j]
            steps_dn, steps_up = [], []
            for _ in range(steps):
                lo, hi = torch.nextafter(lo, torch.tensor(-1e9)), torch.nextafter(hi, torch.tensor(1e9))
                steps_dn.append(lo)
                steps_up.append(hi)
            for s in steps_dn[::-1] + [l0[j]] + steps_up:
                r = l0.clone()
                r[j] = s
                rows.append(r)
            break
    for other in (-100.0, -30.0):
        r = torch.full((nb,), other)
        r[-1] = 0.0
        rows.append(r)
    return torch.stack(rows)
