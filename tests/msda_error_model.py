"""Error model of the deformable-attention sampling kernels (csrc/msda.cu), shared by the GPU tests that hold every dispatch
path to it (tests/test_msda_error_model_gpu.py) and by the CPU test that checks the bounds are sharp
(tests/test_msda_error_model_host_logic.py).

Reference.  The semantics of the reference kernel (ms_deform_im2col_cuda.cuh, restated by oracle/msda_oracle.c) in float64,
with one exception: the image coordinate of a sample is the kernels' fp32 x = fl32(loc * W - 0.5), formed here as
(loc.double() * W - 0.5).float().double().  The float64 product and difference are exact when |loc| >= 2^-30 or loc == 0,
so the one rounding to fp32 equals the kernels' fmaf.  floor(x) picks the cell and d out / d loc jumps at a cell line; with
the same coordinate, kernel and reference pick the same cell and take the same one-sided derivative.  Everything after the
coordinate is float64.

Magnitudes, from the same gather (w_k >= 0 the bilinear weights, v_k the corners, g = grad_out, u = 2^-24):

    out          S = sum_lp |a| sum_k w_k |v_k|
    grad_attn    sum_c |g_c| sum_k w_k |v_kc|
    grad_loc     W |a| sum_c |g_c| (hy (|v1c| + |v2c|) + ly (|v3c| + |v4c|)),  and for y: H |a| ... (hx (|v1| + |v3|) + lx ...)
    grad_value   S_i = sum |w g a| over the contributions to element i, and their count n_i

Bounds, per element: |y - r| <= C u mag for outputs with a fixed accumulation order, and <= C_GV (u sqrt(n_i) S_i + FLT_MIN n_i)
for the value gradient, whose atomics change the order from run to run and flush subnormal addends and sums to zero
(red / atom .add.f32 do: an absolute error below FLT_MIN per contribution).  Where mag == 0 (points outside the image, non-finite
locations, rows nothing samples) the kernel must give an exact zero.

Below FLT_MIN an fp32 rounding errs by up to half of ETA = 2^-149 absolutely, whatever the magnitude; a softmax over
logits of +-100 produces such weights.  So every bound carries ETA times the number k of terms of the element (valid corners;
times D for the channel reductions; n_i for the value gradient): |y - r| <= C (u mag + ETA k).  The fused softmax rounds
l_j - max l in fp32, a relative error of u |l_j - max l| in exp: its weights' magnitude is
a_j (1 + |l_j - max l| + sum_i a_i |l_i - max l|) (softmax_mag).

The constants are twice the worst ratio measured on an H100 over every element of the GPU tests' cases.  A kernel that
tests x >= -1, drops the last column, loses one contribution of a hot value-gradient row, scales grad_loc by the wrong side
or skips the softmax's max subtraction exceeds them: tests/test_msda_error_model_host_logic.py checks both directions on a
float32 simulation.
"""
import math

import torch

from tc_error_model import assert_rel  # noqa: F401  (re-exported: |y - ref| <= c * mag per element)

F32, F64 = torch.float32, torch.float64
U32 = 2.0 ** -24
ETA = 2.0 ** -149

FLT_MIN = 2.0 ** -126

# Twice the worst ratio measured on an H100 80GB HBM3 (700 W power limit) over every element of
# tests/test_msda_error_model_gpu.py, every path and mode.
C_OUT = 19.6      # worst 9.83: msda_fwd_d32_kernel, 2000 queries colliding in one 2x2 patch per level (64-term fmaf chain)
C_GA = 5.5        # worst 2.79: generic backward, D = 1
C_GL = 6.3        # worst 3.17: generic backward, D = 1
C_GV = 8.3        # worst 4.20: the fused backward's vector-reduction scatter, decoder call (Lq = 550, 6-d boxes); op paths 3.34
C_FUSED = 7.4     # worst 3.72: fused grad_logits, logits over +-100; grad_offsets 1.81
C_PART = 23.5     # worst 11.79: fused box partials, logits over +-100, 6-d boxes
C_PREP = 8.0      # worst 4.02: pre-processing softmax, L = 4, P = 4; loc 1.82, grad_offsets 1.93, grad_logits 3.66

# the reference's largest per-chunk gather: (points x 4 corners x D) float64 elements
_CHUNK = 1 << 24


def coord(loc, size):
    """The kernels' fp32 image coordinate fl32(loc * size - 0.5), as float64."""
    return (loc.to(F64) * size - 0.5).to(F32).to(F64)


def _gather(loc, shapes, lsi, S, M):
    """Bilinear set-up of every point of `loc` (B, Q, M, L, P, 2): weights w (.., 4) (0 for corners off the image),
    the rows of value.view(B*S*M, D) they read (0 where invalid), the validity mask, and lx, ly, hx, hy (.., 1)."""
    B, Q, _, L, P, _ = loc.shape
    dev = loc.device
    Hs = shapes[:, 0].to(dev).view(1, 1, 1, L, 1)
    Ws = shapes[:, 1].to(dev).view(1, 1, 1, L, 1)
    x, y = coord(loc[..., 0], Ws.to(F64)), coord(loc[..., 1], Hs.to(F64))
    inside = (y > -1) & (x > -1) & (y < Hs) & (x < Ws)
    xf = torch.where(inside, torch.floor(x), torch.zeros_like(x))
    yf = torch.where(inside, torch.floor(y), torch.zeros_like(y))
    lx = torch.where(inside, x - xf, torch.zeros_like(x))
    ly = torch.where(inside, y - yf, torch.zeros_like(y))
    hx, hy = 1 - lx, 1 - ly
    x0, y0 = xf.long(), yf.long()
    b = torch.arange(B, device=dev).view(B, 1, 1, 1, 1)
    m = torch.arange(M, device=dev).view(1, 1, M, 1, 1)
    start = lsi.to(dev).view(1, 1, 1, L, 1)
    ws, rows, oks = [], [], []
    for dy, dx, w in ((0, 0, hy * hx), (0, 1, hy * lx), (1, 0, ly * hx), (1, 1, ly * lx)):
        yy, xx = y0 + dy, x0 + dx
        ok = inside & (yy >= 0) & (yy <= Hs - 1) & (xx >= 0) & (xx <= Ws - 1)
        row = ((b * S + start + yy * Ws + xx) * M + m)
        ws.append(torch.where(ok, w, torch.zeros_like(w)))
        rows.append(torch.where(ok, row, torch.zeros_like(row)))
        oks.append(ok)
    return (torch.stack(ws, -1), torch.stack(rows, -1), torch.stack(oks, -1),
            *(t.unsqueeze(-1) for t in (lx, ly, hx, hy)))


def reference(value, shapes, lsi, loc, attn, grad_out=None, attn_mag=None):
    """float64 forward (and backward when grad_out is given) of the sampling op with the kernels' fp32 coordinate, and the
    magnitudes of the bounds.  Runs on the inputs' device, chunked over queries.  attn_mag replaces |a| in every magnitude
    (softmax_mag for weights an fp32 softmax produced).  Returns a dict: out, mag_out, cnt_out and, with grad_out,
    grad_value, gv_sum (S_i), gv_n (n_i, per element), grad_loc, mag_gl, grad_attn, mag_ga, cnt_pt (D x the valid corners of
    each point)."""
    B, S, M, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    vf = value.reshape(B * S * M, D).to(F64)
    r = {"out": torch.zeros(B, Lq, M, D, dtype=F64, device=value.device)}
    r["mag_out"] = torch.zeros_like(r["out"])
    r["cnt_out"] = torch.zeros(B, Lq, M, 1, dtype=F64, device=value.device)
    r["cnt_pt"] = torch.zeros(attn.shape, dtype=F64, device=value.device)
    if grad_out is not None:
        r["grad_value"] = torch.zeros(B * S * M, D, dtype=F64, device=value.device)
        r["gv_sum"] = torch.zeros_like(r["grad_value"])
        r["gv_n"] = torch.zeros(B * S * M, dtype=F64, device=value.device)
        r["grad_loc"] = torch.zeros(loc.shape, dtype=F64, device=value.device)
        r["mag_gl"] = torch.zeros_like(r["grad_loc"])
        r["grad_attn"] = torch.zeros(attn.shape, dtype=F64, device=value.device)
        r["mag_ga"] = torch.zeros_like(r["grad_attn"])
    Ws = shapes[:, 1].to(value.device, F64).view(1, 1, 1, L, 1)
    Hs = shapes[:, 0].to(value.device, F64).view(1, 1, 1, L, 1)
    step = max(1, _CHUNK // max(1, B * M * L * P * 4 * D))
    for q0 in range(0, Lq, step):
        q = slice(q0, min(Lq, q0 + step))
        w, rows, ok, lx, ly, hx, hy = _gather(loc[:, q], shapes, lsi, S, M)
        a = attn[:, q].to(F64).unsqueeze(-1)                           # (B, Q, M, L, P, 1)
        am = (attn_mag[:, q].to(F64).unsqueeze(-1) if attn_mag is not None else a.abs())
        nk = ok.sum(-1).to(F64)                                        # valid corners per point
        r["cnt_out"][:, q] = nk.sum((3, 4)).unsqueeze(-1)
        r["cnt_pt"][:, q] = D * nk
        v = vf[rows] * ok.unsqueeze(-1)                                # (B, Q, M, L, P, 4, D)
        va = v.abs()
        r["out"][:, q] = torch.einsum("bqmlpk,bqmlpkd->bqmd", a * w, v)
        r["mag_out"][:, q] = torch.einsum("bqmlpk,bqmlpkd->bqmd", am * w, va)
        if grad_out is None:
            continue
        g = grad_out[:, q].reshape(B, -1, M, 1, 1, 1, D).to(F64)
        s = (v * g).sum(-1)                                            # (B, Q, M, L, P, 4): sum_c g_c v_kc
        sa = (va * g.abs()).sum(-1)
        r["grad_attn"][:, q] = (w * s).sum(-1)
        r["mag_ga"][:, q] = (w * sa).sum(-1)
        s1, s2, s3, s4 = s.unbind(-1)
        t1, t2, t3, t4 = sa.unbind(-1)
        a0, am0 = a[..., 0], am[..., 0]
        lx, ly, hx, hy = (t[..., 0] for t in (lx, ly, hx, hy))
        r["grad_loc"][:, q, ..., 0] = Ws * a0 * (hy * (s2 - s1) + ly * (s4 - s3))
        r["grad_loc"][:, q, ..., 1] = Hs * a0 * (hx * (s3 - s1) + lx * (s4 - s2))
        r["mag_gl"][:, q, ..., 0] = Ws * am0 * (hy * (t1 + t2) + ly * (t3 + t4))
        r["mag_gl"][:, q, ..., 1] = Hs * am0 * (hx * (t1 + t3) + lx * (t2 + t4))
        c = (w * a).unsqueeze(-1) * g                                  # (B, Q, M, L, P, 4, D): contributions w a g
        ca = (w * am).unsqueeze(-1) * g.abs()
        idx = rows.reshape(-1)
        r["grad_value"].index_add_(0, idx, c.reshape(-1, D))
        r["gv_sum"].index_add_(0, idx, ca.reshape(-1, D))
        r["gv_n"].index_add_(0, idx, ok.reshape(-1).to(F64))
    r["out"] = r["out"].reshape(B, Lq, M * D)
    r["mag_out"] = r["mag_out"].reshape(B, Lq, M * D)
    r["cnt_out"] = r["cnt_out"].expand(B, Lq, M, D).reshape(B, Lq, M * D)
    if grad_out is not None:
        for k in ("grad_value", "gv_sum"):
            r[k] = r[k].reshape(B, S, M, D)
        r["gv_n"] = r["gv_n"].reshape(B, S, M, 1).expand(B, S, M, D)
    return r


def gv_mag(r):
    """u sqrt(n_i) S_i + FLT_MIN n_i: the scale of the value-gradient bound."""
    return U32 * r["gv_n"].sqrt() * r["gv_sum"] + FLT_MIN * r["gv_n"]


def scale(r, k):
    """u mag + ETA k of output k of a reference dict (the value gradient: gv_mag)."""
    if k == "grad_value":
        return gv_mag(r)
    if k == "out":
        return U32 * r["mag_out"] + ETA * r["cnt_out"]
    if k == "grad_attn":
        return U32 * r["mag_ga"] + ETA * r["cnt_pt"]
    return U32 * r["mag_gl"] + ETA * r["cnt_pt"].unsqueeze(-1)


def check(name, got, r, paths=("out", "grad_value", "grad_loc", "grad_attn")):
    """Hold the kernel outputs `got` (dict name -> tensor) to the bounds; returns {output: worst ratio}."""
    consts = {"out": C_OUT, "grad_attn": C_GA, "grad_loc": C_GL, "grad_value": C_GV}
    return {k: assert_rel(f"{name} {k}", got[k].reshape(r[k].shape), r[k], scale(r, k), consts[k]) for k in paths if k in got}


# ---- the module's pre-processing (ms_deform_attn.py:145-155) in float64 -------------------------------------------------------
def softmax64(logits, M, L, P):
    """float64 softmax over each unit's L*P logits -> (B, Lq, M, L, P)."""
    B, Lq = logits.shape[:2]
    return torch.softmax(logits.to(F64).view(B, Lq, M, L * P), -1).view(B, Lq, M, L, P)


def softmax_mag(logits, M, L, P):
    """Magnitude of fp32 softmax weights, (B, Lq, M, L, P): a_j (1 + |d_j| + sum_i a_i |d_i|), d = l - max l."""
    B, Lq = logits.shape[:2]
    lg = logits.to(F64).view(B, Lq, M, L * P)
    d = (lg - lg.amax(-1, keepdim=True)).abs()
    a = torch.softmax(lg, -1)
    return (a * (1 + d + (a * d).sum(-1, keepdim=True))).view(B, Lq, M, L, P)


def offset_scale(ref, shapes, M, L, P):
    """d loc / d offset in float64, (B, Lq, 1, L, 1, 2): 1 / (W, H) for 2-d references, (l + r, t + b) / (2 P) for 6-d boxes."""
    B, Lq = ref.shape[:2]
    r = ref.to(F64)
    if ref.shape[-1] == 2:
        s = (1.0 / shapes.to(ref.device, F64).flip(-1)).view(1, 1, 1, L, 1, 2).expand(B, Lq, 1, L, 1, 2)
    else:
        s = torch.stack((r[..., 2] + r[..., 3], r[..., 4] + r[..., 5]), -1).view(B, Lq, 1, L, 1, 2) * (0.5 / P)
    return s


def prep_loc(off, ref, shapes, M, L, P):
    """float64 sampling locations from fp32 offsets (B, Lq, M*L*P*2) and references, and their magnitude |ref| + |off s|."""
    B, Lq = off.shape[:2]
    o = off.to(F64).view(B, Lq, M, L, P, 2)
    s = offset_scale(ref, shapes, M, L, P)
    rxy = ref.to(F64)[..., :2].view(B, Lq, 1, L, 1, 2)
    return rxy + o * s, rxy.abs() + (o * s).abs()


def softmax_grad(a, mag_a, ga, mag_ga):
    """d logits of a softmax: a_j (ga_j - sum_i a_i ga_i) per unit (last dim flattened), and its magnitude
    mag_a_j (mag_ga_j + sum_i a_i mag_ga_i).  All float64, shape (B, Lq, M, L*P)."""
    dot = (a * ga).sum(-1, keepdim=True)
    return a * (ga - dot), mag_a * (mag_ga + (a * mag_ga).sum(-1, keepdim=True))


# ---- inputs at the edges -------------------------------------------------------------------------------------------------------
def loc_for(target, size):
    """fp32 locations whose kernel coordinate fl32(loc * size - 0.5) is exactly `target` (float64 tensor of fp32 values),
    searched among the nearest floats to (target + 0.5) / size.  Returns (loc, hit mask)."""
    base = ((target + 0.5) / size).to(F32)
    best, hit = base.clone(), coord(base, size) == target
    for k in (1, -1, 2, -2, 3, -3):
        c = base
        toward = torch.full_like(base, math.inf if k > 0 else -math.inf)
        for _ in range(abs(k)):
            c = torch.nextafter(c, toward)
        h = (coord(c, size) == target) & ~hit
        best, hit = torch.where(h, c, best), hit | h
    return best, hit


def edge_targets(n):
    """The coordinates the kernels' predicates and corner tests branch on, for a side of n pixels: -1 (excluded),
    nextafter(-1, 0), -0.5 (loc = 0), 0, an interior integer, n - 1, n - 1/4 (in (n - 1, n)), n (excluded)."""
    t = [-1.0, float(torch.nextafter(torch.tensor(-1.0), torch.tensor(0.0))), -0.5, 0.0, float(n // 2), n - 1.0, n - 0.25,
         float(n)]
    return torch.tensor(t, dtype=F64)


def make_inputs(shapes, B, Lq, M, D, P, seed, device="cpu", kind="plain", edges=True):
    """Seeded inputs (value, shapes, lsi, loc, attn, grad_out) of the op, fp32, with a share of exact-edge points.

    kind: 'plain' (softmax weights, randn values); 'signed' (unnormalised weights of both signs); 'offset' (values
    1000 + randn: v2 - v1 cancels); 'nonfinite' (a share of locations +-1e30, +-inf, NaN); 'collide' (every query of a
    batch samples inside one 2x2 patch per level).  With edges, every 3rd point has x on an edge target, every 5th y, and
    every 7th both (the image corners).  Returns the tensors and the number of points that landed exactly on each kind of
    target, per axis: {'x': tensor(8), 'y': tensor(8)}."""
    g = torch.Generator().manual_seed(seed)
    shapes_t = torch.as_tensor(shapes, dtype=torch.long)
    lsi = torch.cat((shapes_t.new_zeros((1,)), shapes_t.prod(1).cumsum(0)[:-1]))
    S, L = int(shapes_t.prod(1).sum()), len(shapes)
    value = torch.randn(B, S, M, D, generator=g)
    if kind == "offset":
        value = value + 1000.0
    loc = torch.rand(B, Lq, M, L, P, 2, generator=g) * 1.2 - 0.1
    if kind == "collide":
        loc = 0.5 + torch.rand(B, Lq, M, L, P, 2, generator=g) * 0.01
        Hs, Ws = shapes_t[:, 0].view(L, 1).double(), shapes_t[:, 1].view(L, 1).double()
        cx = (torch.floor(Ws * 0.5 - 0.5) + 0.5 + 0.5) / Ws                  # the middle of one cell, per level
        cy = (torch.floor(Hs * 0.5 - 0.5) + 0.5 + 0.5) / Hs
        jit = torch.rand(B, Lq, M, L, P, 2, generator=g, dtype=F64) * 0.8 - 0.4
        loc[..., 0] = (cx.view(1, 1, 1, L, 1) + jit[..., 0] / Ws.view(1, 1, 1, L, 1)).float()
        loc[..., 1] = (cy.view(1, 1, 1, L, 1) + jit[..., 1] / Hs.view(1, 1, 1, L, 1)).float()
    logits = torch.randn(B, Lq, M, L * P, generator=g)
    attn = torch.softmax(logits, -1).view(B, Lq, M, L, P)
    if kind == "signed":
        attn = (torch.randn(B, Lq, M, L, P, generator=g) * 2).float()
    grad_out = torch.randn(B, Lq, M * D, generator=g)
    landed = {"x": torch.zeros(8, dtype=torch.long), "y": torch.zeros(8, dtype=torch.long)}
    if edges and kind != "collide":
        flat = loc.view(-1, L, P, 2)
        n = flat.shape[0]
        idx = torch.arange(n * P).view(n, P)
        for ax, side, every in ((0, 1, 3), (1, 0, 5)):
            for l in range(L):
                size = int(shapes_t[l, side])
                t = edge_targets(size)
                sel = (idx + l) % every == 0
                sel |= (idx + l) % 7 == 0
                k = torch.randint(0, len(t), (n, P), generator=g)
                lo, hit = loc_for(t[k], size)
                use = sel & hit
                flat[:, l, :, ax] = torch.where(use, lo, flat[:, l, :, ax])
                landed["x" if ax == 0 else "y"] += torch.bincount(k[use], minlength=len(t))
    if kind == "nonfinite":
        special = torch.tensor([1e30, -1e30, math.inf, -math.inf, math.nan])
        pick = torch.rand(loc.shape, generator=g) < 0.15
        vals = special[torch.randint(0, 5, loc.shape, generator=g)]
        loc = torch.where(pick, vals, loc)
    return (value, shapes_t, lsi, loc.contiguous(), attn.contiguous(), grad_out), landed
