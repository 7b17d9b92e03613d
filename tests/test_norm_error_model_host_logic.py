"""The bounds of tests/norm_error_model.py are sharp, checked without a GPU.  A float32 emulation of csrc/norm.cu in the
kernels' accumulation order -- GroupNorm: thread mapping and per-thread chains of gn_stats_kernel (default mode: pixel
blocks of up to 64 per image) and gn_stats_group_kernel (reproducible mode: one CTA per (group, image)), the double combine,
then gn_apply_kernel's formula; LayerNorm: add_ln_fwd_kernel's two-pass row statistics over a warp's lanes -- meets the
bounds with the shipped algorithm, and breaks them with unshifted E[x^2] - E[x]^2 statistics summed in fp32 chains, and
with each arithmetic mutant: statistics of the neighbouring group, the ReLU mask dropped in the backward, the clamp of the
variance removed, a shift that differs between the threads of one group."""
import math

import pytest
import torch

import norm_error_model as em

F32, F64 = torch.float32, torch.float64
EPS = 1e-5


# ---- GroupNorm emulation -------------------------------------------------------------------------------------------------
def gn_sums(x, G, path, shift="group", chain=F64):
    """Per-(b, g) float64 sums of the shifted values and of their squares, as the statistics kernel forms them: each thread
    adds its channel quad per pixel in fp32 (((v.x + v.y) + v.z) + v.w) and accumulates those over its pixels in `chain`
    (double; fp32 in the kernels before the shift), the threads' partials meet in double.  shift: 'group'
    (K[b][g] = x[b][0][first channel of g]), 'none' (raw sums), or 'thread' (each thread subtracts the first value of its
    own chain: differs between the threads of a group).  Returns (K, su, sq)."""
    B, HW, C = x.shape
    cpg = C // G
    qpg = cpg // 4
    K = x[:, 0, ::cpg].clone() if shift != "none" else torch.zeros(B, G)
    if path == "default":
        blocks = min((HW + 255) // 256, 64)
        ppb = (HW + blocks - 1) // blocks
        ranges = [(p0, min(HW, p0 + ppb)) for p0 in range(0, HW, ppb)]
        pls = 256 // (C // 4)
    else:
        ranges = [(0, HW)]
        pls = 256 // qpg
    su, sq = torch.zeros(B, G, dtype=F64), torch.zeros(B, G, dtype=F64)
    kq = K.repeat_interleave(cpg // 4, dim=1).view(B, 1, C // 4, 1)      # the group's shift, per channel quad
    for p0, p1 in ranges:
        n = p1 - p0
        steps = -(-n // pls)
        seg = torch.zeros(B, steps * pls, C)
        valid = torch.zeros(B, steps * pls, 1, dtype=torch.bool)
        seg[:, :n], valid[:, :n] = x[:, p0:p1], True
        seg, valid = seg.view(B, steps, pls, C // 4, 4), valid.view(B, steps, pls, 1, 1)
        k = seg[:, 0, :, :, :1] if shift == "thread" else kq             # 'thread': x at the chain's first pixel
        v = torch.where(valid, seg - k.unsqueeze(1), torch.zeros(()))
        s, ss = torch.zeros(B, pls, C // 4, dtype=chain), torch.zeros(B, pls, C // 4, dtype=chain)
        for j in range(steps):
            q = v[:, j]
            s = s + (((q[..., 0] + q[..., 1]) + q[..., 2]) + q[..., 3]).to(chain)
            qq = q * q
            ss = ss + (((qq[..., 0] + qq[..., 1]) + qq[..., 2]) + qq[..., 3]).to(chain)
        su += s.to(F64).view(B, pls, G, qpg).sum((1, 3))
        sq += ss.to(F64).view(B, pls, G, qpg).sum((1, 3))
    return K, su, sq


def rsqrt32(v):
    return (1.0 / torch.sqrt(v.to(F64))).to(F32)


def gn_forward(x, gamma, beta, G, path, algo="shifted", relu=False, mutant=None):
    """gn_apply_kernel after the statistics.  algo: 'shifted' (shipped) or 'raw' (fp32 chains of x and x^2, no clamp: the
    kernels before the shift).  mutant: 'neighbour' (group g reads the statistics of g + 1), 'thread_shift', 'clamp' (raw
    sums, but the variance clamped at 0)."""
    B, HW, C = x.shape
    n = HW * (C // G)
    if algo == "raw":
        _, su, sq = gn_sums(x, G, path, "none", F32)
        mu = su / n
        mean, var = mu.to(F32), sq / n - mu * mu
        if mutant == "clamp":
            var = var.clamp_min(0.0)
    else:
        K, su, sq = gn_sums(x, G, path, "thread" if mutant == "thread_shift" else "group")
        d = su / n
        mean, var = (K.to(F64) + d).to(F32), (sq / n - d * d).clamp_min(0.0)
    rstd = rsqrt32(var.to(F32) + torch.tensor(EPS, dtype=F32))
    if mutant == "neighbour":
        mean, rstd = mean.roll(-1, 1), rstd.roll(-1, 1)
    mb = mean.repeat_interleave(C // G, 1).view(B, 1, C)
    rb = rstd.repeat_interleave(C // G, 1).view(B, 1, C)
    y = ((x - mb) * rb) * gamma + beta
    return (y.clamp_min(0.0) if relu else y), mean, rstd


def gn_backward(dy, x, y, gamma, mean, rstd, G, relu, mutant=None):
    """gn_bwd_*: d = dy masked by y > 0 (unless mutant == 'no_mask'); per-group sums of d*gamma and d*gamma*xhat met in
    double; dx per element in fp32."""
    B, HW, C = x.shape
    n = HW * (C // G)
    d = dy * (y > 0) if relu and mutant != "no_mask" else dy
    mb = mean.repeat_interleave(C // G, 1).view(B, 1, C)
    rb = rstd.repeat_interleave(C // G, 1).view(B, 1, C)
    xh = (x - mb) * rb
    gy = d * gamma
    m1 = (gy.to(F64).view(B, HW, G, -1).sum((1, 3)) / n).to(F32).repeat_interleave(C // G, 1).view(B, 1, C)
    m2 = ((gy * xh).to(F64).view(B, HW, G, -1).sum((1, 3)) / n).to(F32).repeat_interleave(C // G, 1).view(B, 1, C)
    dx = rb * ((gy - m1) - xh * m2)
    return dx, (d * xh).to(F64).sum((0, 1)).to(F32), d.to(F64).sum((0, 1)).to(F32)


def gn_inputs(B, HW, C, G, offsets=(0.0, 30.0, 1000.0), constants=(10.1, 30.1), seed=0):
    """randn plus a per-group offset cycling through `offsets`; the last len(constants) groups of image 0 are constant."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, HW, C, generator=g)
    off = torch.tensor([offsets[i % len(offsets)] for i in range(G)]).repeat_interleave(C // G)
    x = x + off
    for i, c in enumerate(constants):
        gi = G - 1 - i
        x[0, :, gi * (C // G):(gi + 1) * (C // G)] = c
    gamma = torch.rand(C, generator=g) + 0.5
    beta = torch.randn(C, generator=g)
    dy = torch.randn(B, HW, C, generator=g)
    return x, gamma, beta, dy


def gn_ratios(x, gamma, beta, G, y, mean, rstd, relu=False, dy=None, bwd=None):
    """Worst ratio of each bound (over its constant's u-magnitude): dict name -> ratio (inf when not finite)."""
    z4 = em.view4(x, G)
    g4, b4 = em.param4(gamma, G), em.param4(beta, G)
    y64, mag, mu, rstd64, m, xh = em.forward(z4, g4, b4, EPS)
    if relu:
        y64 = y64.clamp_min(0.0)
    r = {"y": _ratio(em.view4(y, G), y64, mag),
         "mean": _ratio(mean.view(mu.shape), mu, em.U32 * m),
         "rstd": _ratio(rstd.view(rstd64.shape).to(F64) / rstd64, torch.ones_like(rstd64), torch.full_like(rstd64, em.U32))}
    if bwd is not None:
        dx, dg, db = bwd
        d4 = em.view4(dy * (y > 0) if relu else dy, G)
        dx64, mag_dx, dxh, mag_dg, mag_db = em.backward(d4, g4, rstd64, m, xh)
        r["dx"] = _ratio(em.view4(dx, G), dx64, mag_dx)
        r["dgamma"] = _ratio(dg, em.param_sum(dxh), em.param_sum(mag_dg))
        r["dbeta"] = _ratio(db, em.param_sum(d4.to(F64)), em.param_sum(mag_db))
    return r


def _ratio(y, ref, mag):
    y = y.to(F64)
    if not bool(torch.isfinite(y).all()):
        return math.inf
    err = (y - ref).abs()
    pos = mag > 0
    if not bool((err[~pos] == 0).all()):
        return math.inf
    return float((err[pos] / mag[pos]).max()) if bool(pos.any()) else 0.0


BOUND = {"y": "C_FWD", "mean": "C_MU", "rstd": "C_RSTD", "dx": "C_BWD", "dgamma": "C_PAR", "dbeta": "C_PAR"}


def _within(r):
    return {k: v <= getattr(em, BOUND[k]) for k, v in r.items()}


# ---- GroupNorm: the shipped algorithm meets the bounds ------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["default", "repro"])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("B,HW,C,G", [(2, 1920, 256, 32), (1, 257, 1024, 32), (2, 3, 64, 16)])
def test_shifted_statistics_meet_the_bounds(path, relu, B, HW, C, G):
    x, gamma, beta, dy = gn_inputs(B, HW, C, G)
    y, mean, rstd = gn_forward(x, gamma, beta, G, path, relu=relu)
    r = gn_ratios(x, gamma, beta, G, y, mean, rstd, relu, dy, gn_backward(dy, x, y, gamma, mean, rstd, G, relu))
    print(path, relu, (B, HW, C, G), {k: f"{v:.2e}" for k, v in r.items()})
    assert all(_within(r).values()), r
    # constant groups (the last two of image 0): y is beta exactly, relu(beta) with the fused ReLU
    cpg = C // G
    for gi in (G - 1, G - 2):
        ch = slice(gi * cpg, (gi + 1) * cpg)
        want = beta[ch].clamp_min(0.0) if relu else beta[ch]
        assert torch.equal(y[0, :, ch], want.expand(HW, cpg))
        assert float(rstd[0, gi]) == float(rsqrt32(torch.tensor(EPS, dtype=F32)))


# ---- GroupNorm: the raw E[x^2] - E[x]^2 statistics break them ----------------------------------------------------------------
@pytest.mark.parametrize("path", ["default", "repro"])
def test_raw_statistics_break_the_forward_bound_at_offset_30(path):
    x, gamma, beta, _ = gn_inputs(1, 1920, 256, 32, offsets=(30.0,), constants=())
    y, mean, rstd = gn_forward(x, gamma, beta, 32, path, algo="raw")
    r = gn_ratios(x, gamma, beta, 32, y, mean, rstd)
    print(path, {k: f"{v:.2e}" for k, v in r.items()})
    assert r["rstd"] > em.C_RSTD
    if path == "default":
        assert r["y"] > em.C_FWD
    # the same input without the offset is fine either way: the defect is the cancellation
    y0, mean0, rstd0 = gn_forward(x - 30.0, gamma, beta, 32, path, algo="raw")
    assert all(_within(gn_ratios(x - 30.0, gamma, beta, 32, y0, mean0, rstd0)).values())


@pytest.mark.parametrize("path,c", [("default", 10.1), ("repro", 30.1)])
def test_raw_statistics_on_a_constant_group(path, c):
    x, gamma, beta, _ = gn_inputs(1, 1920, 256, 32, offsets=(0.0,), constants=(c,))
    y, mean, rstd = gn_forward(x, gamma, beta, 32, path, algo="raw")
    want = float(rsqrt32(torch.tensor(EPS, dtype=F32)))
    got = float(rstd[0, 31])
    print(path, c, "rstd", got, "want", want)
    assert not math.isfinite(got) or abs(got / want - 1) > 1e-2
    assert not torch.equal(y[0, :, 248:], beta[248:].expand(1920, 8))


# ---- GroupNorm: mutants ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["default", "repro"])
def test_neighbouring_group_statistics_break_the_bound(path):
    x, gamma, beta, _ = gn_inputs(1, 240, 256, 32, offsets=(0.0,), constants=())
    x = x * torch.linspace(0.5, 2.0, 32).repeat_interleave(8)                # groups of different spread
    y, mean, rstd = gn_forward(x, gamma, beta, 32, path, mutant="neighbour")
    assert gn_ratios(x, gamma, beta, 32, y, mean, rstd)["y"] > em.C_FWD


@pytest.mark.parametrize("path", ["default", "repro"])
def test_dropped_relu_mask_breaks_the_backward_bound(path):
    x, gamma, beta, dy = gn_inputs(2, 240, 256, 32, offsets=(0.0,), constants=())
    y, mean, rstd = gn_forward(x, gamma, beta, 32, path, relu=True)
    r = gn_ratios(x, gamma, beta, 32, y, mean, rstd, True, dy, gn_backward(dy, x, y, gamma, mean, rstd, 32, True, "no_mask"))
    assert r["dx"] > em.C_BWD and r["dgamma"] > em.C_PAR and r["dbeta"] > em.C_PAR


def test_removed_clamp_breaks_the_bound():
    """The clamp is what keeps a variance that rounds below -eps finite.  With shifted sums a constant group's sums are
    exactly 0, so the clamp is shown where the rounding happens: the raw sums of a constant group of 10.1 give var = -7e-5;
    clamped, rstd meets its bound; unclamped, it is NaN."""
    x, gamma, beta, _ = gn_inputs(1, 1920, 256, 32, offsets=(0.0,), constants=(10.1,))
    _, _, rstd = gn_forward(x, gamma, beta, 32, "default", algo="raw", mutant="clamp")
    _, _, rstd_nc = gn_forward(x, gamma, beta, 32, "default", algo="raw")
    ok = gn_ratios(x[:, :, 248:], gamma[248:], beta[248:], 1, x[:, :, 248:], torch.zeros(1, 1), rstd[:, 31:])
    bad = gn_ratios(x[:, :, 248:], gamma[248:], beta[248:], 1, x[:, :, 248:], torch.zeros(1, 1), rstd_nc[:, 31:])
    assert ok["rstd"] <= em.C_RSTD
    assert bad["rstd"] > em.C_RSTD


@pytest.mark.parametrize("path", ["default", "repro"])
def test_thread_dependent_shift_breaks_the_bound(path):
    x, gamma, beta, _ = gn_inputs(1, 1920, 256, 32, offsets=(0.0, 30.0), constants=())
    y, mean, rstd = gn_forward(x, gamma, beta, 32, path, mutant="thread_shift")
    r = gn_ratios(x, gamma, beta, 32, y, mean, rstd)
    assert r["mean"] > em.C_MU and r["y"] > em.C_FWD


# ---- LayerNorm: the two-pass row statistics meet the bounds -------------------------------------------------------------------
def warp_sum(v):
    """v[..., 32] lane values -> the xor butterfly's result (every lane ends with the same value; lane 0's is returned)."""
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[..., idx ^ o]
    return v[..., 0]


def ln_forward(z, gamma, beta):
    """add_ln_fwd_kernel on z = x + drop(res): lane l owns float4 i*32 + l; per-lane fp32 chains, butterfly, two passes."""
    M, C = z.shape
    NV = C // 128
    zq = z.view(M, NV, 32, 4)
    s = torch.zeros(M, 32)
    for i in range(NV):
        q = zq[:, i]
        s = s + (((q[..., 0] + q[..., 1]) + q[..., 2]) + q[..., 3])
    mean = warp_sum(s) * torch.tensor(1.0 / C, dtype=F32)
    a = zq - mean.view(M, 1, 1, 1)
    v = torch.zeros(M, 32)
    for i in range(NV):
        q = a[:, i] * a[:, i]
        v = v + (((q[..., 0] + q[..., 1]) + q[..., 2]) + q[..., 3])
    rstd = rsqrt32(warp_sum(v) * torch.tensor(1.0 / C, dtype=F32) + torch.tensor(EPS, dtype=F32))
    y = ((z - mean[:, None]) * rstd[:, None]) * gamma + beta
    return y, mean, rstd


@pytest.mark.parametrize("C", [128, 1024])
@pytest.mark.parametrize("kind", ["plain", "offset", "near_constant"])
def test_layernorm_two_pass_meets_the_bounds(C, kind):
    g = torch.Generator().manual_seed(C)
    M = 257
    z = torch.randn(M, C, generator=g)
    if kind == "offset":
        z = z + 1e3
    elif kind == "near_constant":
        z = 3.0 + 1e-4 * z                                                     # sigma^2 = 1e-8 << eps
    gamma, beta = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    y, mean, rstd = ln_forward(z, gamma, beta)
    y64, mag, mu, rstd64, m, _ = em.forward(em.view4(z), em.param4(gamma), em.param4(beta), EPS)
    r = {"y": _ratio(em.view4(y), y64, mag), "mean": _ratio(mean.view(mu.shape), mu, em.U32 * m),
         "rstd": _ratio(rstd.view(rstd64.shape).to(F64) / rstd64, torch.ones_like(rstd64), torch.full_like(rstd64, em.U32))}
    print(C, kind, {k: f"{v:.2e}" for k, v in r.items()})
    assert all(_within(r).values()), r
