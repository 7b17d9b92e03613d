"""The fused head chains (csrc/heads.cu) and the elementwise helpers around the GEMMs (csrc/elementwise.cu) against float64
per element (tests/heads_error_model.py), at their edges: inverse_sigmoid's clamp kinks one ulp either side, saturated
sigmoids, the height clamp at exactly 1, distinct image heights and focal lengths per image, centres on pixel lines and
one ulp / one cell / far outside the map, 1-pixel maps, thousands of queries on one 2x2 patch, weighted depths a few ulps
around integers and at dmax, bins outside [0, dmax], empty cluster ranks, every resize pair up to 48, column sums of one
fp32 chain per lane, and the exact operations bit for bit.

The C entry points are called directly, every output pre-filled with NaN (a random prior where the call accumulates), so
an element a kernel does not write fails.  Every case runs in the default mode and in reproducible mode, where a second
call must give the same bits."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import heads_error_model as em
import monodetr_b200
from monodetr_b200 import _lib, tc

pytestmark = pytest.mark.gpu

F32 = torch.float32
F64 = torch.float64
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst |y-ref|/(u*mag) per constant:")
    for k, (r, case) in sorted(WORST.items()):
        print(f"  {k}: {r:.3e}  ({case})")


@pytest.fixture(params=[False, True], ids=["default", "reproducible"])
def repro(request):
    prev = monodetr_b200.set_deterministic(request.param)
    yield request.param
    monodetr_b200.set_deterministic(prev)


def _check(key, case, y, ref, mag):
    r = em.assert_rel(f"{key} {case}", y, ref, mag, getattr(em, key))
    if r > WORST.get(key, (-1.0, ""))[0]:
        WORST[key] = (r, case)


class _Worst:
    """The worst ratio over many small calls, checked once."""

    def __init__(self):
        self.r, self.case, self.bad = 0.0, "", None

    def add(self, case, y, ref, mag):
        y = y.to(F64)
        if not bool(torch.isfinite(y).all()):
            self.bad = self.bad or f"{case}: not finite"
        err = (y - ref).abs()
        pos = mag > 0
        if bool((err[~pos] != 0).any()):
            self.bad = self.bad or f"{case}: elements with zero magnitude are not exact"
        if bool(pos.any()):
            r = float((err[pos] / mag[pos]).max())
            if r > self.r:
                self.r, self.case = r, case

    def check(self, key, what):
        assert self.bad is None, self.bad
        _check(key, f"{what}, worst at {self.case}", torch.zeros(1), torch.tensor([self.r], dtype=F64), torch.ones(1, dtype=F64))


def _nan(*shape):
    return torch.full(shape, float("nan"), device="cuda")


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _run(fn, repro):
    """fn() -> tuple of outputs; in reproducible mode a second call must give the same bits."""
    out = fn()
    torch.cuda.synchronize()
    if repro:
        again = fn()
        torch.cuda.synchronize()
        for i, (a, b) in enumerate(zip(out, again)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"reproducible mode: output {i} differs between two calls"
    return out


def _f32(v):
    return torch.tensor(v, dtype=F32)


def _next(v, toward):
    return float(torch.nextafter(_f32(v), _f32(toward)))


# ---- box refinement ---------------------------------------------------------------------------------------------------------
def _ref_edges():
    e = float(_f32(1e-5))
    one_e = float(_f32(1.0) - _f32(e))
    vals = [0.0, -0.0, 1.0, e, one_e, 0.5, -0.25, 1.75, -3.0, 4.0, _next(0, -1), _next(1, 2)]
    for v in (e, one_e, 0.0, 1.0):
        vals += [_next(v, -1), _next(v, 2)]
    return torch.tensor(vals, dtype=F32)


@pytest.mark.parametrize("rd", [2, 6])
@pytest.mark.parametrize("n", [1, 37, 4100])
def test_box_refine(rd, n, repro):
    g = _gen(100 * rd + n)
    vals = _ref_edges().cuda()
    ref = torch.rand(n, rd, device="cuda", generator=g)
    flat = ref.view(-1)
    k = min(flat.numel(), 4 * vals.numel())
    flat[:k] = vals[torch.arange(k, device="cuda") % vals.numel()]
    tmp = torch.randn(n, 6, device="cuda", generator=g) * 3
    tmp[1::4] = 30.0
    tmp[2::4] = -30.0
    dy = torch.randn(n, 6, device="cuda", generator=g)

    def fn():
        y = _nan(n, 6)
        _lib.call("mdb_box_refine_forward_f32", tmp, ref, y, n, rd)
        dtmp, dref, dtmp2 = _nan(n, 6), _nan(n, rd), _nan(n, 6)
        _lib.call("mdb_box_refine_backward_f32", dy, y, ref, dtmp, dref, n, rd)
        _lib.call("mdb_box_refine_backward_f32", dy, y, ref, dtmp2, None, n, rd)     # detached reference: no dref
        return y, dtmp, dref, dtmp2

    y, dtmp, dref, dtmp2 = _run(fn, repro)
    case = f"rd={rd} n={n}"
    _check("C_BOX_FWD", case, y, *em.box_refine_fwd(tmp, ref))
    g64, gm, dr64, drm = em.box_refine_bwd(dy, y, ref)
    _check("C_BOX_BWD", case + " dtmp", dtmp, g64, gm)
    _check("C_BOX_BWD", case + " dref", dref, dr64, drm)
    assert torch.equal(dtmp2, dtmp)


# ---- bilinear centres -------------------------------------------------------------------------------------------------------
def _centre_edges(S):
    """Map coordinates in [0, 1] space (0 -> pixel 0, 1 -> pixel S - 1) at the edges of a side of S pixels."""
    cell = 1.0 / max(S - 1, 1)
    vals = [0.0, 1.0, _next(0, -1), _next(1, 2), -cell, 1 + cell, -7.0, 8.0, 0.5]
    vals += [float(_f32(k * cell)) for k in range(0, S, max(1, S // 5))]
    vals += [_next(k * cell, -1) for k in (1, S - 2) if 0 < k < S]
    return torch.tensor(vals, dtype=F32)


def _centres(B, N, H, W, g, patch=False):
    """(B, N, 2) coordinates in [0, 1] space: edge values on both axes cycling through every combination, the rest random."""
    c = torch.rand(B, N, 2, device="cuda", generator=g) * 1.3 - 0.15
    if patch:                                                  # every query inside the cell (x 5..6, y 3..4)
        c[..., 0] = (5 + torch.rand(B, N, device="cuda", generator=g)) / (W - 1)
        c[..., 1] = (3 + torch.rand(B, N, device="cuda", generator=g)) / (H - 1)
        return c
    ex, ey = _centre_edges(W).cuda(), _centre_edges(H).cuda()
    k = torch.arange(B * N, device="cuda")
    m = min(B * N, 2 * ex.numel() * ey.numel())
    c.view(-1, 2)[:m, 0] = ex[k[:m] % ex.numel()]
    c.view(-1, 2)[:m, 1] = ey[(k[:m] // ex.numel()) % ey.numel()]
    return c


def _hn_edges(ih):
    """Box heights hn with fp32(hn * ih) just below, at and just above 1."""
    hn0 = _f32(1.0) / _f32(ih)
    cands = [hn0]
    for _ in range(6):
        cands = [torch.nextafter(cands[0], _f32(0))] + cands + [torch.nextafter(cands[-1], _f32(1))]
    prods = [float(h * _f32(ih)) for h in cands]
    below = max((p, i) for i, p in enumerate(prods) if p < 1)[1]
    above = min((p, i) for i, p in enumerate(prods) if p > 1)[1]
    at = [i for i, p in enumerate(prods) if p == 1]
    return [float(cands[i]) for i in [below, above] + at]


HD_CASES = [(8, 300, 24, 80, False), (3, 50, 1, 9, False), (2, 40, 7, 1, False), (1, 5, 1, 1, False), (2, 0, 24, 80, False),
            (1, 4096, 24, 80, True)]


@pytest.mark.parametrize("B,N,H,W,patch", HD_CASES)
def test_head_depth(B, N, H, W, patch, repro):
    g = _gen(B * 1000 + N + H)
    coord = torch.rand(B, N, 6, device="cuda", generator=g) * 0.1
    coord[..., :2] = _centres(B, N, H, W, g, patch)
    ih = torch.tensor([375.0 - 7 * b for b in range(B)], device="cuda")
    sizes = torch.stack((torch.full((B,), 1242.0, device="cuda"), ih), -1)
    calibs = torch.zeros(B, 3, 4, device="cuda")
    calibs[:, 0, 0] = torch.tensor([700.0 + 13.5 * b for b in range(B)], device="cuda")
    for b in range(B):                                          # the height clamp at exactly 1 and one ulp either side
        hs = _hn_edges(float(ih[b]))
        for j, hn in enumerate(hs[:N]):
            coord[b, j, 4], coord[b, j, 5] = hn, 0.0
        if N > len(hs):
            coord[b, len(hs), 4:] = 1e-4
    size3d = torch.randn(B, N, 3, device="cuda", generator=g) + 1.5
    reg = torch.randn(B, N, 2, device="cuda", generator=g)
    reg.view(-1, 2)[3::7, 0] = 20.0
    reg.view(-1, 2)[5::7, 0] = -20.0
    wd = torch.rand(B, H, W, device="cuda", generator=g) * 60
    dout = torch.randn(B, N, 2, device="cuda", generator=g)

    def fn():
        out = _nan(B, N, 2)
        _lib.call("mdb_head_depth_forward_f32", coord, size3d, reg, wd, calibs, sizes, out, B, N, H, W)
        dc, ds, dr, dm = _nan(B, N, 6), _nan(B, N, 3), _nan(B, N, 2), _nan(B, H, W)
        _lib.call("mdb_head_depth_backward_f32", dout, coord, size3d, reg, calibs, sizes, dc, ds, dr, dm, B, N, H, W)
        return out, dc, ds, dr, dm

    out, dc, ds, dr, dm = _run(fn, repro)
    case = f"B={B} N={N} H={H} W={W}" + (" patch" if patch else "")
    if N:
        _check("C_HD_FWD", case, out[..., 0], *em.head_depth_fwd(coord, size3d, reg, wd, calibs, sizes))
        assert torch.equal(out[..., 1], reg[..., 1])
    r = em.head_depth_bwd(dout, coord, size3d, reg, calibs, sizes, H, W)
    assert bool((dc[..., :4] == 0).all()) and bool((ds[..., 1:] == 0).all())
    if N:
        _check("C_HD_BWD", case + " dcoord4", dc[..., 4], *r["dhn"])
        _check("C_HD_BWD", case + " dcoord5", dc[..., 5], *r["dhn"])
        _check("C_HD_BWD", case + " dsize0", ds[..., 0], *r["dsize0"])
        _check("C_HD_BWD", case + " dreg0", dr[..., 0], *r["dreg0"])
        assert torch.equal(dr[..., 1], dout[..., 1])
    _check("C_HD_MAP", case + " dmap", dm, *r["dmap"])


# ---- depth-map lookup (grid_sample) ---------------------------------------------------------------------------------------
DS_CASES = [(2, 24, 80, 500, False), (1, 1, 1, 7, False), (3, 1, 9, 50, False), (2, 7, 1, 50, False), (1, 24, 80, 4096, True)]


@pytest.mark.parametrize("B,H,W,N,patch", DS_CASES)
def test_depth_sample(B, H, W, N, patch, repro):
    g = _gen(B * 7 + H * 3 + N)
    xy = _centres(B, N, H, W, g, patch) * 2 - 1
    depth = torch.rand(B, H, W, device="cuda", generator=g) * 60
    dout = torch.randn(B, N, device="cuda", generator=g)

    def fn():
        out, dd = _nan(B, N), _nan(B, H, W)
        _lib.call("mdb_depth_sample_forward_f32", depth, xy, out, B, H, W, N)
        _lib.call("mdb_depth_sample_backward_f32", dout, xy, dd, B, H, W, N)
        return out, dd

    out, dd = _run(fn, repro)
    case = f"B={B} H={H} W={W} N={N}" + (" patch" if patch else "")
    u = em.grid_xy32(xy)
    x0, y0, lx, ly = em.corners(u[..., 0], u[..., 1], H, W)
    if N:
        v, m = em.bilinear_fwd(depth, x0, y0, lx, ly)
        _check("C_SAMPLE_FWD", case, out, v, em.U32 * m)
    v, m = em.bilinear_bwd(dout, x0, y0, lx, ly, H, W)
    _check("C_SAMPLE_BWD", case + " ddepth", dd, v, em.U32 * m)


# ---- depth predictor tail -----------------------------------------------------------------------------------------------------
def _model_bins(nb, dmax):
    """depth_predictor.py's LID bins: nb - 1 centres in (0, dmax) and dmax."""
    if nb == 1:
        return torch.tensor([dmax * 0.37], dtype=F32)
    idx = torch.linspace(0, nb - 2, nb - 1)
    bs = 2 * (dmax - 1e-3) / ((nb - 1) * nb)
    return torch.cat(((idx + 0.5).pow(2) * bs / 2 - bs / 8 + 1e-3, torch.tensor([dmax])))


def _dt_inputs(npix, nb, E, kind, g):
    """(logits (npix, nb), bins (nb,), dmax) for the kinds: edges, flat, alternate, own."""
    dmax = float(E - 1)
    if kind == "own":                                          # bins outside [0, dmax]; dmax short of E - 1 so that e1 != e0
        dmax = E - 1.5
        bins = torch.linspace(-5.0, dmax + 5.0, nb)[torch.randperm(nb, generator=torch.Generator().manual_seed(nb))]
        if nb == 1:
            bins = torch.tensor([dmax + 2.0])
        logits = torch.randn(npix, nb, generator=torch.Generator().manual_seed(npix + nb)) * 8
        return logits.cuda(), bins.cuda(), dmax
    bins = _model_bins(nb, dmax)
    if kind == "flat":
        return torch.zeros(npix, nb, device="cuda"), bins.cuda(), dmax
    if kind == "alternate":
        lg = torch.full((npix, nb), -30.0)
        lg[0::2, nb // 3] = 0.0
        lg[1::2, (2 * nb) // 3] = 0.0
        lg[:, nb - 1] = -2.0
        return lg.cuda(), bins.cuda(), dmax
    rows = list(em.edge_logits(bins, dmax)) if nb > 32 else []
    last = torch.full((nb,), -30.0)                            # all mass on the last bin: wd == dmax, fi == ci == E - 1
    last[-1] = 0.0
    rows.append(last)
    n_rand = max(npix - len(rows), 0)
    lg = torch.cat([torch.stack(rows)[:npix], torch.randn(n_rand, nb, generator=torch.Generator().manual_seed(nb)) * 3])
    return lg.cuda(), bins.cuda(), dmax


DT_CASES = [(15360, 81, 61, 256, "edges"), (15360, 81, 61, 256, "flat"), (15360, 81, 61, 256, "alternate"),
            (15360, 96, 61, 132, "own"), (15360, 33, 61, 128, "edges"), (7, 33, 61, 128, "edges"), (15, 32, 2, 4, "edges"),
            (1, 1, 2, 4, "edges"), (1, 81, 61, 256, "edges"), (0, 81, 61, 256, "edges"), (15, 96, 61, 256, "own"),
            (7, 1, 61, 132, "own"), (15360, 81, 2, 4, "edges")]


@pytest.mark.parametrize("npix,nb,E,C,kind", DT_CASES)
def test_depth_tail(npix, nb, E, C, kind, repro):
    g = _gen(npix + nb + E + C)
    logits, bins, dmax = _dt_inputs(npix, nb, E, kind, g)
    emb = torch.randn(E, C, device="cuda", generator=g)
    d_ip = torch.randn(npix, C, device="cuda", generator=g)
    d_wd = torch.randn(npix, device="cuda", generator=g)
    zeros = torch.zeros(npix, C, device="cuda")
    bwd_launches = 2 if repro else 1

    def fn():
        wd, ip = _nan(npix), _nan(npix, C)
        _lib.call("mdb_depth_tail_forward_f32", logits, bins, emb, wd, ip, npix, nb, E, C, dmax)
        outs = [wd, ip]
        for dip, dwd in ((d_ip, d_wd), (d_ip, None), (zeros, d_wd)):    # both, only d_ip, only d_wd
            dl, de = _nan(npix, nb), _nan(E, C)
            _lib.call("mdb_depth_tail_backward_f32", logits, bins, emb, dip, dwd, dl, de, npix, nb, E, C, dmax,
                      launches=bwd_launches)
            outs += [dl, de]
        return tuple(outs)

    outs = _run(fn, repro)
    wd, ip = outs[:2]
    case = f"npix={npix} nb={nb} E={E} C={C} {kind}"
    (w64, wm), (i64, im) = em.depth_tail_fwd(logits, bins, emb, wd, dmax)
    _check("C_DT_WD", case, wd, w64, wm)
    _check("C_DT_IP", case, ip, i64, im)
    for (dip, dwd, what), dl, de in zip(((d_ip, d_wd, "both"), (d_ip, None, "d_ip only"), (zeros, d_wd, "d_wd only")),
                                         outs[2::2], outs[3::2]):
        (l64, lm), (e64, emag) = em.depth_tail_bwd(logits, bins, emb, dip, dwd, wd, dmax)
        _check("C_DT_DLOGITS", f"{case} {what}", dl, l64, lm)
        _check("C_DT_DEMB", f"{case} {what}", de, e64, emag)
    if kind == "edges" and npix == 15360 and E == 61:             # the construction reached the integers and dmax
        x = wd.clamp(0, dmax)
        near = (x - x.round()).abs() <= 4 * torch.finfo(F32).eps * x.clamp(min=1)
        assert int(near.sum()) >= 100 and int((x == dmax).sum()) >= 2


# ---- sum_k mean(x_k^2) -------------------------------------------------------------------------------------------------------
SMS_CASES = [[1], [7], [1, 7, 1_200_000] * 10 + [1, 7], [20_900_001, 7]]


@pytest.mark.parametrize("ns", SMS_CASES, ids=["1", "7", "32", "20.9M"])
def test_sum_mean_squares(ns, repro):
    g = _gen(len(ns) + ns[0])
    xs = [torch.randn(n, device="cuda", generator=g) + (3.0 if k % 3 == 0 else 0.0) for k, n in enumerate(ns)]
    count = len(xs)
    nums = (ctypes.c_longlong * count)(*ns)
    dloss = torch.tensor(1.7, device="cuda")

    def fn():
        loss = _nan()
        _lib.call("mdb_sum_mean_squares_forward_f32", count, xs, nums, loss)
        gs = [_nan(n) for n in ns]
        _lib.call("mdb_sum_mean_squares_backward_f32", count, xs, gs, nums, dloss)
        return (loss, *gs)

    loss, *gs = _run(fn, repro)
    (l64, lm), grads = em.sum_mean_squares(xs, dloss)
    case = f"count={count} n_max={max(ns)}"
    _check("C_SMS_FWD", case, loss, l64, lm)
    for gk, (r, m) in zip(gs, grads):
        _check("C_SMS_BWD", case, gk, r, m)


# ---- mean3, scale: bit-exact --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4, 1000, 2 * 24 * 80 * 256])
def test_mean3_scale_exact(n, repro):
    g = _gen(n)
    a, b, c, dy = (torch.randn(n, device="cuda", generator=g) * 1e3 for _ in range(4))
    a[:4] = torch.tensor([1e-40, -3e38, 0.0, -0.0])
    b[:4] = torch.tensor([2e-40, -3e38, -0.0, -0.0])
    dy[:4] = torch.tensor([1e-40, 3e38, -0.0, 7.0])

    def fn():
        o, s = _nan(n), _nan(n)
        _lib.call("mdb_mean3_f32", a, b, c, o, n)
        _lib.call("mdb_scale_f32", dy, s, n, 1.0 / 3.0)
        return o, s

    o, s = _run(fn, repro)
    ac, bc, cc, dc = (t.cpu() for t in (a, b, c, dy))
    assert torch.equal(o.cpu().view(torch.int32), ((ac + bc + cc) / torch.full_like(ac, 3.0)).view(torch.int32))
    assert torch.equal(s.cpu().view(torch.int32), (dc * torch.tensor(1.0 / 3.0, dtype=F32)).view(torch.int32))


# ---- stem and max-pool -----------------------------------------------------------------------------------------------------
SIDES = [1, 2, 6, 7, 8, 63, 64, 65]


def _stem_params(g):
    w = torch.randn(64, 3, 7, 7, device="cuda", generator=g) / 147 ** 0.5
    scale = torch.rand(64, device="cuda", generator=g) + 0.5
    scale[::3] *= -1                                          # negative FrozenBN scales
    bias = torch.randn(64, device="cuda", generator=g)
    return w, scale, bias


def _stem(x, w, scale, bias):
    B, _, H, W = x.shape
    Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
    y = _nan(B, Ho, Wo, 64)
    _lib.call("mdb_stem_conv7x7_bn_relu_f32", x, w, scale, bias, y, B, H, W)
    return y


def _pool(y):
    B, H, W, C = y.shape
    p = _nan(B, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C)
    _lib.call("mdb_maxpool3x3s2_nhwc_f32", y, p, B, H, W, C)
    return p


def _stem_case(B, H, W, g, repro, wk):
    x = torch.randn(B, 3, H, W, device="cuda", generator=g)
    w, scale, bias = _stem_params(g)
    prev = tc.get_precision()
    try:
        tc.set_precision("tf32x3")
        y, p = _run(lambda: (lambda yy: (yy, _pool(yy)))(_stem(x, w, scale, bias)), repro)
        tc.set_precision("tf32")                               # the stem then rounds its output to TF32 for its consumer
        (yr,) = _run(lambda: (_stem(x, w, scale, bias),), repro)
    finally:
        tc.set_precision(prev)
    ref, mag = em.stem(x, w, scale, bias)
    wk.add(f"B={B} H={H} W={W}", y, ref, mag)
    assert torch.equal(yr.view(torch.int32), em.round_tf32(y).view(torch.int32)), f"tf32 stem H={H} W={W}"
    assert torch.equal(p.permute(0, 3, 1, 2), F.max_pool2d(y.permute(0, 3, 1, 2), 3, 2, 1)), f"max-pool H={H} W={W}"


@pytest.mark.parametrize("H", SIDES)
def test_stem_and_maxpool(H, repro):
    g = _gen(H)
    wk = _Worst()
    for W in SIDES:
        _stem_case(3, H, W, g, repro, wk)
    wk.check("C_STEM", f"H={H}")


def test_stem_full_size(repro):
    wk = _Worst()
    _stem_case(3, 384, 1280, _gen(1), repro, wk)
    wk.check("C_STEM", "384x1280")


@pytest.mark.parametrize("C", [4, 68, 256])
@pytest.mark.parametrize("H,W", [(1, 1), (2, 7), (65, 64), (96, 320)])
def test_maxpool_channels(C, H, W, repro):
    x = torch.randn(2, H, W, C, device="cuda", generator=_gen(C + H))
    (p,) = _run(lambda: (_pool(x),), repro)
    assert torch.equal(p.permute(0, 3, 1, 2), F.max_pool2d(x.permute(0, 3, 1, 2), 3, 2, 1))


# ---- bilinear resize -------------------------------------------------------------------------------------------------------------
def _resize(x, Ho, Wo):
    B, Hi, Wi, C = x.shape
    y = _nan(B, Ho, Wo, C)
    _lib.call("mdb_upsample_bilinear_nhwc_forward_f32", x, y, B, Hi, Wi, Ho, Wo, C)
    return y


def _resize_bwd(dy, Hi, Wi):
    B, Ho, Wo, C = dy.shape
    dx = _nan(B, Hi, Wi, C)
    _lib.call("mdb_upsample_bilinear_nhwc_backward_f32", dy, dx, B, Hi, Wi, Ho, Wo, C)
    return dx


@pytest.mark.parametrize("axis", ["H", "W"])
def test_resize_every_pair(axis, repro):
    """Every (in, out) pair in 1..48 on one axis, the other axis 3 -> 5, C = 4: up- and downscales."""
    g = _gen(7 if axis == "H" else 8)
    wf, wb = _Worst(), _Worst()
    for n_in in range(1, 49):
        shape = (1, n_in, 3, 4) if axis == "H" else (1, 3, n_in, 4)
        x = torch.randn(*shape, device="cuda", generator=g)
        for n_out in range(1, 49):
            Ho, Wo = (n_out, 5) if axis == "H" else (5, n_out)
            dy = torch.randn(1, Ho, Wo, 4, device="cuda", generator=g)
            y, dx = _run(lambda: (_resize(x, Ho, Wo), _resize_bwd(dy, shape[1], shape[2])), repro)
            case = f"{axis}: {n_in} -> {n_out}"
            wf.add(case, y.cpu(), *em.resize_fwd(x.cpu(), Ho, Wo))
            wb.add(case, dx.cpu(), *em.resize_bwd(dy.cpu(), shape[1], shape[2]))
    wf.check("C_RESIZE_FWD", f"axis {axis}")
    wb.check("C_RESIZE_BWD", f"axis {axis}")


@pytest.mark.parametrize("src,dst", [((12, 40), (24, 80)), ((6, 20), (12, 40))])
def test_resize_model_pairs(src, dst, repro):
    g = _gen(src[0])
    x = torch.randn(2, *src, 256, device="cuda", generator=g)
    dy = torch.randn(2, *dst, 256, device="cuda", generator=g)
    y, dx = _run(lambda: (_resize(x, *dst), _resize_bwd(dy, *src)), repro)
    case = f"{src} -> {dst}"
    _check("C_RESIZE_FWD", case, y, *em.resize_fwd(x, *dst))
    _check("C_RESIZE_BWD", case, dx, *em.resize_bwd(dy, *src))


# ---- column sums ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [0, 1, 7, 8, 9, 511, 512, 513, 81600])
@pytest.mark.parametrize("acc", [0, 1])
def test_colsum(M, acc, repro):
    g = _gen(M + acc)
    wk = _Worst()
    for N in (1, 31, 32, 33, 256, 1025):
        x = torch.randn(max(M, 1), N, device="cuda", generator=g) + 1.0  # a positive mean: partial sums grow along each chain
        prior = torch.randn(N, device="cuda", generator=g) * 100

        def fn():
            out = prior.clone() if acc else _nan(N)
            _lib.call("mdb_colsum_f32", x, out, M, N, acc)
            return (out,)

        (out,) = _run(fn, repro)
        wk.add(f"M={M} N={N} acc={acc}", out, *em.colsum(x[:M], prior if acc else None))
    wk.check("C_COLSUM", f"M={M} acc={acc}")


# ---- relu_backward, round_tf32: bit-exact ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1.0, 1.0 / 0.9])
def test_relu_backward_exact(scale, repro):
    g = _gen(3)
    ys = torch.tensor([0.0, -0.0, 1.401298464324817e-45, 1.0, -1.0, -1.401298464324817e-45, 3e38, -3e38], device="cuda")
    n = 4096
    y = ys[torch.arange(n, device="cuda") % ys.numel()]
    dy = torch.randn(n, device="cuda", generator=g) * 1e3
    dy[::9] = 3e38
    dy[1::11] = -0.0

    def fn():
        o = _nan(n)
        _lib.call("mdb_relu_backward_f32", dy, y, o, n, scale)
        return (o,)

    (o,) = _run(fn, repro)
    assert torch.equal(o.view(torch.int32), em.relu_backward(dy, y, scale).view(torch.int32))


def _tf32_patterns():
    bits = []
    for base in (0x3F800000, 0x40490000, 0x00000000, 0x00400000, 0x7F000000, 0x01000000):   # normal, denormal, large, small
        for low in (0x0FFF, 0x1000, 0x1001, 0x0000, 0x1FFF, 0x3000, 0x2FFF):
            bits.append(base | low)
    bits += [0x3FFFF000, 0x3FFFFFFF, 0x007FF000, 0x007FFFFF, 0x00000001, 0x00001000,     # carries into the exponent; denormals
             0x7F7FE000, 0x7F7FEFFF, 0x7F7FF000, 0x7F7FFFFF,                                # the top of the finite range
             0x7F800000, 0x7FC00000, 0x7F800001, 0x7FFFFFFF]                                # inf, NaN
    bits += [b | 0x80000000 for b in bits]
    t = torch.tensor([b - (1 << 32) if b >= 1 << 31 else b for b in bits], dtype=torch.int32)
    rnd = torch.randint(-(1 << 31), 1 << 31, (1 << 20,), generator=torch.Generator().manual_seed(5), dtype=torch.int64)
    return torch.cat((t, rnd.to(torch.int32))).view(F32)


def test_round_tf32_exact(repro):
    x = _tf32_patterns().cuda()
    n = x.numel()

    def fn():
        o = _nan(n)
        _lib.call("mdb_round_tf32_f32", x, o, n)
        return (o,)

    (o,) = _run(fn, repro)
    got, ref = o.cpu(), em.round_tf32(x.cpu())
    nan = torch.isnan(x.cpu())                                       # a NaN's output bits are not pinned
    assert torch.equal(got[~nan].view(torch.int32), ref[~nan].view(torch.int32))
    top = torch.tensor([0x7F7FEFFF, 0x7F7FF000, 0x7F7FFFFF], dtype=torch.int32).view(F32)   # pinned: no saturation
    assert em.round_tf32(top).tolist() == [float.fromhex("0x1.ffcp+127"), float("inf"), float("inf")]


# ---- documented refusals ---------------------------------------------------------------------------------------------------------
def _refused(name, out, *args):
    out.fill_(7.0)
    with pytest.raises(RuntimeError):
        _lib.call(name, *args)
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()), f"{name} wrote its output although it refused the call"


def test_refusals(repro):
    a = torch.randn(64, device="cuda")
    o = torch.empty(64, device="cuda")
    _refused("mdb_mean3_f32", o, a, a, a, o, 6)
    _refused("mdb_scale_f32", o, a, o, 6, 0.5)
    _refused("mdb_relu_backward_f32", o, a, a, o, 6, 1.0)
    x = torch.randn(1, 4, 4, 6, device="cuda")
    y = torch.empty(1, 8, 8, 6, device="cuda")
    _refused("mdb_upsample_bilinear_nhwc_forward_f32", y, x, y, 1, 4, 4, 8, 8, 6)
    _refused("mdb_upsample_bilinear_nhwc_backward_f32", x, y, x, 1, 4, 4, 8, 8, 6)
    _refused("mdb_maxpool3x3s2_nhwc_f32", y, x, y, 1, 4, 4, 6)
    npix = 8
    lg, bins, emb = torch.randn(npix * 97, device="cuda"), torch.rand(97, device="cuda"), torch.randn(97 * 260, device="cuda")
    wd, ip, dip = torch.empty(npix, device="cuda"), torch.empty(npix * 260, device="cuda"), torch.randn(npix * 260, device="cuda")
    dl, de = torch.empty(npix * 97, device="cuda"), torch.empty(97 * 260, device="cuda")
    for nb, E, C in ((97, 61, 256), (81, 61, 260), (81, 61, 6)):
        _refused("mdb_depth_tail_forward_f32", ip, lg, bins, emb, wd, ip, npix, nb, E, C, 1.0)
    for nb, E, C in ((97, 61, 256), (81, 61, 260), (81, 61, 6), (81, 97, 256)):          # E * C * 4 > 96 KiB last
        _refused("mdb_depth_tail_backward_f32", de, lg, bins, emb, dip, None, dl, de, npix, nb, E, C, 1.0)
    xs = [a] * 33
    loss = torch.empty((), device="cuda")
    _refused("mdb_sum_mean_squares_forward_f32", loss, 33, xs, (ctypes.c_longlong * 33)(*([64] * 33)), loss)
    gs = [torch.empty(64, device="cuda") for _ in range(33)]
    _refused("mdb_sum_mean_squares_backward_f32", gs[0], 33, xs, gs, (ctypes.c_longlong * 33)(*([64] * 33)), loss)
