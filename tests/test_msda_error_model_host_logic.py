"""The bounds of tests/msda_error_model.py are sharp, checked without a GPU.  The float64 reference equals the float64 C oracle
where the coordinate is exact in fp32; the fp32 C oracle (a simulation of the generic kernel's arithmetic with the same
coordinate) and a float32 torch simulation meet every bound at exact-edge points, colliding rows and cancelling inputs; a
value-gradient row summed in random orders meets the atomic bound; and each arithmetic mutant of the kernels breaks a bound:
the image test x >= -1, the corner test dropping the last column, one contribution lost from a hot value-gradient row, grad_loc
scaled by H instead of W, a softmax without its max subtraction at logits of +-100, and the last unit of a ragged tail left
unwritten."""
import math

import numpy as np
import pytest
import torch

import msda_error_model as em
from oracle import msda as oracle_msda

F32, F64 = torch.float32, torch.float64
POW2 = [(8, 16), (4, 8), (2, 4), (1, 2), (1, 1)]
SMALL = [(6, 20), (3, 10), (2, 5), (1, 1)]
EDGE_LEVELS = [(5, 7), (1, 6), (4, 1), (2, 2), (4, 8)]


def _ratio(y, ref, mag):
    """Worst |y - ref| / mag, inf when y is not finite or an element with mag == 0 is not exact."""
    y = y.to(F64)
    if not bool(torch.isfinite(y).all()):
        return math.inf
    err = (y - ref).abs()
    pos = mag > 0
    if not bool((err[~pos] == 0).all()):
        return math.inf
    return float((err[pos] / mag[pos]).max()) if bool(pos.any()) else 0.0


def ratios(got, r):
    """{output: worst ratio in units of u (the value gradient per sqrt(n_i))} of the outputs in `got`."""
    return {k: _ratio(y.reshape(r[k].shape), r[k], em.scale(r, k)) for k, y in got.items()}


BOUND = {"out": "C_OUT", "grad_attn": "C_GA", "grad_loc": "C_GL", "grad_value": "C_GV"}


def _within(res):
    return {k: v <= getattr(em, BOUND[k]) for k, v in res.items()}


def _oracle32(ins):
    value, shapes, lsi, loc, attn, grad_out = (t.numpy() for t in ins)
    out = oracle_msda.msda_forward(value, shapes, lsi, loc, attn)
    gv, gl, ga = oracle_msda.msda_backward(value, shapes, lsi, loc, attn, grad_out)
    return {"out": torch.from_numpy(out), "grad_value": torch.from_numpy(gv), "grad_loc": torch.from_numpy(gl),
            "grad_attn": torch.from_numpy(ga)}


# ---- float32 simulation of the generic kernels, with mutants --------------------------------------------------------------------
def simulate(value, shapes, lsi, loc, attn, grad_out, mutant=None):
    """msda_fwd_generic_kernel / msda_bwd_generic_kernel in float32, vectorised over points (per-point sums in fp32 in the
    kernel's order, channel sums in torch's).  Mutants: 'ge_minus1' (image test x >= -1), 'last_column' (corner test
    x0 + 1 < W - 1), 'h_for_w' (grad_loc x of the last level scaled by H), 'lost' (the largest contribution to the hottest
    value-gradient row of the coarsest level is not added)."""
    B, S, M, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    Hs = shapes[:, 0].view(1, 1, 1, L, 1)
    Ws = shapes[:, 1].view(1, 1, 1, L, 1)
    x = em.coord(loc[..., 0], Ws.double()).float()
    y = em.coord(loc[..., 1], Hs.double()).float()
    xin = (x >= -1) if mutant == "ge_minus1" else (x > -1)
    inside = (y > -1) & xin & (y < Hs) & (x < Ws)
    xf = torch.where(inside, torch.floor(x), torch.zeros_like(x))
    yf = torch.where(inside, torch.floor(y), torch.zeros_like(y))
    lx = torch.where(inside, x - xf, torch.zeros_like(x))              # the kernels skip points off the image
    ly = torch.where(inside, y - yf, torch.zeros_like(y))
    hx, hy = 1 - lx, 1 - ly
    x0, y0 = xf.long(), yf.long()
    rig_lim = Ws - 2 if mutant == "last_column" else Ws - 1
    b = torch.arange(B).view(B, 1, 1, 1, 1)
    m = torch.arange(M).view(1, 1, M, 1, 1)
    vf = value.reshape(-1, D)
    vs, ws, rows, oks = [], [], [], []
    for dy, dx, w in ((0, 0, hy * hx), (0, 1, hy * lx), (1, 0, ly * hx), (1, 1, ly * lx)):
        yy, xx = y0 + dy, x0 + dx
        ok = inside & (yy >= 0) & (yy <= Hs - 1) & (xx >= 0) & (xx <= (rig_lim if dx else Ws - 1))
        row = torch.where(ok, (b * S + lsi.view(1, 1, 1, L, 1) + yy * Ws + xx) * M + m, torch.zeros_like(yy))
        vs.append(vf[row] * ok.unsqueeze(-1))
        ws.append(w)
        rows.append(row)
        oks.append(ok)
    a = attn.unsqueeze(-1)
    bil = ((ws[0].unsqueeze(-1) * vs[0] + ws[1].unsqueeze(-1) * vs[1]) + ws[2].unsqueeze(-1) * vs[2]) + ws[3].unsqueeze(-1) * vs[3]
    bil = torch.where(inside.unsqueeze(-1), bil, torch.zeros_like(bil))
    acc = torch.zeros(B, Lq, M, D)
    for l in range(L):
        for p in range(P):
            acc = acc + a[:, :, :, l, p] * bil[:, :, :, l, p]
    got = {"out": acc.reshape(B, Lq, M * D)}
    g = grad_out.view(B, Lq, M, 1, 1, D)
    tg = g * a
    ga = (g * bil).sum(-1)
    gx = (tg * (hy.unsqueeze(-1) * (vs[1] - vs[0]) + ly.unsqueeze(-1) * (vs[3] - vs[2]))).sum(-1)
    gy = (tg * (hx.unsqueeze(-1) * (vs[2] - vs[0]) + lx.unsqueeze(-1) * (vs[3] - vs[1]))).sum(-1)
    zero = torch.zeros_like(ga)
    sx = Ws.float().expand_as(gx).clone()
    if mutant == "h_for_w":
        sx[:, :, :, L - 1] = float(shapes[L - 1, 0])
    got["grad_attn"] = torch.where(inside, ga, zero)
    got["grad_loc"] = torch.stack((torch.where(inside, sx * gx, zero), torch.where(inside, Hs * gy, zero)), -1)
    contrib = torch.stack([(w.unsqueeze(-1) * tg) * ok.unsqueeze(-1) for w, ok in zip(ws, oks)], -2)   # (.., 4, D)
    idx = torch.stack(rows, -1)
    if mutant == "lost":
        lvl = torch.zeros_like(idx, dtype=torch.bool)
        lvl[:, :, :, L - 1] = True
        sel = torch.stack(oks, -1) & lvl
        hot = torch.bincount(idx[sel], minlength=B * S * M).argmax()
        cand = (idx == hot) & sel
        mag = torch.where(cand.unsqueeze(-1), contrib.abs(), torch.zeros_like(contrib))[..., 0]
        drop = mag.reshape(-1).argmax()
        contrib.view(-1, D)[drop] = 0
    gv = torch.zeros(B * S * M, D).index_add_(0, idx.reshape(-1), contrib.reshape(-1, D))
    got["grad_value"] = gv.view(B, S, M, D)
    return got


def _case(kind, shapes=EDGE_LEVELS, B=2, Lq=40, M=3, D=5, P=4, seed=1, edges=True):
    ins, landed = em.make_inputs(shapes, B, Lq, M, D, P, seed, kind=kind, edges=edges)
    return ins, landed


# ---- the reference is the oracle's float64 arithmetic where the coordinate is exact --------------------------------------------
@pytest.mark.parametrize("kind", ["plain", "signed"])
def test_reference_equals_the_float64_oracle_on_exact_coordinates(kind):
    """loc = k / 1024 on power-of-two levels: loc * W - 0.5 is exact in fp32 and in float64, so the reference and the
    float64 C oracle sample the same points and agree to float64 rounding, edges included (k spans x = -1 .. W)."""
    ins, _ = em.make_inputs(POW2, 2, 30, 3, 7, 4, 5, kind=kind, edges=False)
    value, shapes, lsi, loc, attn, grad_out = ins
    g = torch.Generator().manual_seed(9)
    loc = (torch.randint(-40, 1100, loc.shape, generator=g).double() / 1024).contiguous()
    loc.view(-1)[:2 * len(POW2)] = torch.tensor([-32 / 1024, 1056 / 1024] * len(POW2), dtype=F64)    # x = -1, y in (H - 1, H)
    value, attn, grad_out = value.double(), attn.double(), grad_out.double()
    r = em.reference(value, shapes, lsi, loc, attn, grad_out)
    npv = [t.numpy() for t in (value, shapes, lsi, loc, attn)]
    out = torch.from_numpy(oracle_msda.msda_forward(*npv))
    gv, gl, ga = (torch.from_numpy(t) for t in oracle_msda.msda_backward(*npv, grad_out.numpy()))
    assert _ratio(out, r["out"], r["mag_out"]) <= 1e-14
    assert _ratio(gv, r["grad_value"], r["gv_sum"]) <= 1e-14
    assert _ratio(gl, r["grad_loc"], r["mag_gl"]) <= 1e-14
    assert _ratio(ga, r["grad_attn"], r["mag_ga"]) <= 1e-14
    assert bool((r["mag_gl"] == 0).any()) and bool((r["mag_gl"] > 0).any())


def test_coordinate_matches_fmaf_at_the_edges():
    """make_inputs puts points exactly on every edge target of every level (the lines the predicates test)."""
    _, landed = _case("plain", Lq=200)
    print(landed)
    assert bool((landed["x"] > 0).all()) and bool((landed["y"] > 0).all())
    lo, hit = em.loc_for(em.edge_targets(16), 16)
    assert bool(hit.all())                                                   # power of two: every target is reachable
    assert torch.equal(em.coord(lo, 16), em.edge_targets(16))


# ---- simulations meet the bounds ------------------------------------------------------------------------------------------------
KINDS = ["plain", "signed", "offset", "nonfinite", "collide"]


@pytest.mark.parametrize("kind", KINDS)
def test_fp32_oracle_meets_the_bounds(kind):
    ins, _ = _case(kind, Lq=60 if kind != "collide" else 300)
    r = em.reference(*ins)
    res = ratios(_oracle32(ins), r)
    print(kind, {k: f"{v:.2f}" for k, v in res.items()})
    assert all(_within(res).values()), res


@pytest.mark.parametrize("kind", KINDS)
def test_fp32_simulation_meets_the_bounds(kind):
    ins, _ = _case(kind, Lq=60 if kind != "collide" else 300)
    r = em.reference(*ins)
    res = ratios(simulate(*ins), r)
    print(kind, {k: f"{v:.2f}" for k, v in res.items()})
    assert all(_within(res).values()), res


def test_random_order_meets_the_value_gradient_bound():
    """The atomics add a row's contributions in any order: 50 random orders of the hottest row, summed sequentially in
    fp32, all meet C_GV u sqrt(n) S."""
    ins, _ = _case("collide", shapes=SMALL, B=1, Lq=400, M=2, D=8)
    value, shapes, lsi, loc, attn, grad_out = ins
    r = em.reference(*ins)
    S = value.shape[1]
    L, P, M, D = loc.shape[3], loc.shape[4], value.shape[2], value.shape[3]
    w, rows, ok, *_ = em._gather(loc, shapes, lsi, S, M)
    tg = (grad_out.view(1, -1, M, 1, 1, D) * attn.unsqueeze(-1))
    contrib = (w.float().unsqueeze(-1) * tg.unsqueeze(-2))                  # fp32 (w rounded once, then w * tg)
    n = r["gv_n"].reshape(-1, D)[:, 0]
    hot = int(n.argmax())
    c = contrib[(rows == hot) & ok].numpy()
    assert c.shape[0] >= 1000
    g = np.random.default_rng(3)
    worst = 0.0
    ref = r["grad_value"].reshape(-1, D)[hot].numpy()
    mag = em.scale(r, "grad_value").reshape(-1, D)[hot].numpy()
    for _ in range(50):
        s = np.cumsum(c[g.permutation(c.shape[0])], axis=0, dtype=np.float32)[-1]
        worst = max(worst, float((np.abs(s.astype(np.float64) - ref) / mag).max()))
    print("n", c.shape[0], "worst", worst)
    assert worst <= em.C_GV


# ---- mutants break them --------------------------------------------------------------------------------------------------------
def test_image_test_ge_minus_one_breaks_grad_loc():
    ins, landed = _case("plain")
    assert int(landed["x"][0]) > 0                                           # points at x = -1 exactly
    r = em.reference(*ins)
    assert _within(ratios(simulate(*ins), r))["grad_loc"]
    assert ratios(simulate(*ins, mutant="ge_minus1"), r)["grad_loc"] > em.C_GL


def test_dropped_last_column_breaks_out():
    ins, _ = _case("plain")
    r = em.reference(*ins)
    assert ratios(simulate(*ins, mutant="last_column"), r)["out"] > em.C_OUT


def test_lost_contribution_breaks_grad_value():
    ins, _ = _case("collide", shapes=SMALL, B=1, Lq=400, M=2, D=8)
    r = em.reference(*ins)
    assert int(r["gv_n"].max()) >= 1000
    assert _within(ratios(simulate(*ins), r))["grad_value"]
    assert ratios(simulate(*ins, mutant="lost"), r)["grad_value"] > em.C_GV


def test_h_for_w_breaks_grad_loc():
    ins, _ = _case("plain")
    r = em.reference(*ins)
    assert ratios(simulate(*ins, mutant="h_for_w"), r)["grad_loc"] > em.C_GL


@pytest.mark.parametrize("subtract_max", [True, False])
def test_softmax_without_max_overflows_at_logits_of_100(subtract_max):
    """The fused kernels' softmax in fp32: with the max subtracted it meets the pre-processing bound at logits spread over
    +-100 and the outputs stay finite; without it expf overflows (> 88.7) and out is NaN."""
    ins, _ = _case("plain", edges=False)
    value, shapes, lsi, loc, attn, grad_out = ins
    B, Lq, M, L, P = attn.shape
    logits = torch.rand(B, Lq, M, L * P, generator=torch.Generator().manual_seed(4)) * 200 - 100
    z = logits - logits.amax(-1, keepdim=True) if subtract_max else logits
    e = torch.exp(z)
    a32 = (e * (1.0 / e.sum(-1, keepdim=True))).view(attn.shape)
    a64 = em.softmax64(logits.view(B, Lq, -1), M, L, P)
    am = em.softmax_mag(logits.view(B, Lq, -1), M, L, P)
    r = em.reference(value, shapes, lsi, loc, a64, grad_out, attn_mag=am)
    res = ratios({"out": simulate(value, shapes, lsi, loc, a32, grad_out)["out"]}, r)
    ra = _ratio(a32, a64, em.U32 * am + em.ETA)
    if subtract_max:
        assert res["out"] <= em.C_OUT and ra <= em.C_PREP
    else:
        assert res["out"] == math.inf and ra == math.inf


def test_unwritten_tail_unit_leaves_nan():
    """Outputs start as NaN: a kernel that skips the last unit of a ragged tail (B Lq M = 15 units) fails isfinite."""
    ins, _ = _case("plain", B=1, Lq=5, M=3)
    r = em.reference(*ins)
    out = torch.full((1, 5, 3 * 5), math.nan)
    full = simulate(*ins)["out"]
    out[:, :, :] = full
    assert _within(ratios({"out": out}, r))["out"]
    out.view(15, 5)[14] = math.nan
    assert ratios({"out": out}, r)["out"] == math.inf
