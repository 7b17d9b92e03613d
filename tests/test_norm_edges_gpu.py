"""LayerNorm and GroupNorm (csrc/norm.cu) against float64 per element (tests/norm_error_model.py), at the shapes and inputs
where normalisation kernels go wrong: one row or pixel, rows that leave cluster ranks of ln_param_grad_kernel empty, the
grid-stride wrap at 81600 rows, pixel counts just past a block and at the 64-block cap, group offsets of 30 and 1000,
constant groups (y must be beta bit for bit), rows with sigma^2 << eps, ReLU outputs that are exactly 0, accumulation into
dgamma / dbeta.  Every case runs in the default mode and twice in reproducible mode (the two bit-identical); each result
meets the bounds on its own."""
import pytest
import torch

import monodetr_b200
import norm_error_model as em
from monodetr_b200 import _lib, functional as Fn, kernels as K

pytestmark = pytest.mark.gpu

F64 = torch.float64
EPS = 1e-5


def _modes(fn):
    """{'default': fn(), 'reproducible': fn()} with a second reproducible call that must give the same bits."""
    prev = monodetr_b200.set_deterministic(False)
    try:
        d = fn()
        monodetr_b200.set_deterministic(True)
        a, b = fn(), fn()
    finally:
        monodetr_b200.set_deterministic(prev)
    for i, (u, v) in enumerate(zip(a, b)):                            # bits, so that two NaNs compare equal
        assert torch.equal(u.view(torch.int32), v.view(torch.int32)), f"reproducible mode: output {i} differs between two calls"
    return {"default": d, "reproducible": a}


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ---- LayerNorm forward -------------------------------------------------------------------------------------------------------
def _ln_inputs(M, C, kind, g):
    x = torch.randn(M, C, device="cuda", generator=g)
    r = torch.randn(M, C, device="cuda", generator=g)
    if kind == "offset":
        x = x + 1e3
    elif kind == "near_constant":                                    # sigma^2 ~ 2e-8 << eps
        x, r = 3.0 + 1e-4 * x, 1e-4 * r
    return x, r


@pytest.mark.parametrize("M", [1, 7, 8, 9, 4097, 81600])
@pytest.mark.parametrize("C", [128, 256, 512, 1024])
def test_layernorm_forward(M, C):
    g = _gen(M * 7 + C)
    gamma, beta = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g)
    g4, b4 = em.param4(gamma), em.param4(beta)
    for kind in ("plain", "offset", "near_constant"):
        x, r = _ln_inputs(M, C, kind, g)
        for res in (None, r):
            outs = _modes(lambda: K.add_layernorm_forward(x, res, gamma, beta, EPS))
            z = (x + res if res is not None else x).to(F64)            # the fp32 sum the kernel normalises
            y64, mag, mu, rstd64, m, _ = em.forward(em.view4(z), g4, b4, EPS)
            for mode, (y, mean, rstd) in outs.items():
                name = f"LN fwd M={M} C={C} {kind} res={res is not None} [{mode}]"
                em.assert_rel(name + " y", em.view4(y), y64, mag, em.C_FWD)
                em.check_stats(name, mean, rstd, mu, rstd64, m)


# ---- LayerNorm backward ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [1, 3, 7, 8, 9, 1000, 81600])
@pytest.mark.parametrize("C", [128, 256, 512])
def test_layernorm_backward(M, C):
    g = _gen(M * 5 + C)
    x, r, dy = (torch.randn(M, C, device="cuda", generator=g) for _ in range(3))
    gamma, beta = torch.rand(C, device="cuda", generator=g) + 0.5, torch.randn(C, device="cuda", generator=g)
    prior_g, prior_b = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)
    seed = torch.tensor([4321], dtype=torch.int64, device="cuda")
    site = 11
    g4 = em.param4(gamma)
    for drop_p in (0.0, 0.1):
        sd = seed if drop_p > 0 else None
        # the kernels' keep mask is mdb_dropout_f32's: the same hash of (seed, site, float4 index) and the same 1/(1-p)
        mask = Fn.dropout_raw(torch.ones_like(x), drop_p, site, seed) if drop_p > 0 else torch.ones_like(x)
        dropped = r * mask
        _, mean, rstd = K.add_layernorm_forward(x, r, gamma, beta, EPS, drop_p, site, sd)

        def run():
            dx, dres, dg, db = K.add_layernorm_backward(dy, x, r, gamma, mean, rstd, drop_p, site, sd)
            dx2 = torch.empty_like(x)
            dres2 = torch.empty_like(x) if drop_p > 0 else None
            ag, ab = prior_g.clone(), prior_b.clone()
            _lib.call("mdb_add_layernorm_backward_f32", dy, x, r, gamma, mean, rstd, dx2, dres2, ag, ab, M, C, drop_p, sd, site, 1,
                      launches=2 if _lib.deterministic() else 1)
            return dx, dres, dg, db, dx2, ag, ab

        outs = _modes(run)
        z = (x + dropped).to(F64)
        _, _, mu, rstd64, m, xh = em.forward(em.view4(z), g4, em.param4(beta), EPS)
        dx64, mag_dx, dxh, mag_dg, mag_db = em.backward(em.view4(dy), g4, rstd64, m, xh)
        dg64, db64 = em.param_sum(dxh), dy.to(F64).sum(0)
        mg, mb = em.param_sum(mag_dg), em.param_sum(mag_db)
        for mode, (dx, dres, dg, db, dx2, ag, ab) in outs.items():
            name = f"LN bwd M={M} C={C} p={drop_p} [{mode}]"
            em.assert_rel(name + " dx", em.view4(dx), dx64, mag_dx, em.C_BWD)
            assert torch.equal(dx2, dx), name                          # accumulate only changes dgamma / dbeta
            if drop_p > 0:
                assert torch.equal(dres, dx * mask), name             # the same mask as mdb_dropout_f32
            em.assert_rel(name + " dgamma", dg, dg64, mg, em.C_PAR)
            em.assert_rel(name + " dbeta", db, db64, mb, em.C_PAR)
            pg, pb = prior_g.to(F64), prior_b.to(F64)
            em.assert_rel(name + " dgamma (accumulate)", ag, pg + dg64, mg + em.U32 * pg.abs(), em.C_PAR)
            em.assert_rel(name + " dbeta (accumulate)", ab, pb + db64, mb + em.U32 * pb.abs(), em.C_PAR)


@pytest.mark.parametrize("C", [128, 256, 512])
def test_layernorm_backward_without_rows(C):
    """M = 0: dgamma / dbeta are zero-filled without accumulate and left untouched with it, in both modes."""
    t = torch.zeros(4 * C, device="cuda")
    gamma = torch.ones(C, device="cuda")
    prev = monodetr_b200.set_deterministic(False)
    try:
        for det in (False, True):
            monodetr_b200.set_deterministic(det)
            for acc in (0, 1):
                dg, db = torch.full((C,), 7.0, device="cuda"), torch.full((C,), -3.0, device="cuda")
                _lib.call("mdb_add_layernorm_backward_f32", t, t, None, gamma, t, t, t, None, dg, db, 0, C, 0.0, None, 0, acc,
                          launches=0)
                torch.cuda.synchronize()
                assert torch.equal(dg, torch.full_like(dg, 7.0 if acc else 0.0)), (det, acc)
                assert torch.equal(db, torch.full_like(db, -3.0 if acc else 0.0)), (det, acc)
    finally:
        monodetr_b200.set_deterministic(prev)


@pytest.mark.parametrize("det", [False, True])
def test_layernorm_unsupported_widths_raise(det):
    prev = monodetr_b200.set_deterministic(det)
    try:
        for C in (96, 1024):
            x = torch.randn(8, C, device="cuda")
            gamma = torch.ones(C, device="cuda")
            mean, rstd = torch.zeros(8, device="cuda"), torch.ones(8, device="cuda")
            with pytest.raises(RuntimeError, match="mdb_add_layernorm_backward_f32"):
                K.add_layernorm_backward(x, x, None, gamma, mean, rstd)
        x = torch.randn(8, 96, device="cuda")
        with pytest.raises(RuntimeError, match="mdb_add_layernorm_forward_f32"):
            K.add_layernorm_forward(x, None, torch.ones(96, device="cuda"), torch.zeros(96, device="cuda"))
    finally:
        monodetr_b200.set_deterministic(prev)


# ---- GroupNorm ---------------------------------------------------------------------------------------------------------------
# (C, G, HW, B): every (C, G) of the model's necks and depth predictor and the kernels' limits, at one pixel, three, a block
# boundary +- 1 (255, 257), the level-0 map (7680) and 16385 = 64 blocks of a ragged 257 pixels (the default mode's cap).
GN_CASES = [(64, 8, 1, 9), (64, 16, 3, 2), (128, 32, 255, 1), (256, 32, 257, 9), (256, 8, 7680, 2), (512, 32, 16385, 2),
            (1024, 32, 3, 9), (1024, 256, 257, 1), (256, 32, 16385, 1), (1024, 32, 16385, 1), (512, 32, 1, 2), (128, 32, 7680, 9),
            (64, 8, 16385, 9), (1024, 256, 255, 2)]
OFFSETS = (0.0, 30.0, 1000.0)


def _gn_inputs(C, G, HW, B, g):
    """randn with group offsets cycling through 0 / 30 / 1000 (shifted by one group per image); group G-1 of image 0 is
    constant 10.1 and group 0 of the last image constant 30.1.  Returns x, gamma, beta, dy and the constant (b, g) list."""
    cpg = C // G
    x = torch.randn(B, HW, G, cpg, device="cuda", generator=g)
    off = torch.tensor([[OFFSETS[(gi + b) % 3] for gi in range(G)] for b in range(B)], device="cuda")
    x = x + off.view(B, 1, G, 1)
    const = [(0, G - 1, 10.1), (B - 1, 0, 30.1)]
    for b, gi, c in const:
        x[b, :, gi] = c
    gamma = torch.rand(C, device="cuda", generator=g) + 0.5
    beta = torch.randn(C, device="cuda", generator=g)
    dy = torch.randn(B, HW, C, device="cuda", generator=g)
    return x.view(B, HW, C).contiguous(), gamma, beta, dy, [(b, gi) for b, gi, _ in const]


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("C,G,HW,B", GN_CASES)
def test_groupnorm(C, G, HW, B, relu):
    g = _gen(C * 131 + G * 17 + HW + B)
    x, gamma, beta, dy, const = _gn_inputs(C, G, HW, B, g)
    cpg = C // G

    def run():
        y, mean, rstd = K.groupnorm_forward(x, gamma, beta, G, EPS, relu)
        dx, dg, db = K.groupnorm_backward(dy, x, y, gamma, mean, rstd, G, relu)
        return y, mean, rstd, dx, dg, db

    outs = _modes(run)
    g4, b4 = em.param4(gamma, G), em.param4(beta, G)
    y64, mag, mu, rstd64, m, xh = em.forward(em.view4(x, G), g4, b4, EPS)
    yr64 = y64.clamp_min(0.0) if relu else y64
    for mode, (y, mean, rstd, dx, dg, db) in outs.items():
        name = f"GN C={C} G={G} HW={HW} B={B} relu={relu} [{mode}]"
        y4 = em.view4(y, G)
        em.assert_rel(name + " y", y4, yr64, mag, em.C_FWD)
        em.check_stats(name, mean, rstd, mu, rstd64, m)
        for b, gi in const:                                            # a constant group: y = beta (relu(beta)) exactly
            want = beta[gi * cpg:(gi + 1) * cpg]
            want = want.clamp_min(0.0) if relu else want
            assert torch.equal(y4[b, :, gi], want.expand(HW, cpg)), f"{name}: constant group ({b}, {gi}) is not beta"
        if relu:                                                       # a clearly negative pre-activation gives +0 exactly
            neg = y64 < -em.C_FWD * mag
            assert bool(neg.any()) or HW * B < 4
            assert bool((y4[neg] == 0).all()), name
        d4 = em.view4(dy * (y > 0) if relu else dy, G)
        dx64, mag_dx, dxh, mag_dg, mag_db = em.backward(d4, g4, rstd64, m, xh)
        em.assert_rel(name + " dx", em.view4(dx, G), dx64, mag_dx, em.C_BWD)
        em.assert_rel(name + " dgamma", dg, em.param_sum(dxh), em.param_sum(mag_dg), em.C_PAR)
        em.assert_rel(name + " dbeta", db, em.param_sum(d4.to(F64)), em.param_sum(mag_db), em.C_PAR)


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("C,G", [(96, 8), (64, 32), (256, 128)])
def test_groupnorm_unsupported_shapes_raise(det, C, G):
    """C = 96: C/4 does not divide the 256 threads; C/G = 2: a group is not a whole number of float4 quads."""
    prev = monodetr_b200.set_deterministic(det)
    try:
        x = torch.randn(2, 5, C, device="cuda")
        gamma, beta = torch.ones(C, device="cuda"), torch.zeros(C, device="cuda")
        with pytest.raises(RuntimeError, match="mdb_groupnorm_forward_f32"):
            K.groupnorm_forward(x, gamma, beta, G)
        mean, rstd = torch.zeros(2, G, device="cuda"), torch.ones(2, G, device="cuda")
        with pytest.raises(RuntimeError, match="mdb_groupnorm_backward_f32"):
            K.groupnorm_backward(x, x, x, gamma, mean, rstd, G)
    finally:
        monodetr_b200.set_deterministic(prev)
