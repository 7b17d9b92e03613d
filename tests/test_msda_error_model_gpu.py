"""The deformable-attention kernels (csrc/msda.cu) against float64 per element (tests/msda_error_model.py), on every dispatch
path: msda_fwd_d32_kernel, msda_fwd_vec_kernel<4|8|16>, msda_bwd_vec_kernel<4|8|16, 4>, the generic fp32 kernels (any L, P, D,
misaligned pointers), the reproducible value gradient, the fused module kernels with 2-d references and 6-d boxes (and the
box partials) and the pre-processing kernels.  The paths meet the edges where sampling kernels go wrong: points exactly on
the lines the image and corner tests compare against, 1x1 / 1xW / Hx1 / 2x2 levels, ragged unit tails and CTAs that walk
several passes, the model's shapes, non-finite and far locations, thousands of contributions to one value row, signed
unnormalised weights, values with a large common offset and softmax logits over +-100.

The C entry points are called directly, every output pre-filled with NaN (the backward zeroes grad_value itself), so an
element a kernel does not write fails isfinite."""
import re

import pytest
import torch

import monodetr_b200
import msda_error_model as em
from monodetr_b200 import _lib

pytestmark = pytest.mark.gpu

F64 = torch.float64
MODEL = [(48, 160), (24, 80), (12, 40), (6, 20)]
EDGE4 = [(1, 1), (1, 9), (7, 1), (2, 2)]                      # 1x1, 1xW, Hx1, 2x2
LEVELS = {1: [(16, 32)], 2: [(1, 9), (7, 1)], 3: [(2, 2), (1, 1), (12, 40)], 4: MODEL, 5: MODEL + [(1, 1)],
          8: MODEL + EDGE4, 9: MODEL + EDGE4 + [(16, 32)]}


def _nan(shape, misaligned=False):
    """A NaN-filled fp32 tensor; misaligned: stored one float past a 16-byte boundary."""
    n = 1
    for s in shape:
        n *= s
    buf = torch.full((n + int(misaligned),), float("nan"), device="cuda")
    return buf[int(misaligned):].view(shape)


def _dev(ins, misaligned=False):
    out = []
    for t in ins:
        if t.is_floating_point():
            d = _nan(t.shape, misaligned)
            d.copy_(t)
            out.append(d)
        else:
            out.append(t.cuda())
    return out


def _run(ins, misaligned=False, reproducible=False):
    """mdb_msda_forward_f32 and mdb_msda_backward_f32 into NaN-filled outputs -> dict of outputs."""
    value, shapes, lsi, loc, attn, grad_out = _dev(ins, misaligned)
    B, S, M, D = value.shape
    _, Lq, _, L, P, _ = loc.shape
    out = _nan((B, Lq, M * D), misaligned)
    _lib.call("mdb_msda_forward_f32", value, shapes, lsi, loc, attn, B, S, M, D, L, Lq, P, out)
    gv, gl, ga = _nan(value.shape, misaligned), _nan(loc.shape, misaligned), _nan(attn.shape, misaligned)
    prev = monodetr_b200.set_deterministic(reproducible)
    try:
        _lib.call("mdb_msda_backward_f32", value, shapes, lsi, loc, attn, grad_out, B, S, M, D, L, Lq, P, gv, gl, ga,
                  launches=2 if reproducible else 1)
    finally:
        monodetr_b200.set_deterministic(prev)
    torch.cuda.synchronize()
    return {"out": out, "grad_value": gv, "grad_loc": gl, "grad_attn": ga}


def _check_op(name, ins, misaligned=False, reproducible=False):
    got = _run(ins, misaligned, reproducible)
    r = em.reference(*(t.cuda() for t in ins))
    return em.check(name, got, r)


def _assert_landed(landed, shapes):
    """Every edge target of em.edge_targets was hit exactly on some level.  A coordinate of exactly 0 needs loc = 1 / (2 W)
    in fp32, so a side that is a power of two; without one, the points nearest 0 on either side stand in for it."""
    for ax, side in (("x", 1), ("y", 0)):
        hit = landed[ax] > 0
        if not any(s[side] & (s[side] - 1) == 0 for s in shapes):
            hit[3] = True
        assert bool(hit.all()), (ax, landed)


# (label, levels, B, Lq, M, D, P, kind, misaligned, reproducible)
CASES = [
    # msda_fwd_d32_kernel + msda_bwd_vec_kernel<8, 4>
    ("d32", 4, 2, 37, 8, 32, 4, "plain", False, False),
    ("d32 signed", 4, 1, 29, 8, 32, 4, "signed", False, False),
    ("d32 offset", 4, 1, 29, 8, 32, 4, "offset", False, False),
    ("d32 collide", 4, 1, 2000, 8, 32, 4, "collide", False, False),
    ("d32 edge levels", "edge4", 2, 33, 8, 32, 4, "plain", False, False),
    ("d32 tail Lq=1", 4, 1, 1, 5, 32, 4, "plain", False, False),
    ("d32 tail multi-pass", 4, 1, 10001, 5, 32, 4, "plain", False, False),
    # msda_fwd_vec_kernel<16> / <4> + msda_bwd_vec_kernel<16, 4> / <4, 4>
    ("vec D=64", 4, 2, 31, 4, 64, 4, "plain", False, False),
    ("vec D=64 edge levels", "edge4", 1, 40, 4, 64, 4, "signed", False, False),
    ("vec D=64 tail", 4, 1, 5, 3, 64, 4, "offset", False, False),
    ("vec D=64 tail multi-pass", 4, 1, 6001, 3, 64, 4, "plain", False, False),
    ("vec D=16", 4, 2, 31, 16, 16, 4, "plain", False, False),
    ("vec D=16 edge levels", "edge4", 1, 40, 16, 16, 4, "offset", False, False),
    ("vec D=16 tail", 4, 1, 7, 3, 16, 4, "signed", False, False),
    ("vec D=16 tail multi-pass", 4, 1, 10001, 7, 16, 4, "plain", False, False),
    ("vec D=16 collide", 4, 1, 1000, 16, 16, 4, "collide", False, False),
    # msda_fwd_vec_kernel<8> at L != 4 + generic backward
    ("vec L=1", 1, 2, 23, 8, 32, 4, "plain", False, False),
    ("vec L=2", 2, 2, 23, 8, 32, 4, "signed", False, False),
    ("vec L=3", 3, 2, 23, 3, 32, 4, "plain", False, False),
    ("vec L=5", 5, 1, 23, 8, 32, 4, "offset", False, False),
    ("vec L=8", 8, 1, 23, 5, 32, 4, "plain", False, False),
    # generic fp32 kernels
    ("generic L=9", 9, 1, 23, 3, 32, 4, "plain", False, False),
    ("generic P=1", 4, 2, 19, 3, 32, 1, "plain", False, False),
    ("generic P=2", "edge4", 2, 19, 3, 32, 2, "signed", False, False),
    ("generic P=3", 4, 1, 19, 8, 32, 3, "offset", False, False),
    ("generic P=8", 4, 1, 19, 3, 32, 8, "plain", False, False),
    ("generic D=1", 4, 2, 19, 3, 1, 4, "plain", False, False),
    ("generic D=8", "edge4", 1, 19, 3, 8, 4, "signed", False, False),
    ("generic D=31", 4, 1, 19, 3, 31, 4, "plain", False, False),
    ("generic D=33", 4, 1, 19, 2, 33, 4, "offset", False, False),
    ("generic D=65", 4, 1, 19, 2, 65, 4, "plain", False, False),
    ("generic D=1025", "edge4", 1, 5, 1, 1025, 4, "plain", False, False),
    ("generic D=33 collide", 4, 1, 500, 2, 33, 4, "collide", False, False),
    ("generic misaligned D=32", 4, 2, 37, 8, 32, 4, "plain", True, False),
    ("generic misaligned D=64", 4, 1, 37, 4, 64, 4, "signed", True, False),
    ("generic misaligned D=16", "edge4", 1, 37, 16, 16, 4, "plain", True, False),
    # reproducible mode: generic backward without the scatter + msda_bwd_value_ordered_kernel
    ("ordered D=32", 4, 2, 37, 8, 32, 4, "plain", False, True),
    ("ordered D=32 collide", 4, 1, 2000, 8, 32, 4, "collide", False, True),
    ("ordered D=33 P=3", "edge4", 1, 23, 3, 33, 3, "signed", False, True),
    ("ordered D=16 offset", 4, 1, 23, 16, 16, 4, "offset", False, True),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_paths_at_the_edges(case):
    label, lv, B, Lq, M, D, P, kind, mis, repro = case
    shapes = EDGE4 if lv == "edge4" else LEVELS[lv]
    ins, landed = em.make_inputs(shapes, B, Lq, M, D, P, seed=len(label) * 97 + Lq, kind=kind)
    if kind != "collide":
        _assert_landed(landed, shapes)
    _check_op(label, ins, mis, repro)


@pytest.mark.parametrize("M,D", [(8, 32), (4, 64), (16, 16)])
def test_encoder_shapes(M, D):
    """The encoder's call at B = 2, Lq = 10200 (every pixel of the four levels queries), for each head width."""
    ins, _ = em.make_inputs(MODEL, 2, 10200, M, D, 4, seed=M * D, kind="plain")
    _check_op(f"encoder M={M} D={D}", ins)


@pytest.mark.parametrize("case", [("d32", 4, 8, 32), ("vec<16>", 4, 4, 64), ("vec<4>", 4, 16, 16), ("vec<8> L=8", 8, 8, 32),
                                  ("generic", 9, 3, 33)], ids=lambda c: c[0])
@pytest.mark.parametrize("reproducible", [False, True])
def test_nonfinite_locations_give_exact_zeros(case, reproducible):
    """Locations of +-1e30, +-inf and NaN lie off the image: they add exactly 0 to out and grad_value and give exactly 0 in
    grad_loc and grad_attn.  (msda_fwd_vec_kernel and msda_bwd_vec_kernel once multiplied the zero corners of such a point by
    the weights of x - floor(x) = NaN.)"""
    label, lv, M, D = case
    ins, _ = em.make_inputs(LEVELS[lv], 2, 41, M, D, 4, seed=D + lv, kind="nonfinite")
    loc = ins[3]
    assert bool((~torch.isfinite(loc)).any()) and bool((loc.abs() == 1e30).any())
    _check_op(f"nonfinite {label}" + (" [reproducible]" if reproducible else ""), ins, reproducible=reproducible)


# ---- the module's fused kernels and the pre-processing ---------------------------------------------------------------------------
def _module_inputs(B, Lq, M, L, P, rd, kind, seed):
    g = torch.Generator().manual_seed(seed)
    shapes = torch.as_tensor(MODEL[:L], dtype=torch.long)
    lsi = torch.cat((shapes.new_zeros((1,)), shapes.prod(1).cumsum(0)[:-1]))
    S = int(shapes.prod(1).sum())
    value = torch.randn(B, S, M, 32, generator=g)
    off = torch.randn(B, Lq, M * L * P * 2, generator=g) * 3
    if kind == "spread":                                          # past the point where expf overflows without the max
        logits = torch.rand(B, Lq, M * L * P, generator=g) * 200 - 100
    else:
        logits = torch.randn(B, Lq, M * L * P, generator=g) * 2
    ref = torch.rand(B, Lq, L, rd, generator=g)
    if rd == 6:                                                   # boxes partly off the image
        ref[..., :2] = ref[..., :2] * 1.4 - 0.2
        ref[..., 2:] *= 0.3
    dout = torch.randn(B, Lq, M * 32, generator=g)
    return [t.cuda() for t in (value, shapes, lsi, off, logits, ref, dout)]


def _prep(off, logits, ref, shapes, B, Lq, M, L, P, rd):
    loc, attn = _nan((B, Lq, M, L, P, 2)), _nan((B, Lq, M, L, P))
    _lib.call("mdb_msda_prep_forward_f32", off, logits, ref, shapes, B, Lq, M, L, P, rd, loc, attn)
    return loc, attn


@pytest.mark.parametrize("L,P", [(4, 4), (2, 2), (4, 2), (1, 4)])
@pytest.mark.parametrize("rd", [2, 6])
@pytest.mark.parametrize("kind", ["plain", "spread"])
def test_preprocessing(L, P, rd, kind):
    """mdb_msda_prep_forward_f32 / _backward_f32: loc = ref + off * s and the softmax, and their gradients, in float64."""
    B, Lq, M = 2, 301, 3
    value, shapes, lsi, off, logits, ref, _ = _module_inputs(B, Lq, M, L, P, rd, kind, seed=L * 10 + P + rd)
    loc, attn = _prep(off, logits, ref, shapes, B, Lq, M, L, P, rd)
    g = torch.Generator(device="cuda").manual_seed(L + P + rd)
    dloc, dattn = torch.randn(loc.shape, device="cuda", generator=g), torch.randn(attn.shape, device="cuda", generator=g)
    doff, dlogits = _nan(off.shape), _nan(logits.shape)
    _lib.call("mdb_msda_prep_backward_f32", dloc, dattn, attn, ref, shapes, B, Lq, M, L, P, rd, doff, dlogits)
    torch.cuda.synchronize()
    name = f"prep L={L} P={P} rd={rd} {kind}"
    loc64, mag = em.prep_loc(off, ref, shapes, M, L, P)
    em.assert_rel(name + " loc", loc, loc64, em.U32 * mag, em.C_PREP)
    a64 = em.softmax64(logits, M, L, P)
    em.assert_rel(name + " attn", attn, a64, em.U32 * em.softmax_mag(logits, M, L, P) + em.ETA, em.C_PREP)
    s = em.offset_scale(ref, shapes, M, L, P)
    d64 = dloc.to(F64) * s
    em.assert_rel(name + " grad_offsets", doff.view(d64.shape), d64, em.U32 * d64.abs(), em.C_PREP)
    a = attn.to(F64).view(B, Lq, M, L * P)
    ga = dattn.to(F64).view(B, Lq, M, L * P)
    dl64, mag_dl = em.softmax_grad(a, a, ga, ga.abs())
    em.assert_rel(name + " grad_logits", dlogits.view(dl64.shape), dl64, em.U32 * mag_dl + em.ETA * (L * P + 1), em.C_PREP)


FUSED = [  # (B, Lq, M, rd, kind)
    (2, 550, 8, 6, "plain"),          # the decoder's call: 6-d boxes partly off the image
    (2, 550, 8, 2, "plain"),
    (2, 37, 1, 2, "plain"), (1, 41, 3, 6, "plain"), (3, 29, 5, 2, "spread"), (1, 1, 5, 6, "plain"),   # tails: M = 1, 3, 5
    (2, 300, 8, 2, "spread"), (1, 77, 3, 6, "spread"),
    (1, 10001, 5, 2, "plain"),        # several passes per CTA with a ragged tail
    (2, 53, 3, 2, "nonfinite"),
]


@pytest.mark.parametrize("case", FUSED, ids=lambda c: "B{}-Lq{}-M{}-rd{}-{}".format(*c))
def test_fused(case):
    """mdb_msda_fused_forward_f32 / _backward_f32 (and _backward_ref_f32 with 6-d boxes) against the float64 op on the
    pre-processing kernel's fp32 locations (the expression the fused kernels evaluate) and the float64 softmax of the logits."""
    B, Lq, M, rd, kind = case
    L, P, D = 4, 4, 32
    value, shapes, lsi, off, logits, ref, dout = _module_inputs(B, Lq, M, L, P, rd, kind, seed=B * Lq + M + rd)
    if kind == "nonfinite":
        g = torch.Generator(device="cuda").manual_seed(1)
        special = torch.tensor([1e30, -1e30, float("inf"), float("-inf"), float("nan")], device="cuda")
        pick = torch.rand(off.shape, device="cuda", generator=g) < 0.15
        off = torch.where(pick, special[torch.randint(0, 5, off.shape, device="cuda", generator=g)], off)
    S = value.shape[1]
    loc, _ = _prep(off, logits, ref, shapes, B, Lq, M, L, P, rd)
    out = _nan((B, Lq, M * D))
    _lib.call("mdb_msda_fused_forward_f32", value, shapes, lsi, off, logits, ref, B, S, M, D, L, Lq, P, rd, out)
    gv, goff, glog = _nan(value.shape), _nan(off.shape), _nan(logits.shape)
    _lib.call("mdb_msda_fused_backward_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, D, L, Lq, P, rd, gv, goff, glog)
    part = None
    if rd == 6 and kind != "nonfinite":                           # an infinite offset has no box gradient
        gv2, goff2, glog2, part = _nan(value.shape), _nan(off.shape), _nan(logits.shape), _nan((B, Lq, M, L, 4))
        _lib.call("mdb_msda_fused_backward_ref_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, D, L, Lq, P, rd,
                  gv2, goff2, glog2, part)
    torch.cuda.synchronize()
    name = "fused B={} Lq={} M={} rd={} {}".format(*case)
    a64 = em.softmax64(logits, M, L, P)
    am = em.softmax_mag(logits, M, L, P)
    r = em.reference(value, shapes, lsi, loc, a64, dout, attn_mag=am)
    em.check(name, {"out": out, "grad_value": gv}, r)
    s = em.offset_scale(ref, shapes, M, L, P)
    cnt = r["cnt_pt"].unsqueeze(-1)
    go64, mag_go = r["grad_loc"] * s, em.U32 * r["mag_gl"] * s.abs() + em.ETA * (cnt + 1)
    em.assert_rel(name + " grad_offsets", goff.view(go64.shape), go64, mag_go, em.C_FUSED)
    flat = (B, Lq, M, L * P)
    gl64, mag_gl = em.softmax_grad(a64.view(flat), am.view(flat), r["grad_attn"].view(flat), r["mag_ga"].view(flat))
    mag_gl = em.U32 * mag_gl + em.ETA * (r["cnt_pt"].view(flat).sum(-1, keepdim=True) + 1)
    em.assert_rel(name + " grad_logits", glog.view(flat), gl64, mag_gl, em.C_FUSED)
    if part is not None:
        em.check(name + " [ref]", {"grad_value": gv2}, r)
        em.assert_rel(name + " [ref] grad_offsets", goff2.view(go64.shape), go64, mag_go, em.C_FUSED)
        em.assert_rel(name + " [ref] grad_logits", glog2.view(flat), gl64, mag_gl, em.C_FUSED)
        o = off.to(F64).view(B, Lq, M, L, P, 2)
        gl, mg = r["grad_loc"], r["mag_gl"]
        p64 = torch.cat((gl.sum(4), (gl * o).sum(4)), -1)
        pmag = torch.cat((mg.sum(4), (mg * o.abs()).sum(4)), -1)
        em.assert_rel(name + " box partials", part, p64, em.U32 * pmag + em.ETA * cnt.sum(4), em.C_PART)


# ---- every row of the dispatch table runs ------------------------------------------------------------------------------------
KERNELS = ["msda_fwd_d32_kernel<false>", "msda_fwd_d32_kernel<true>", "msda_fwd_vec_kernel<4>", "msda_fwd_vec_kernel<8>",
           "msda_fwd_vec_kernel<16>", "msda_fwd_generic_kernel<float>", "msda_bwd_vec_kernel<4,4,false,false>",
           "msda_bwd_vec_kernel<8,4,false,false>", "msda_bwd_vec_kernel<16,4,false,false>",
           "msda_bwd_generic_kernel<float,true>", "msda_bwd_generic_kernel<float,false>",
           "msda_bwd_value_ordered_kernel<float>", "msda_bwd_vec_kernel<8,4,true,false>", "msda_bwd_vec_kernel<8,4,true,true>",
           "msda_prep_fwd_kernel", "msda_prep_bwd_kernel"]


def test_every_dispatch_path_runs():
    """One representative case per row of the dispatch table under torch.profiler: each kernel above appears, so the cases of
    this file keep reaching the path they are named after if the dispatch changes."""
    from torch.profiler import ProfilerActivity, profile
    reps = [(4, 8, 32, 4, False, False), (4, 4, 64, 4, False, False), (4, 16, 16, 4, False, False), (2, 8, 32, 4, False, False),
            (9, 3, 32, 4, False, False), (4, 8, 32, 4, True, False), (4, 8, 32, 4, False, True)]
    inputs = [em.make_inputs(LEVELS[lv], 1, 9, M, D, P, seed=1)[0] for lv, M, D, P, _, _ in reps]
    B, Lq, M, L, P, rd = 1, 9, 8, 4, 4, 6
    value, shapes, lsi, off, logits, ref, dout = _module_inputs(B, Lq, M, L, P, rd, "plain", seed=3)
    S = value.shape[1]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for ins, (_, _, _, _, mis, repro) in zip(inputs, reps):
            _run(ins, mis, repro)
        loc, attn = _prep(off, logits, ref, shapes, B, Lq, M, L, P, rd)
        d = _nan(off.shape), _nan(logits.shape)
        _lib.call("mdb_msda_prep_backward_f32", loc, attn, attn, ref, shapes, B, Lq, M, L, P, rd, *d)
        _lib.call("mdb_msda_fused_forward_f32", value, shapes, lsi, off, logits, ref, B, S, M, 32, L, Lq, P, rd, _nan(dout.shape))
        _lib.call("mdb_msda_fused_backward_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, 32, L, Lq, P, rd,
                  _nan(value.shape), *d)
        _lib.call("mdb_msda_fused_backward_ref_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, 32, L, Lq, P, rd,
                  _nan(value.shape), *d, _nan((B, Lq, M, L, 4)))
        torch.cuda.synchronize()
    names = {re.sub(r"\s+", "", e.name) for e in prof.events()}
    missing = [k for k in KERNELS if not any(k in n for n in names)]
    assert not missing, f"kernels that did not run: {missing}; seen: {sorted(n for n in names if 'msda' in n)}"
