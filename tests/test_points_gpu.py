"""The deformable-attention kernels at 2 and 8 sampling points per level (csrc/msda.cu: msda_fwd_vec_pts_kernel,
msda_fwd_d32_pts_kernel, msda_bwd_vec_pts_kernel), the pre-processing kernels at every count from 1 to 8, and the model at the
point counts of tests/golden/points.npz, against float64 per element (tests/msda_error_model.py) and the reference."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import msda_error_model as em
import test_msda_error_model_gpu as base     # the float64 checks of the 4-point kernels, reused at other counts
from oracle import monodetr_torch as om
import oracle_points as op

pytestmark = pytest.mark.gpu

F64 = torch.float64

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gen_golden_points import VARIANTS  # noqa: E402
from gen_golden_reference_pins import sampled_forward  # noqa: E402

OUT_KEYS = ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")

# (label, levels, B, Lq, M, D, P, kind, misaligned, reproducible)
CASES = [(f"P={P} {lbl}", lv, B, Lq, M, D, P, kind, mis, repro)
         for P in (2, 8)
         for lbl, lv, B, Lq, M, D, kind, mis, repro in [
             ("d32", 4, 2, 37, 8, 32, "plain", False, False),
             ("d32 signed edge levels", "edge4", 2, 33, 8, 32, "signed", False, False),
             ("d32 collide", 4, 1, 2000, 8, 32, "collide", False, False),
             ("d32 tail multi-pass", 4, 1, 10001, 5, 32, "plain", False, False),
             ("vec D=64", 4, 2, 31, 4, 64, "plain", False, False),
             ("vec D=64 edge levels", "edge4", 1, 40, 4, 64, "offset", False, False),
             ("vec D=64 tail", 4, 1, 6001, 3, 64, "plain", False, False),
             ("vec D=16", 4, 2, 31, 16, 16, "signed", False, False),
             ("vec D=16 edge levels tail", "edge4", 1, 7, 3, 16, "offset", False, False),
             ("vec D=16 collide", 4, 1, 1000, 16, 16, "collide", False, False),
             ("vec L=3", 3, 2, 23, 3, 32, "plain", False, False),
             ("vec L=8", 8, 1, 23, 5, 32, "plain", False, False),
             ("generic misaligned D=32", 4, 2, 37, 8, 32, "plain", True, False),
             ("generic misaligned D=16", "edge4", 1, 37, 16, 16, "signed", True, False),
             ("ordered D=32", 4, 1, 37, 8, 32, "plain", False, True),
         ]]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_paths_at_the_edges(case):
    label, lv, B, Lq, M, D, P, kind, mis, repro = case
    shapes = base.EDGE4 if lv == "edge4" else base.LEVELS[lv]
    ins, landed = em.make_inputs(shapes, B, Lq, M, D, P, seed=len(label) * 97 + Lq + P, kind=kind)
    if kind != "collide":
        base._assert_landed(landed, shapes)
    base._check_op(label, ins, mis, repro)


@pytest.mark.parametrize("P", [2, 8])
@pytest.mark.parametrize("M,D", [(8, 32), (4, 64), (16, 16)])
def test_encoder_shapes(P, M, D):
    ins, _ = em.make_inputs(base.MODEL, 2, 10200, M, D, P, seed=M * D + P, kind="plain")
    base._check_op(f"encoder P={P} M={M} D={D}", ins)


@pytest.mark.parametrize("P", [2, 8])
@pytest.mark.parametrize("lv,M,D", [(4, 8, 32), (4, 4, 64), (4, 16, 16), (8, 8, 32)])
@pytest.mark.parametrize("reproducible", [False, True])
def test_nonfinite_locations_give_exact_zeros(P, lv, M, D, reproducible):
    ins, _ = em.make_inputs(base.LEVELS[lv], 2, 41, M, D, P, seed=D + lv + P, kind="nonfinite")
    assert bool((~torch.isfinite(ins[3])).any())
    base._check_op(f"nonfinite P={P} L={lv} D={D}" + (" [reproducible]" if reproducible else ""), ins, reproducible=reproducible)


@pytest.mark.parametrize("P", [1, 3, 5, 6, 7, 8])
@pytest.mark.parametrize("rd", [2, 6])
@pytest.mark.parametrize("kind", ["plain", "spread"])
def test_preprocessing(P, rd, kind):
    base.test_preprocessing(4, P, rd, kind)


def test_preprocessing_refuses_more_than_32_pairs():
    value, shapes, lsi, off, logits, ref, _ = base._module_inputs(1, 5, 2, 4, 8, 2, "plain", seed=0)
    loc, attn = base._nan((1, 5, 2, 4, 9, 2)), base._nan((1, 5, 2, 4, 9))
    with pytest.raises(RuntimeError):
        base._lib.call("mdb_msda_prep_forward_f32", off, logits, ref, shapes, 1, 5, 2, 4, 9, 2, loc, attn)


def _check_fused(P, case):
    """mdb_msda_fused_forward_f32 / _backward_f32 (and _backward_ref_f32 with 6-d boxes) at P points against the float64 op on the
    pre-processing kernel's fp32 locations and the float64 softmax of the logits -- tests/test_msda_error_model_gpu.py's
    4-point check at P points.  A box partial sums a level's P per-point terms: its bound grows like gamma_(P-1), so the
    constant calibrated at P = 4 is scaled by (P - 1) / 3."""
    B, Lq, M, rd, kind = case
    L, D = 4, 32
    value, shapes, lsi, off, logits, ref, dout = base._module_inputs(B, Lq, M, L, P, rd, kind, seed=B * Lq + M + rd + P)
    if kind == "nonfinite":
        g = torch.Generator(device="cuda").manual_seed(1)
        special = torch.tensor([1e30, -1e30, float("inf"), float("-inf"), float("nan")], device="cuda")
        pick = torch.rand(off.shape, device="cuda", generator=g) < 0.15
        off = torch.where(pick, special[torch.randint(0, 5, off.shape, device="cuda", generator=g)], off)
    S = value.shape[1]
    nan = base._nan
    loc, _ = base._prep(off, logits, ref, shapes, B, Lq, M, L, P, rd)
    out = nan((B, Lq, M * D))
    base._lib.call("mdb_msda_fused_forward_f32", value, shapes, lsi, off, logits, ref, B, S, M, D, L, Lq, P, rd, out)
    gv, goff, glog = nan(value.shape), nan(off.shape), nan(logits.shape)
    base._lib.call("mdb_msda_fused_backward_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, D, L, Lq, P, rd, gv, goff,
                   glog)
    part = None
    if rd == 6 and kind != "nonfinite":                           # an infinite offset has no box gradient
        gv2, goff2, glog2, part = nan(value.shape), nan(off.shape), nan(logits.shape), nan((B, Lq, M, L, 4))
        base._lib.call("mdb_msda_fused_backward_ref_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, D, L, Lq, P, rd,
                       gv2, goff2, glog2, part)
    torch.cuda.synchronize()
    name = "fused P={} B={} Lq={} M={} rd={} {}".format(P, *case)
    a64, am = em.softmax64(logits, M, L, P), em.softmax_mag(logits, M, L, P)
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
        em.assert_rel(name + " box partials", part, p64, em.U32 * pmag + em.ETA * cnt.sum(4), em.C_PART * max(P - 1, 3) / 3)


@pytest.mark.parametrize("P", [2, 8])
@pytest.mark.parametrize("case", base.FUSED, ids=lambda c: "B{}-Lq{}-M{}-rd{}-{}".format(*c))
def test_fused(P, case):
    _check_fused(P, case)


def test_every_new_instance_runs():
    """Each P = 2 / 8 instance appears under torch.profiler."""
    import re
    from torch.profiler import ProfilerActivity, profile
    want = [f"{k}<{a}>" for P in (2, 8) for k, a in
            [("msda_fwd_vec_pts_kernel", f"4,{P}"), ("msda_fwd_vec_pts_kernel", f"8,{P}"), ("msda_fwd_vec_pts_kernel", f"16,{P}"),
             ("msda_fwd_d32_pts_kernel", f"true,{P}"),
             ("msda_bwd_vec_pts_kernel", f"4,4,{P},false,false"), ("msda_bwd_vec_pts_kernel", f"8,4,{P},false,false"),
             ("msda_bwd_vec_pts_kernel", f"16,4,{P},false,false"), ("msda_bwd_vec_pts_kernel", f"8,4,{P},true,false"),
             ("msda_bwd_vec_pts_kernel", f"8,4,{P},true,true")]] + ["msda_prep_fwd_any_kernel", "msda_prep_bwd_any_kernel"]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for P in (2, 8):
            for lv, M, D in ((4, 8, 32), (2, 8, 32), (4, 4, 64), (4, 16, 16)):
                base._run(em.make_inputs(base.LEVELS[lv], 1, 9, M, D, P, seed=1)[0])
            B, Lq, M, L, rd = 1, 9, 8, 4, 6
            value, shapes, lsi, off, logits, ref, dout = base._module_inputs(B, Lq, M, L, P, rd, "plain", seed=3)
            S = value.shape[1]
            d = base._nan(off.shape), base._nan(logits.shape)
            loc, attn = base._prep(off, logits, ref, shapes, B, Lq, M, L, P, rd)
            base._lib.call("mdb_msda_prep_backward_f32", loc, attn, attn, ref, shapes, B, Lq, M, L, P, rd, *d)
            base._lib.call("mdb_msda_fused_forward_f32", value, shapes, lsi, off, logits, ref, B, S, M, 32, L, Lq, P, rd,
                           base._nan(dout.shape))
            base._lib.call("mdb_msda_fused_backward_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, 32, L, Lq, P, rd,
                           base._nan(value.shape), *d)
            base._lib.call("mdb_msda_fused_backward_ref_f32", value, shapes, lsi, off, logits, ref, dout, B, S, M, 32, L, Lq, P,
                           rd, base._nan(value.shape), *d, base._nan((B, Lq, M, L, 4)))
        torch.cuda.synchronize()
    names = {re.sub(r"\s+", "", e.name) for e in prof.events()}
    missing = [k for k in want if not any(k in n for n in names)]
    assert not missing, f"kernels that did not run: {missing}; seen: {sorted(n for n in names if 'msda' in n)}"


# ---- the model --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "points.npz"))


def _model(points, load=True, **kw):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    torch.manual_seed(0)
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, enc_n_points=points[0], dec_n_points=points[1], dropout=0.0, **kw))
    if load:
        m.load_state_dict(om.with_aliases(op.deterministic_state_dict(op.points_cfg(*points))))
    for mod in m.modules():              # the depth encoder hard-codes dropout 0.1 (depth_predictor.py:49-50)
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return m.cuda()


@pytest.mark.parametrize("tag", list(VARIANTS))
def test_model_matches_the_reference(tag, golden):
    """Eval outputs at 192 x 640 and train outputs at 96 x 320 against the unmodified reference; finite gradients."""
    points = VARIANTS[tag]
    m = _model(points).eval()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=192, W=640)
    with torch.no_grad():
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{tag}.fwd_eval_{k}", out[k].float().cpu().numpy()), rtol=2e-2,
                                   atol=2e-3, err_msg=k)
    m.train()
    images, calibs, sizes = om.synthetic_inputs(1, 0, H=96, W=320)
    out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
    for k in OUT_KEYS:
        np.testing.assert_allclose(*sampled_forward(golden, f"{tag}.fwd_train_{k}", out[k].detach().float().cpu().numpy()),
                                   rtol=2e-2, atol=2e-3, err_msg=k)
    om.surrogate_loss(out).backward()
    assert all(torch.isfinite(p.grad).all() for p in m.parameters() if p.grad is not None)


STAGES = ("backbone", "input_proj", "depth_predictor", "depthaware_transformer.encoder", "depthaware_transformer.decoder.layers",
          "depthaware_transformer.decoder", "depthaware_transformer", "query_embed", "tgt_embed", "refpoint_embed", "class_embed",
          "bbox_embed", "dim_embed_3d", "angle_embed", "depth_embed")


def _dab_oracle(points):
    """tests/oracle_dab.py's use_dab model with the point counts of tests/oracle_points.py: (cfg, weights, forward)."""
    import oracle_dab as od
    cfg = dict(op.points_cfg(*points), use_dab=True)
    saved = om.state_dict_spec
    om.state_dict_spec = lambda c=cfg: od.state_dict_spec(c, base_spec=op.state_dict_spec(c))
    try:
        sd = om.deterministic_state_dict(cfg)
    finally:
        om.state_dict_spec = saved
    for name in sd:
        if name.endswith("sampling_offsets.bias"):
            sd[name] = op.sampling_offsets_bias(op.n_points_of(cfg, name)).to(sd[name].dtype)

    def forward(sd, images, calibs, sizes, training):
        with op._variant(cfg):
            return od.forward(sd, images, calibs, sizes, training=training, cfg=cfg)
    return cfg, sd, forward


@pytest.mark.parametrize("points,dab", [((2, 2), False), ((8, 8), False), ((3, 6), False), ((4, 8), True), ((8, 2), True)])
def test_gradients_per_stage(points, dab):
    """Frozen sampling locations, 192 x 640, B = 2: every gradient against the CPU oracle, with the bars of
    tests/test_model_grad_gpu.py (median < 1e-3; every tensor < 2e-2, query_embed < 5e-2; max-norm and L2).  use_dab: the first
    decoder layer's shared boxes take the box-partial (REFGRAD) kernel, so the anchors' gradient checks its reduction."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    if dab:
        cfg, sd0, oracle_forward = _dab_oracle(points)
    else:
        cfg, sd0 = op.points_cfg(*points), op.deterministic_state_dict(op.points_cfg(*points))
        oracle_forward = lambda sd, *a, training: op.forward(sd, *a, training=training, cfg=cfg)      # noqa: E731
    m = _model(points, load=False, use_dab=dab)
    m.load_state_dict(om.with_aliases(sd0))
    m.train()
    images, calibs, sizes = om.synthetic_inputs(2, 11, H=192, W=640)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in sd0.items()}
        om.surrogate_loss(oracle_forward(sd, images, calibs, sizes, training=True)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    params = dict(m.named_parameters())
    for name, p in params.items():        # analytically zero (see tests/test_backbone_variants_gpu.py)
        if name.endswith(("sa_kcontent_proj.bias", "sa_kpos_proj.bias")) and p.grad is not None:
            wmax = float(params[name[:-len("bias")] + "weight"].grad.abs().max())
            assert float(p.grad.abs().max()) <= 5e-3 * wmax and float(sd[name].grad.abs().max()) <= 1e-4 * wmax, name
            p.grad = None
    by_name = om.with_aliases(sd)
    per_stage, rel_max, rel_l2 = {}, [], []
    for name, p in m.named_parameters():
        if not p.requires_grad or p.grad is None:
            continue
        gref = by_name[name].grad
        assert gref is not None, name
        scale = float(gref.abs().max())
        if scale < 1e-7:
            continue
        d = p.grad.cpu() - gref
        r, l2 = float(d.abs().max()) / scale, float(d.norm() / gref.norm())
        rel_max.append(r)
        rel_l2.append(l2)
        # use_dab's query-scale MLP scales the query position of every decoder layer: query_embed's role, and its bar
        stage = "query_embed" if name.startswith("depthaware_transformer.decoder.query_scale.") else \
            next(s for s in STAGES if name.startswith(s))
        cur = per_stage.get(stage, (0.0, 0.0, ""))
        per_stage[stage] = (max(cur[0], r), max(cur[1], l2), name if r > cur[0] else cur[2])
    print(points, dab, {k: f"{v[0]:.1e} {v[1]:.1e}" for k, v in per_stage.items()},
          "median", f"{float(np.median(rel_max)):.2e} {float(np.median(rel_l2)):.2e}", "tensors", len(rel_max))
    assert len(rel_max) > 240
    if dab:
        assert "refpoint_embed" in per_stage
    assert float(np.median(rel_max)) < 1e-3 and float(np.median(rel_l2)) < 1e-3
    for stage, (r, l2, name) in per_stage.items():
        assert r < (5e-2 if stage == "query_embed" else 2e-2) and l2 < 2e-2, (stage, name, r, l2)


def _setup(dev, points, B=2):
    from bench_extras import CRIT_CFG, synthetic_targets
    from monodetr_b200 import build_monodetr
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, enc_n_points=points[0], dec_n_points=points[1], dropout=0.1))
    model = model.to(dev).train()
    crit = build_criterion(CRIT_CFG).to(dev).train()
    bucket = FlatGradBucket(model)
    opt = FusedAdamW(model, bucket, lr=2e-4, weight_decay=1e-4, device_step=True)
    images, calibs, sizes = (t.to(dev) for t in synthetic_batch(B, seed=77))
    tg = {k: v.to(dev) for k, v in synthetic_targets(77, B).items()}
    state = {}

    def it():
        bucket.zero()
        out = model(images, calibs, None, sizes)
        losses = crit(out, tg)
        crit.weighted_sum().backward()
        opt.step()
        state["out"], state["losses"] = out, losses

    def snapshot():
        out = state["out"]
        flat = [out[k] for k in OUT_KEYS] + [v for a in out["aux_outputs"] for _, v in sorted(a.items())]
        losses = [state["losses"][k] for k in sorted(state["losses"])]
        grads = [p.grad for p in model.parameters() if p.grad is not None]
        return [t.detach().clone() for t in flat], [t.detach().clone() for t in losses], [t.clone() for t in grads], \
            [p.detach().clone() for p in model.parameters()]
    return bucket, it, snapshot


def _assert_equal(a, b):
    for name, xs, ys in zip(("outputs", "losses", "gradients", "parameters"), a, b):
        assert len(xs) == len(ys), name
        assert all(bool(torch.isfinite(x).all()) for x in xs), name
        bad = [i for i, (x, y) in enumerate(zip(xs, ys)) if not torch.equal(x, y)]
        assert not bad, (name, len(bad), len(xs))


def test_training_iterations_are_bit_reproducible_eager_and_as_a_cuda_graph():
    """Reproducible mode at 8 / 8 points: two training iterations (forward with dropout, the device criterion, backward,
    FusedAdamW) give identical bits twice eagerly, and a replayed CUDA graph of the iteration gives the eager bits."""
    import monodetr_b200
    from monodetr_b200 import kernels as K, tc
    dev = torch.device("cuda", torch.cuda.current_device())
    prev, prev_prec = monodetr_b200.set_deterministic(True), tc.get_precision()
    tc.set_precision("bf16x3")
    try:
        runs = []
        for _ in range(2):
            _, it, snap = _setup(dev, (8, 8))
            K.reseed(dev, 4242)
            for _ in range(2):
                it()
            runs.append(snap())
        assert len(runs[0][2]) == 313
        _assert_equal(runs[0], runs[1])

        _, it_a, snap_a = _setup(dev, (8, 8))
        bucket_b, it_b, snap_b = _setup(dev, (8, 8))
        K.reseed(dev, 99)
        for _ in range(3):
            it_a()
        eager = snap_a()
        K.reseed(dev, 99)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(2):
                it_b()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            it_b()
        bucket_b.freeze_sources()
        graph.replay()
        torch.cuda.synchronize()
        _assert_equal(eager, snap_b())
    finally:
        tc.set_precision(prev_prec)
        monodetr_b200.set_deterministic(prev)
