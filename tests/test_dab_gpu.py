"""GPU: the anchor-box query branch (use_dab) -- its kernels (csrc/dab.cu) against fp64 restatements, the whole model against
the unmodified reference (tests/golden/dab.npz), per-stage gradients against the CPU oracle (tests/oracle_dab.py), and a
bit-reproducible training iteration, eager and as a replayed CUDA graph."""
import json
import math
import os

import numpy as np
import pytest
import torch

import monodetr_b200
from oracle import monodetr_torch as om
import oracle_dab as od          # tests/oracle_dab.py

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a.double().cpu() - b.double().cpu()).abs().max() / b.double().abs().max().clamp_min(1e-30))


def _sine64(box):
    """gen_sineembed_for_position in fp64 (the fp32 constants of the reference: 2pi and dim_t rounded to fp32)."""
    dim_t = torch.arange(128, dtype=torch.float32, device=box.device)
    dim_t = (10000 ** (2 * (dim_t // 2) / 128)).double()
    scale = float(torch.tensor(2 * math.pi, dtype=torch.float32))
    out = []
    for i in (1, 0, 2, 3, 4, 5):
        p = box[..., i, None] * scale / dim_t
        out.append(torch.stack((p[..., 0::2].sin(), p[..., 1::2].cos()), -1).flatten(-2))
    return torch.cat(out, -1)


# ---- kernels -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 550, 4400])
def test_sine_embedding_forward_and_backward(n):
    from monodetr_b200 import functional as Fn
    g = torch.Generator(device="cuda").manual_seed(n)
    box = torch.rand(n, 6, device="cuda", generator=g)
    box[: n // 7] = box[: n // 7] * 1.4 - 0.2                       # a few outside [0, 1] (nothing clamps the embedding)
    box.requires_grad_(True)
    out = Fn.sine_embed(box)
    ref = od.gen_sineembed_for_position(box.detach()[None])[0]
    assert out.shape == (n, 768)
    b64 = box.detach().double().requires_grad_(True)
    r64 = _sine64(b64)
    assert float((out.detach().double() - r64.detach()).abs().max()) < 2e-6          # |p| <= 2 pi: a few fp32 ulps of the argument
    assert float((out.detach() - ref).abs().max()) < 2e-6                     # and the reference's own fp32 expression
    gout = torch.randn(n, 768, device="cuda", generator=g)
    out.backward(gout)
    r64.backward(gout.double())
    assert _rel(box.grad, b64.grad) < 1e-5


@pytest.mark.parametrize("shared", [True, False])
def test_query_pos_product(shared):
    from monodetr_b200 import functional as Fn
    B, rows, C = 8, 550, 256
    g = torch.Generator(device="cuda").manual_seed(3)
    raw = torch.randn(*(() if shared else (B,)), rows, C, device="cuda", generator=g).requires_grad_(True)
    for with_scale in (False, True):
        scale = torch.randn(B, rows, C, device="cuda", generator=g).requires_grad_(True) if with_scale else None
        qp = Fn.query_pos(scale, raw, B)
        want = raw.detach().expand(B, rows, C) * (scale.detach() if with_scale else 1.0)
        assert torch.equal(qp, want)
        gout = torch.randn(B, rows, C, device="cuda", generator=g)
        raw.grad = None
        qp.backward(gout)
        r64 = raw.detach().double().requires_grad_(True)
        s64 = scale.detach().double().requires_grad_(True) if with_scale else None
        (r64.expand(B, rows, C) * (s64 if with_scale else 1.0)).backward(gout.double())
        assert _rel(raw.grad, r64.grad) < 1e-6
        if with_scale:
            assert torch.equal(scale.grad, gout * raw.detach().expand(B, rows, C))
        # the batch sum is fixed-order: the same bits every time
        raw2 = raw.detach().clone().requires_grad_(True)
        Fn.query_pos(scale.detach() if with_scale else None, raw2, B).backward(gout)
        assert torch.equal(raw2.grad, raw.grad)


def _decoder_msda_inputs(B, Lq, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    M, L, P, D = 8, 4, 4, 32
    hw = [(12, 40), (6, 20), (3, 10), (2, 5)]
    shapes = torch.tensor(hw, dtype=torch.long, device="cuda")
    lsi = torch.cat((shapes.new_zeros(1), shapes.prod(1).cumsum(0)[:-1]))
    S = sum(h * w for h, w in hw)
    value = torch.randn(B, S, M, D, device="cuda", generator=g)
    off = torch.randn(B, Lq, M * L * P * 2, device="cuda", generator=g) * 3.0
    logits = torch.randn(B, Lq, M * L * P, device="cuda", generator=g)
    boxes = torch.rand(Lq, 6, device="cuda", generator=g)
    boxes[:, 2:] = boxes[:, 2:] * 0.3                                  # wide boxes near the borders: samples fall off the image
    boxes[: Lq // 4, :2] = boxes[: Lq // 4, :2] * 0.05
    boxes[Lq // 4: Lq // 2, :2] = 1.0 - boxes[Lq // 4: Lq // 2, :2] * 0.05
    return value, shapes, lsi, off, logits, boxes, (M, L, P)


def _box_grad_reference(value, shapes, lsi, loc, attn, gout, off, P):
    """The shared-box gradient from the fp64 MSDA backward at the given (fp32) sampling locations plus the analytic box chain in
    fp64, and the queries none of whose samples lies within 1e-5 of a cell border.  d(bilinear)/d(location) jumps at the borders,
    and the fp64 path floors loc * W - 0.5 where the fp32 kernels floor its fp32 rounding: only those queries are held to the
    fp64 values element for element."""
    from monodetr_b200.msda import ms_deform_attn_backward
    B, Lq, M, L = loc.shape[:4]
    _, gl64, _ = ms_deform_attn_backward(value.double(), shapes, lsi, loc.double(), attn.double(), gout.double(), 64)
    gl64 = gl64.view(*loc.shape)
    o64 = off.detach().double().view(*loc.shape)
    dxy = gl64.sum(dim=(0, 2, 3, 4))
    dwh = (gl64 * o64).sum(dim=(0, 2, 3, 4)) * (0.5 / P)
    want = torch.stack((dxy[:, 0], dxy[:, 1], dwh[:, 0], dwh[:, 0], dwh[:, 1], dwh[:, 1]), -1)
    wh = torch.stack((shapes[:, 1], shapes[:, 0]), -1).double()[None, None, None, :, None, :]
    cell = loc.double() * wh - 0.5
    near = ((cell - cell.round()).abs() < 1e-5).flatten(2).any(-1).any(0)        # (Lq,)
    return want, ~near


def test_msda_shared_box_gradient():
    """Decoder shape (B = 8, Lq = 550, 6-d boxes shared by the batch): the box gradient of the two-step path against the fp64
    MSDA backward at the same sampling locations plus the analytic box chain in fp64, at the MSDA fp32 bar."""
    from monodetr_b200 import functional as Fn
    from monodetr_b200.msda import ms_deform_attn_backward
    B, Lq = 8, 550
    value, shapes, lsi, off, logits, boxes, (M, L, P) = _decoder_msda_inputs(B, Lq, 5)
    boxes.requires_grad_(True)
    loc, attn = Fn._MsdaPrepShared.apply(off, logits, boxes, shapes, M, L, P)
    assert float(((loc < 0) | (loc > 1)).float().mean()) > 0.05               # a good share of the samples is off the image
    out = Fn.msda(value, shapes, lsi, loc, attn)
    gout = torch.randn_like(out)
    out.backward(gout)
    want, keep = _box_grad_reference(value, shapes, lsi, loc.detach(), attn.detach(), gout, off, P)
    assert float(keep.float().mean()) > 0.9
    got = boxes.grad.double()
    np.testing.assert_allclose(got[keep].cpu().numpy(), want[keep].cpu().numpy(), rtol=1e-4, atol=1e-5 * float(want.abs().max()))
    # per-image mode of the same entry point, on the fp32 backward's d loc: its batch sum in fp64 is the shared gradient
    from monodetr_b200 import _lib
    gl32 = ms_deform_attn_backward(value, shapes, lsi, loc.detach(), attn.detach(), gout, 64)[1].contiguous()
    per = torch.empty(B, Lq, 6, device="cuda")
    _lib.call("mdb_msda_ref_grad_f32", gl32, off.contiguous(), B, Lq, M, L, P, 0, per)
    g = gl32.double().view(B, Lq, M, L, P, 2)
    o = off.double().view(B, Lq, M, L, P, 2)
    dxy_b = g.sum(dim=(2, 3, 4))
    dwh_b = (g * o).sum(dim=(2, 3, 4)) * (0.5 / P)
    want_b = torch.stack((dxy_b[..., 0], dxy_b[..., 1], dwh_b[..., 0], dwh_b[..., 0], dwh_b[..., 1], dwh_b[..., 1]), -1)
    np.testing.assert_allclose(per.double().cpu().numpy(), want_b.cpu().numpy(), rtol=1e-4,
                               atol=1e-5 * float(want_b.abs().max()))
    np.testing.assert_allclose(got.cpu().numpy(), want_b.sum(0).cpu().numpy(), rtol=1e-4, atol=1e-5 * float(want.abs().max()))


@pytest.mark.parametrize("B", [1, 8])
def test_fused_msda_box_gradient(B):
    """mdb_msda_fused_backward_ref_f32 + mdb_msda_ref_partials_reduce_f32 at the decoder shape (Lq = 550, 6-d boxes shared by the
    batch, samples off the image edges): the box gradient against the fp64 MSDA backward at the same sampling locations plus the
    analytic box chain in fp64, at the MSDA fp32 bar; offsets / logits gradients identical to mdb_msda_fused_backward_f32's."""
    from monodetr_b200 import _lib, functional as Fn
    from monodetr_b200.msda import ms_deform_attn_backward
    Lq = 550
    value, shapes, lsi, off, logits, boxes, (M, L, P) = _decoder_msda_inputs(B, Lq, 21 + B)
    boxes.requires_grad_(True)
    off.requires_grad_(True)
    logits.requires_grad_(True)
    n0 = _lib.launch_count()
    out = Fn.msda_shared_boxes(value, shapes, lsi, off, logits, boxes, M, L, P)
    gout = torch.randn_like(out)
    out.backward(gout)
    assert _lib.launch_count() - n0 == 3                      # fused forward, fused backward with partials, box reduction
    loc, attn = Fn._MsdaPrepShared.apply(off.detach(), logits.detach(), boxes.detach(), shapes, M, L, P)
    assert float(((loc < 0) | (loc > 1)).float().mean()) > 0.05
    want, keep = _box_grad_reference(value, shapes, lsi, loc, attn, gout, off, P)
    assert float(keep.float().mean()) > 0.9
    got = boxes.grad.double()
    np.testing.assert_allclose(got[keep].cpu().numpy(), want[keep].cpu().numpy(), rtol=1e-4, atol=1e-5 * float(want.abs().max()))
    # every query, border samples included, against the fp32 backward's d loc at the same locations (same floors), chained in fp64
    gl32 = ms_deform_attn_backward(value, shapes, lsi, loc, attn, gout, 64)[1].double().view(*loc.shape)
    o = off.detach().double().view(*loc.shape)
    dxy, dwh = gl32.sum(dim=(0, 2, 3, 4)), (gl32 * o).sum(dim=(0, 2, 3, 4)) * (0.5 / P)
    want32 = torch.stack((dxy[:, 0], dxy[:, 1], dwh[:, 0], dwh[:, 0], dwh[:, 1], dwh[:, 1]), -1)
    np.testing.assert_allclose(got.cpu().numpy(), want32.cpu().numpy(), rtol=1e-4, atol=1e-5 * float(want.abs().max()))
    refc = boxes.detach()[None, :, None].expand(B, Lq, L, 6).contiguous()
    _, goff, glog = Fn.msda_fused_backward_raw(value, shapes, lsi, off.detach(), logits.detach(), refc, gout)
    assert torch.equal(goff, off.grad) and torch.equal(glog, logits.grad)
    # no box gradient wanted (eval / no_grad): the plain fused forward, the same values
    with torch.no_grad():
        out2 = Fn.msda_shared_boxes(value, shapes, lsi, off, logits, boxes, M, L, P)
    assert torch.equal(out2, out.detach())


def test_anchor_gradient_near_the_clamp():
    """sigmoid(refpoint_embed) at logits up to +-14, where inverse_sigmoid's clamp at 1e-5 switches terms off, through the
    level-0 box (box refinement's reference gradient) plus the sine and deformable-attention contributions."""
    from monodetr_b200 import functional as Fn
    B, nq = 3, 550
    g = torch.Generator(device="cuda").manual_seed(9)
    w = torch.randn(nq, 6, device="cuda", generator=g) * 2
    w[:60] = torch.linspace(-14.0, 14.0, 360, device="cuda").view(60, 6)
    w.requires_grad_(True)
    tmp = torch.randn(B, nq, 6, device="cuda", generator=g)
    a, b, c = (torch.randn(*s, device="cuda", generator=g) for s in ((nq, 6), (nq, 6), (B, nq, 6)))
    r_sine, r_msda, r_head = Fn.anchors(w, B)
    assert torch.equal(r_sine, r_msda) and torch.equal(r_head, r_sine.expand(B, nq, 6))
    y = Fn.box_refine(tmp, r_head)
    ((r_sine * a).sum() + (r_msda * b).sum() + (y * c).sum()).backward()
    r64 = r_sine.detach().double().requires_grad_(True)                    # the fp32 anchors: the clamp decides alike
    y64 = (tmp.double() + om.inverse_sigmoid(r64.expand(B, nq, 6))).sigmoid()
    ((r64 * a.double()).sum() + (r64 * b.double()).sum() + (y64 * c.double()).sum()).backward()
    want = r64.grad * r64.detach() * (1 - r64.detach())
    assert _rel(w.grad, want) < 1e-5
    clamped = (r64.detach() < 1e-5) | (1 - r64.detach() < 1e-5)
    assert int(clamped.sum()) > 0


# ---- the whole model ---------------------------------------------------------------------------------------------------------
def _model(dropout=0.0):
    from monodetr_b200 import build_monodetr
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    m, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, use_dab=True, dropout=dropout))
    m.load_state_dict(om.with_aliases(od.deterministic_state_dict()))
    if dropout == 0.0:
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
            if isinstance(mod, torch.nn.MultiheadAttention):
                mod.dropout = 0.0
    return m.cuda()


def _flat(out):
    items = [(k, out[k]) for k in ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits")]
    items += [(f"aux{i}_{k}", v) for i, a in enumerate(out["aux_outputs"]) for k, v in a.items()]
    return items


@pytest.fixture(scope="module")
def golden(golden_dir):
    return np.load(os.path.join(golden_dir, "dab.npz"))


@pytest.mark.parametrize("precision", ["bf16x3", "tf32x3"])
def test_model_matches_the_reference(precision, golden):
    """Eval at 1 x 192 x 640, train mode (dropout off) at 1 and 2 x 96 x 320: every output incl. aux within 1e-3
    (max|a - b| / max|b| over the stored elements)."""
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from gen_golden_reference_pins import sampled_forward
    from monodetr_b200 import tc
    prev = tc.get_precision()
    tc.set_precision(precision)
    try:
        m = _model()
        for training, B, (H, W), prefix in ((False, 1, (192, 640), "fwd_eval"), (True, 1, (96, 320), "b1.fwd_train"),
                                            (True, 2, (96, 320), "b2.fwd_train")):
            m.train(training)
            images, calibs, sizes = om.synthetic_inputs(B, 0, H=H, W=W)
            with torch.no_grad():
                out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
            worst = []
            for k, v in _flat(out):
                a, b = sampled_forward(golden, f"{prefix}_{k}", v.float().cpu().numpy())
                rel = float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-12))
                worst.append((rel, k))
                assert rel < 1e-3, (prefix, k, rel)
            print(precision, prefix, "worst", max(worst))
    finally:
        tc.set_precision(prev)


STAGES = ("backbone", "input_proj", "depth_predictor", "depthaware_transformer.encoder", "depthaware_transformer.decoder.layers",
          "depthaware_transformer.decoder.query_scale", "depthaware_transformer.decoder.ref_point_head",
          "depthaware_transformer.level_embed", "tgt_embed", "refpoint_embed", "class_embed", "bbox_embed", "dim_embed_3d",
          "angle_embed", "depth_embed")


@pytest.mark.parametrize("B,H,W", [(1, 192, 640), (2, 192, 640)])
def test_gradients_per_stage(B, H, W):
    """Frozen sampling locations: every gradient against the CPU oracle, with the bars of tests/test_model_grad_gpu.py
    (median < 1e-3, every tensor < 2e-2, max-norm and L2), the anchors and the DAB MLPs included; query_scale_bbox gets none."""
    from monodetr_b200.ms_deform_attn import MSDeformAttn
    m = _model().train()
    images, calibs, sizes = om.synthetic_inputs(B, 11, H=H, W=W)
    MSDeformAttn.freeze_sampling_locations = True
    om.FREEZE_SAMPLING = True
    try:
        out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
        om.surrogate_loss(out).backward()
        torch.cuda.synchronize()
        sd = {k: v.clone().requires_grad_(v.dtype.is_floating_point) for k, v in od.deterministic_state_dict().items()}
        om.surrogate_loss(od.forward(sd, images, calibs, sizes, training=True)).backward()
    finally:
        MSDeformAttn.freeze_sampling_locations = False
        om.FREEZE_SAMPLING = False
    assert all(p.grad is None for p in m.depthaware_transformer.decoder.query_scale_bbox.parameters())
    params = dict(m.named_parameters())
    for name, p in params.items():        # analytically zero (see tests/test_backbone_variants_gpu.py)
        if name.endswith(("sa_kcontent_proj.bias", "sa_kpos_proj.bias")) and p.grad is not None:
            wmax = float(params[name[:-len("bias")] + "weight"].grad.abs().max())
            assert float(p.grad.abs().max()) <= 5e-3 * wmax and float(sd[name].grad.abs().max()) <= 1e-4 * wmax, name
            p.grad = None
    per_stage, rel_max, rel_l2 = {}, [], []
    for name, p in m.named_parameters():
        if name.startswith(("depthaware_transformer.decoder.bbox_embed", "depthaware_transformer.decoder.dim_embed")):
            continue
        if not p.requires_grad or p.grad is None:
            continue
        gref = sd[name].grad
        assert gref is not None, name
        scale = float(gref.abs().max())
        if scale < 1e-7:
            continue
        d = p.grad.cpu() - gref
        r, l2 = float(d.abs().max()) / scale, float(d.norm() / gref.norm())
        rel_max.append(r)
        rel_l2.append(l2)
        stage = next(s for s in STAGES if name.startswith(s))
        cur = per_stage.get(stage, (0.0, 0.0, ""))
        per_stage[stage] = (max(cur[0], r), max(cur[1], l2), name if r > cur[0] else cur[2])
    print(B, {k: f"{v[0]:.1e} {v[1]:.1e}" for k, v in per_stage.items()},
          "median", f"{float(np.median(rel_max)):.2e} {float(np.median(rel_l2)):.2e}", "tensors", len(rel_max))
    for s in ("tgt_embed", "refpoint_embed", "depthaware_transformer.decoder.query_scale",
              "depthaware_transformer.decoder.ref_point_head"):
        assert s in per_stage, s
    assert float(np.median(rel_max)) < 1e-3 and float(np.median(rel_l2)) < 1e-3
    for stage, (r, l2, name) in per_stage.items():
        assert r < 2e-2 and l2 < 2e-2, (stage, name, r, l2)


def test_anchor_gradient_matches_the_reference_at_batch_2(golden):
    """Unfrozen sampling locations, B = 2: the whole anchor gradient (head box + sine embedding + the deformable attention's
    box gradient, summed over the batch) against the reference's, in L2 (bilinear-border noise bounds the max-norm)."""
    m = _model().train()
    images, calibs, sizes = om.synthetic_inputs(2, 0, H=96, W=320)
    out = m(images.cuda(), calibs.cuda(), None, sizes.cuda())
    om.surrogate_loss(out).backward()
    full = golden["b2.grad_full.refpoint_embed.weight"]
    got = m.refpoint_embed.weight.grad.cpu().numpy()
    assert float(np.linalg.norm(got - full) / np.linalg.norm(full)) < 2e-2
    names = json.loads(golden["b2.grad_names"].tobytes())
    assert "refpoint_embed.weight" in names


# ---- reproducible mode and graph capture ---------------------------------------------------------------------------------------
def _setup(dev, B=2):
    from bench_extras import CRIT_CFG, synthetic_targets
    from monodetr_b200 import build_monodetr, tc
    from monodetr_b200.bench_model import synthetic_batch
    from monodetr_b200.criterion import build_criterion
    from monodetr_b200.ddp import FlatGradBucket
    from monodetr_b200.monodetr import DEFAULT_MODEL_CFG
    from monodetr_b200.optim import FusedAdamW
    tc.set_precision("bf16x3")
    torch.manual_seed(0)
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, use_dab=True, dropout=0.1))
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
        flat = [v for _, v in _flat(out)]
        losses = [state["losses"][k] for k in sorted(state["losses"])]
        grads = [p.grad for p in model.parameters() if p.grad is not None]
        return [t.detach().clone() for t in flat], [t.detach().clone() for t in losses], [t.clone() for t in grads], \
            [p.detach().clone() for p in model.parameters()]
    return model, bucket, it, snapshot


def _assert_equal(a, b):
    for name, xs, ys in zip(("outputs", "losses", "gradients", "parameters"), a, b):
        assert len(xs) == len(ys), name
        bad = [i for i, (x, y) in enumerate(zip(xs, ys)) if not torch.equal(x, y)]
        assert not bad, (name, len(bad), len(xs))


def test_training_iteration_is_bit_reproducible_eager_and_as_a_cuda_graph():
    """Reproducible mode, use_dab: forward with dropout, the device criterion, backward and FusedAdamW give identical bits
    twice eagerly, and a replayed CUDA graph of the whole iteration (captured without a host synchronisation) gives the
    eager bits."""
    from monodetr_b200 import kernels as K
    dev = torch.device("cuda", torch.cuda.current_device())
    prev = monodetr_b200.set_deterministic(True)
    try:
        runs = []
        for _ in range(2):
            model, _, it, snap = _setup(dev)
            K.reseed(dev, 4242)
            it()
            runs.append(snap())
        assert model.refpoint_embed.weight.grad is not None and model.tgt_embed.weight.grad is not None
        _assert_equal(runs[0], runs[1])

        _, _, it_a, snap_a = _setup(dev)
        _, bucket_b, it_b, snap_b = _setup(dev)
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
        torch.cuda.set_sync_debug_mode("error")
        try:
            with torch.cuda.graph(graph):
                it_b()
        finally:
            torch.cuda.set_sync_debug_mode("default")
        bucket_b.freeze_sources()
        graph.replay()
        torch.cuda.synchronize()
        _assert_equal(eager, snap_b())
    finally:
        monodetr_b200.set_deterministic(prev)
