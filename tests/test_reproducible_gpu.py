"""Reproducible mode (monodetr_b200.set_deterministic(True)) on the GPU.

Per kernel: two calls give the same bits, and the result holds the bars of the default path (tests/test_attn_norm_gpu.py,
tests/test_heads_gpu.py).  The NHWC bilinear resize against F.interpolate.  The whole training iteration (forward with dropout ->
device SetCriterion -> backward -> FusedAdamW) twice from the same state, as a replayed CUDA graph, and under
torch.use_deterministic_algorithms(True).  The per-stage gradient comparison with the oracle in this mode."""
import pytest
import torch
import torch.nn.functional as F

import monodetr_b200
from monodetr_b200 import _lib, kernels as K

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-12))


@pytest.fixture
def repro():
    prev = monodetr_b200.set_deterministic(True)
    try:
        yield
    finally:
        monodetr_b200.set_deterministic(prev)


def _twice(fn):
    """fn() twice in reproducible mode (bit-identical), and once in the default mode."""
    a, b = fn(), fn()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    monodetr_b200.set_deterministic(False)
    try:
        d = fn()
    finally:
        monodetr_b200.set_deterministic(True)
    return a, d


# ---- LayerNorm -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,C", [(1000, 128), (81600, 256), (4400, 256), (777, 512), (3, 256)])
def test_layernorm_backward(repro, M, C):
    g = torch.Generator(device="cuda").manual_seed(M + C)
    x, r, dy = (torch.randn(M, C, device="cuda", generator=g) for _ in range(3))
    gamma, beta = 1 + 0.1 * torch.randn(C, device="cuda", generator=g), 0.1 * torch.randn(C, device="cuda", generator=g)
    seed = torch.tensor([12345], dtype=torch.int64, device="cuda")
    prior_g, prior_b = torch.randn(C, device="cuda", generator=g), torch.randn(C, device="cuda", generator=g)

    def run():
        y, mean, rstd = K.add_layernorm_forward(x, r, gamma, beta, 1e-5, 0.1, 7, seed)
        dx, dres, dg, db = K.add_layernorm_backward(dy, x, r, gamma, mean, rstd, 0.1, 7, seed)
        dx2, dres2 = torch.empty_like(x), torch.empty_like(x)
        ag, ab = prior_g.clone(), prior_b.clone()                 # accumulate = 1
        _lib.call("mdb_add_layernorm_backward_f32", dy, x, r, gamma, mean, rstd, dx2, dres2, ag, ab, M, C, 0.1, seed, 7, 1,
                  launches=2 if _lib.deterministic() else 1)
        return y, dx, dres, dg, db, ag, ab

    (y, dx, dres, dg, db, ag, ab), dflt = _twice(run)
    for a, b in zip((y, dx, dres), dflt[:3]):
        assert torch.equal(a, b)                                  # same per-row kernels in both modes
    assert _rel(dg, dflt[3]) < 1e-5 and _rel(db, dflt[4]) < 1e-5
    assert torch.allclose(ag, prior_g + dg, rtol=1e-6, atol=1e-6) and torch.allclose(ab, prior_b + db, rtol=1e-6, atol=1e-6)
    # accumulate = 1 in the default mode: atomics onto the prior, in another order than the accumulate = 0 call's
    assert _rel(dflt[5], prior_g + dflt[3]) < 1e-5 and _rel(dflt[6], prior_b + dflt[4]) < 1e-5
    # against torch without dropout (the mask of the kernels is a hash, not torch's RNG)
    yn, mean, rstd = K.add_layernorm_forward(x, r, gamma, beta, 1e-5)
    _, _, dgn, dbn = K.add_layernorm_backward(dy, x, r, gamma, mean, rstd)
    gr, br = gamma.clone().requires_grad_(), beta.clone().requires_grad_()
    ref = F.layer_norm(x + r, (C,), gr, br, 1e-5)
    ref.backward(dy)
    assert _rel(yn, ref.detach()) < 1e-5
    assert _rel(dgn, gr.grad) < 1e-4 and _rel(dbn, br.grad) < 1e-4


# ---- GroupNorm -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("HW", [7680, 1920, 480, 120])          # the four levels of a 1280 x 384 image
@pytest.mark.parametrize("relu", [False, True])
def test_groupnorm(repro, HW, relu):
    B, C, G = 2, 256, 32
    g = torch.Generator(device="cuda").manual_seed(HW + relu)
    x = torch.randn(B, HW, C, device="cuda", generator=g) * 2 + 0.5
    gamma, beta = 1 + 0.1 * torch.randn(C, device="cuda", generator=g), 0.1 * torch.randn(C, device="cuda", generator=g)
    dy = torch.randn(B, HW, C, device="cuda", generator=g)

    def run():
        y, mean, rstd = K.groupnorm_forward(x, gamma, beta, G, 1e-5, relu)
        dx, dg, db = K.groupnorm_backward(dy, x, y, gamma, mean, rstd, G, relu)
        return y, mean, rstd, dx, dg, db

    (y, mean, rstd, dx, dg, db), dflt = _twice(run)
    assert _rel(y, dflt[0]) < 1e-5 and _rel(dx, dflt[3]) < 1e-4 and _rel(dg, dflt[4]) < 1e-5 and _rel(db, dflt[5]) < 1e-5
    xr, gr, br = x.clone().requires_grad_(), gamma.clone().requires_grad_(), beta.clone().requires_grad_()
    ref = F.group_norm(xr.transpose(1, 2), G, gr, br, 1e-5).transpose(1, 2)
    if relu:
        ref = F.relu(ref)
    ref.backward(dy)
    assert _rel(y, ref.detach()) < 1e-5
    assert _rel(dx, xr.grad) < 1e-4
    assert _rel(dg, gr.grad) < 1e-4 and _rel(db, br.grad) < 1e-4


# ---- heads -------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N,H,W", [(2, 550, 24, 80), (1, 7, 5, 9)])
def test_head_depth_and_depth_sample_backward(repro, B, N, H, W):
    from monodetr_b200 import functional as Fn
    g = torch.Generator(device="cuda").manual_seed(B * 10 + N)
    coord = torch.rand(B, N, 6, device="cuda", generator=g)
    coord[..., :2] = coord[..., :2] * 1.3 - 0.15                  # some centres outside the map
    coord[0, :4, :2] = torch.tensor([[0.5, 0.5], [0.5, 0.5], [0.0, 0.0], [1.0, 1.0]], device="cuda")   # shared corners, map edges
    size3d, reg = torch.randn(B, N, 3, device="cuda", generator=g), torch.randn(B, N, 2, device="cuda", generator=g)
    wd = torch.rand(B, H, W, device="cuda", generator=g) * 60
    calibs = torch.zeros(B, 3, 4, device="cuda"); calibs[:, 0, 0] = 721.5377
    sizes = torch.tensor([[1242., 375.]], device="cuda").repeat(B, 1)
    dout = torch.randn(B, N, 2, device="cuda", generator=g)
    xy = (coord[..., :2] - 0.5) * 2

    def run():
        ins = [t.clone().requires_grad_() for t in (coord, size3d, reg, wd)]
        grads = torch.autograd.grad(Fn.head_depth(*ins, calibs, sizes), ins, dout)
        w = wd.clone().requires_grad_()
        (gs,) = torch.autograd.grad(Fn.depth_sample(w, xy), w, dout[..., 0])
        return (*grads, gs)

    a, dflt = _twice(run)
    for x, y in zip(a[:3], dflt[:3]):
        assert torch.equal(x, y)
    assert torch.allclose(a[3], dflt[3], rtol=1e-4, atol=1e-5 * float(dflt[3].abs().max()))
    w = wd.clone().requires_grad_()
    (ref,) = torch.autograd.grad(F.grid_sample(w.unsqueeze(1), xy.unsqueeze(2), mode="bilinear", align_corners=True).view(B, N),
                                 w, dout[..., 0])
    assert torch.allclose(a[4], ref, rtol=1e-4, atol=1e-5 * float(ref.abs().max()))
    assert torch.allclose(a[3], ref / 3, rtol=1e-4, atol=1e-5 * float(ref.abs().max()))


@pytest.mark.parametrize("B,H,W,flat", [(2, 24, 80, False), (8, 24, 80, True), (1, 3, 5, False)])
def test_depth_tail_backward(repro, B, H, W, flat):
    from monodetr_b200 import functional as Fn
    g = torch.Generator(device="cuda").manual_seed(B + H)
    nb, E, C, dmax = 81, 61, 256, 60.0
    logits = torch.zeros(B, H, W, nb, device="cuda") if flat else torch.randn(B, H, W, nb, device="cuda", generator=g) * 3
    idx = torch.linspace(0, nb - 2, nb - 1, device="cuda")
    bin_size = 2 * (dmax - 1e-3) / ((nb - 1) * nb)
    bins = torch.cat(((idx + 0.5).pow(2) * bin_size / 2 - bin_size / 8 + 1e-3, torch.tensor([dmax], device="cuda")))
    emb = torch.randn(E, C, device="cuda", generator=g)
    d_ip, d_wd = torch.randn(B, H, W, C, device="cuda", generator=g), torch.randn(B, H, W, device="cuda", generator=g)

    def run():
        lg, em = logits.clone().requires_grad_(), emb.clone().requires_grad_()
        wd, ip = Fn.depth_tail(lg, bins, em, dmax)
        return (wd, ip, *torch.autograd.grad((wd, ip), (lg, em), (d_wd, d_ip)))

    a, dflt = _twice(run)
    for x, y in zip(a[:3], dflt[:3]):
        assert torch.equal(x, y)
    assert _rel(a[3], dflt[3]) < 1e-5
    l2, e2 = logits.clone().requires_grad_(), emb.clone().requires_grad_()
    rwd = (F.softmax(l2, dim=-1) * bins).sum(-1)
    x = rwd.clamp(min=0, max=dmax)
    fl = x.floor()
    delta = (x - fl).unsqueeze(-1)
    rip = F.embedding(fl.long(), e2) * (1 - delta) + F.embedding((fl.long() + 1).clamp(max=E - 1), e2) * delta
    _, re = torch.autograd.grad((rwd, rip), (l2, e2), (d_wd, d_ip))
    assert _rel(a[3], re) < 1e-4


def test_sum_mean_squares(repro):
    from monodetr_b200 import functional as Fn
    g = torch.Generator(device="cuda").manual_seed(0)
    xs = [torch.randn(s, device="cuda", generator=g) for s in [(8, 550, 3), (8, 550, 6), (8, 550, 24), (7,), (8, 81, 24, 80)]]
    a, dflt = _twice(lambda: (Fn.sum_mean_squares(xs),))
    ref = sum((x.double() ** 2).mean() for x in xs)
    assert abs(float(a[0]) - float(ref)) < 1e-5 * float(ref)
    assert abs(float(a[0]) - float(dflt[0])) < 1e-5 * float(ref)


# ---- bilinear resize ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,Hi,Wi,Ho,Wo", [(2, 12, 40, 24, 80), (1, 6, 20, 12, 40), (2, 7, 13, 24, 80), (1, 24, 80, 10, 33)])
def test_upsample_bilinear_nhwc(B, Hi, Wi, Ho, Wo):
    """12x40 -> 24x80: the model at 1280x384; 6x20 -> 12x40: at 192x640; then a non-integer up- and down-scale."""
    from monodetr_b200 import functional as Fn
    g = torch.Generator(device="cuda").manual_seed(Hi * Wo)
    x = torch.randn(B, Hi, Wi, 256, device="cuda", generator=g)
    dy = torch.randn(B, Ho, Wo, 256, device="cuda", generator=g)
    xr = x.clone().requires_grad_()
    y = Fn.upsample_bilinear_nhwc(xr, (Ho, Wo))
    (dx,) = torch.autograd.grad(y, xr, dy)
    (dx2,) = torch.autograd.grad(Fn.upsample_bilinear_nhwc(xr, (Ho, Wo)), xr, dy)
    assert torch.equal(dx, dx2)
    xt = x.clone().requires_grad_()
    ref = F.interpolate(xt.permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear").permute(0, 2, 3, 1)
    (rdx,) = torch.autograd.grad(ref, xt, dy)
    print(f"{Hi}x{Wi} -> {Ho}x{Wo}: forward bit-identical to F.interpolate: {torch.equal(y, ref)}, max rel {_rel(y, ref.detach()):.1e}; "
          f"backward max rel {_rel(dx, rdx):.1e}")
    assert _rel(y, ref.detach()) < 1e-6
    assert _rel(dx, rdx) < 1e-5


# ---- the whole training iteration --------------------------------------------------------------------------------------------
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
    model, _ = build_monodetr(dict(DEFAULT_MODEL_CFG, dropout=0.1))
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
        flat = [out[k] for k in sorted(out) if torch.is_tensor(out[k])]
        flat += [a[k] for a in out.get("aux_outputs", []) for k in sorted(a)]
        losses = [state["losses"][k] for k in sorted(state["losses"])]
        grads = [p.grad for p in model.parameters() if p.grad is not None]
        params = [p for p in model.parameters()]
        return [t.detach().clone() for t in flat], [t.detach().clone() for t in losses], [t.clone() for t in grads], \
            [t.detach().clone() for t in params]
    return model, bucket, it, snapshot


def _assert_equal(a, b):
    names = ("outputs", "losses", "gradients", "parameters")
    for name, xs, ys in zip(names, a, b):
        assert len(xs) == len(ys), name
        bad = [i for i, (x, y) in enumerate(zip(xs, ys)) if not torch.equal(x, y)]
        assert not bad, (name, len(bad), len(xs))


def test_training_iteration_is_bit_reproducible_eager_and_as_a_cuda_graph(repro):
    dev = torch.device("cuda", torch.cuda.current_device())
    runs = []
    for _ in range(2):
        _, _, it, snap = _setup(dev)
        K.reseed(dev, 4242)
        it()
        runs.append(snap())
    assert len(runs[0][1]) == 26 and len(runs[0][2]) == 313
    _assert_equal(runs[0], runs[1])

    # a replayed CUDA graph gives the eager bits: two eager iterations on a second copy, the third eager (A) or replayed (B)
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
    with torch.cuda.graph(graph):
        it_b()
    bucket_b.freeze_sources()
    graph.replay()
    torch.cuda.synchronize()
    _assert_equal(eager, snap_b())


def test_training_iteration_under_torch_deterministic_algorithms(repro):
    dev = torch.device("cuda", torch.cuda.current_device())
    _, _, it, snap = _setup(dev)
    K.reseed(dev, 7)
    torch.use_deterministic_algorithms(True)
    try:
        it()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(False)
    assert all(torch.isfinite(t).all() for t in snap()[1])


# ---- correctness in reproducible mode --------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,H,W,freeze", [(1, 192, 640, False), (2, 384, 1280, True)])
def test_gradients_per_stage_in_reproducible_mode(repro, B, H, W, freeze):
    from test_model_grad_gpu import test_gradients_per_stage
    test_gradients_per_stage(B, H, W, freeze)
