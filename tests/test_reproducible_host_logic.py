"""CPU: host logic of the reproducible mode (mdb_set_deterministic) through the stand-in device library (tests/fake_device_lib.py).

In reproducible mode the depth predictor resizes a CUDA map with the library's NHWC bilinear kernel instead of F.interpolate (whose
CUDA backward scatters with atomics; depth_predictor.library_resize).  The stand-in library gets host versions of those two entry
points here, and the model-level test routes the resize through them as on the GPU.  The default mode never reaches them and launches exactly as many kernels as before."""
import pytest
import torch
import torch.nn.functional as F

from oracle import monodetr_torch as om
from test_model_host_logic import _build, _rel

NEW_ENTRY_POINTS = ("mdb_upsample_bilinear_nhwc_forward_f32", "mdb_upsample_bilinear_nhwc_backward_f32")


def _upsample(x, Ho, Wo):
    """Bilinear resize as include/monodetr_b200.h states it (src = in/out * (dst + 0.5) - 0.5 clamped at 0, i1 = i0 + (i0 < in - 1)),
    x (B, H, W, C), restated with torch indexing."""
    def axis(n_in, n_out):
        src = ((torch.arange(n_out, dtype=torch.float32) + 0.5) * (float(n_in) / float(n_out)) - 0.5).clamp(min=0)
        i0 = src.long()
        i1 = torch.where(i0 < n_in - 1, i0 + 1, i0)
        l1 = src - i0.float()
        return i0, i1, 1 - l1, l1
    h0, h1, hl0, hl1 = axis(x.shape[1], Ho)
    w0, w1, wl0, wl1 = axis(x.shape[2], Wo)
    hl0, hl1, wl0, wl1 = hl0.view(1, -1, 1, 1), hl1.view(1, -1, 1, 1), wl0.view(1, 1, -1, 1), wl1.view(1, 1, -1, 1)
    r0, r1 = x[:, h0], x[:, h1]
    return hl0 * (wl0 * r0[:, :, w0] + wl1 * r0[:, :, w1]) + hl1 * (wl0 * r1[:, :, w0] + wl1 * r1[:, :, w1])


def _add_resize_entry_points(fake):
    """Host implementations of the two resize entry points on the stand-in library (the model calls them only in reproducible mode)."""
    from fake_device_lib import f32

    def forward(x, y, B, Hi, Wi, Ho, Wo, C, stream):
        f32(y, B, Ho, Wo, C).copy_(_upsample(f32(x, B, Hi, Wi, C), Ho, Wo))
        return 0

    def backward(dy, dx, B, Hi, Wi, Ho, Wo, C, stream):
        with torch.enable_grad():
            x = torch.zeros(B, Hi, Wi, C, requires_grad=True)
            (g,) = torch.autograd.grad(_upsample(x, Ho, Wo), x, f32(dy, B, Ho, Wo, C))
        f32(dx, B, Hi, Wi, C).copy_(g)
        return 0
    fake.mdb_upsample_bilinear_nhwc_forward_f32 = forward
    fake.mdb_upsample_bilinear_nhwc_backward_f32 = backward


def _step(m, batch):
    from monodetr_b200 import _lib
    from monodetr_b200.bench_model import surrogate_loss
    m.train()
    images, calibs, sizes = om.synthetic_inputs(batch, 0, H=96, W=320)
    n0 = _lib.launch_count()
    out = m(images, calibs, None, sizes)
    n1 = _lib.launch_count()
    surrogate_loss(out).backward()
    return out, (images, calibs, sizes), n1 - n0, _lib.launch_count() - n1


def test_reproducible_mode_uses_the_library_resize_and_matches_the_oracle(monkeypatch):
    fake, m, sd = _build(monkeypatch, "bf16x3")
    _add_resize_entry_points(fake)
    fake.deterministic = 1
    from monodetr_b200 import depth_predictor
    monkeypatch.setattr(depth_predictor, "library_resize", lambda x: True)      # the host tensors stand for CUDA ones

    def no_interpolate(*a, **k):
        raise AssertionError("F.interpolate reached in reproducible mode")
    monkeypatch.setattr(F, "interpolate", no_interpolate)
    out, (images, calibs, sizes), _, _ = _step(m, 2)
    monkeypatch.undo()          # the oracle below is plain torch

    for fn in NEW_ENTRY_POINTS:
        assert fake.calls.get(fn, 0) == 1, fn

    sdg = {k: (v.clone().requires_grad_() if v.is_floating_point() else v) for k, v in sd.items()}
    ref = om.forward(sdg, images, calibs, sizes, training=True)
    om.surrogate_loss(ref).backward()
    for k in ("pred_logits", "pred_boxes", "pred_3d_dim", "pred_depth", "pred_angle", "pred_depth_map_logits"):
        assert _rel(out[k].detach(), ref[k].detach()) < 1e-4, (k, _rel(out[k].detach(), ref[k].detach()))
    by_name = om.with_aliases(sdg)
    errs = []
    for name, p in m.named_parameters():
        want = by_name[name].grad
        if not p.requires_grad or p.grad is None:
            continue
        errs.append((_rel(p.grad, want), name, float(want.abs().max())))
    errs.sort()
    assert len(errs) == 313
    # the bars of tests/test_model_host_logic.py in BF16x3
    assert errs[len(errs) // 2][0] < 1e-3, errs[len(errs) // 2]
    for err, name, scale in errs:
        assert err < 1e-1 or scale < 1e-6, (name, err, scale)


@pytest.mark.parametrize("B,Hi,Wi,Ho,Wo", [(2, 3, 10, 6, 20), (1, 7, 13, 24, 80), (1, 24, 80, 10, 33)])
def test_resize_wrapper_matches_interpolate(monkeypatch, B, Hi, Wi, Ho, Wo):
    """functional.upsample_bilinear_nhwc through the C ABI (pointers, sizes) against F.interpolate, forward and backward."""
    fake, _, _ = _build(monkeypatch)
    _add_resize_entry_points(fake)
    from monodetr_b200 import functional as Fn
    g = torch.Generator().manual_seed(Hi * Wo)
    x = torch.randn(B, Hi, Wi, 8, generator=g, requires_grad=True)
    dy = torch.randn(B, Ho, Wo, 8, generator=g)
    y = Fn.upsample_bilinear_nhwc(x, (Ho, Wo))
    (dx,) = torch.autograd.grad(y, x, dy)
    ref = F.interpolate(x.permute(0, 3, 1, 2), size=(Ho, Wo), mode="bilinear").permute(0, 2, 3, 1)
    (rdx,) = torch.autograd.grad(ref, x, dy)
    # (the kernel's arithmetic against torch's CUDA resize is pinned by tests/test_reproducible_gpu.py; torch's CPU resize rounds its
    # source indices of a non-integer scale slightly differently, ~4e-6 here)
    assert y.shape == ref.shape and _rel(y.detach(), ref.detach()) < 1e-5 and _rel(dx, rdx) < 1e-5
    assert fake.calls["mdb_upsample_bilinear_nhwc_forward_f32"] == 1 and fake.calls["mdb_upsample_bilinear_nhwc_backward_f32"] == 1


@pytest.mark.parametrize("deterministic", [False, True])
def test_launch_counts(monkeypatch, deterministic):
    """Default mode: 232 forward and 428 backward launches for one BF16x3 step, never an entry point of the reproducible mode.
    Reproducible mode (238 / 461) also takes the two-step MSDA path in the encoder, the library's resize, a second launch per
    LayerNorm and head-depth backward for the parameter / map gradients, and the depth tail's ordered embedding gradient."""
    fake, m, _ = _build(monkeypatch, "bf16x3")
    if deterministic:
        _add_resize_entry_points(fake)
        from monodetr_b200 import depth_predictor
        monkeypatch.setattr(depth_predictor, "library_resize", lambda x: True)
    fake.deterministic = int(deterministic)
    _, _, n_fwd, n_bwd = _step(m, 1)
    if deterministic:
        assert (n_fwd, n_bwd) == (238, 461)
    else:
        assert (n_fwd, n_bwd) == (232, 428)
        for fn in NEW_ENTRY_POINTS:
            assert fake.calls.get(fn, 0) == 0, fn


@pytest.mark.parametrize("env,expect", [("1", "1"), (None, "0")])
def test_environment_switch_starts_the_library_in_reproducible_mode(env, expect):
    """MDB_DETERMINISTIC=1 (e.g. for two bench.py runs compared file for file): the loaded library is in reproducible mode."""
    import os
    import subprocess
    import sys
    e = {k: v for k, v in os.environ.items() if k != "MDB_DETERMINISTIC"}
    if env is not None:
        e["MDB_DETERMINISTIC"] = env
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", "from monodetr_b200 import _lib; print(_lib.lib().mdb_get_deterministic())"],
                         cwd=root, env=e, capture_output=True, text=True, check=True).stdout
    assert out.strip() == expect
