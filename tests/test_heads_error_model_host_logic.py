"""The bounds of tests/heads_error_model.py are sharp: fp32 emulations of the kernels (csrc/heads.cu, csrc/elementwise.cu),
in the kernels' order where the order matters (the depth-tail softmax sums as a warp butterfly, colsum's per-lane chains
and slab split in both modes, the resize source index and window), meet the bounds with the constants the GPU test uses,
and each mutant of the shipped arithmetic breaks the bound it targets.  CPU only."""
import numpy as np
import torch

import heads_error_model as em

F32 = torch.float32
F64 = torch.float64
NUM_SMS = 132                                                   # H100 SXM


def _meets(key, y, ref, mag):
    """|y - ref| <= C * mag per element, zero-magnitude elements exact, y finite."""
    y = y.to(F64)
    if not bool(torch.isfinite(y).all()):
        return False
    err = (y - ref).abs()
    pos = mag > 0
    if bool((err[~pos] != 0).any()):
        return False
    return not bool(pos.any()) or float((err[pos] / mag[pos]).max()) <= getattr(em, key)


def _f32(v):
    return torch.tensor(v, dtype=F32)


def _fma32(a, b, c):
    """fp32 fma: the product of two floats is exact in float64; one rounding of the sum (to float64, then float32 -- a double
    rounding that can differ from a true fma only on exact float64 ties, which these inputs do not reach)."""
    return (a.to(F64) * b.to(F64) + c.to(F64)).to(F32)


# ---- box refinement -----------------------------------------------------------------------------------------------------------
def _box_bwd32(dy, y, ref, strict=False):
    g = dy * y * (1 - y)
    eps = _f32(1e-5)
    inside = (ref >= 0) & (ref <= 1)
    lo = ref > eps if strict else ref >= eps
    hi = (1 - ref) > eps if strict else (1 - ref) >= eps
    d = torch.where(inside & lo, 1 / ref, torch.zeros_like(ref)) + torch.where(inside & hi, 1 / (1 - ref), torch.zeros_like(ref))
    return g, g[:, :ref.shape[1]] * d


def test_box_refine_dref_clamp_convention():
    e = _f32(1e-5)
    vals = torch.stack([e, _f32(1) - e, torch.nextafter(e, _f32(1)), _f32(0.5), _f32(0), _f32(1)])
    ref = vals.repeat(4, 1)[:, :6].reshape(-1, 2)
    n = ref.shape[0]
    g = torch.Generator().manual_seed(0)
    tmp, dy = torch.randn(n, 6, generator=g), torch.randn(n, 6, generator=g)
    y = torch.sigmoid(tmp)
    _, _, r, m = em.box_refine_bwd(dy, y, ref)
    assert _meets("C_BOX_BWD", _box_bwd32(dy, y, ref)[1], r, m)
    assert not _meets("C_BOX_BWD", _box_bwd32(dy, y, ref, strict=True)[1], r, m)


# ---- query depth ----------------------------------------------------------------------------------------------------------------
def _hd_inputs():
    g = torch.Generator().manual_seed(1)
    B, N, H, W = 2, 64, 6, 9
    coord = torch.rand(B, N, 6, generator=g) * 0.1
    coord[..., :2] = torch.rand(B, N, 2, generator=g)
    cell = 1.0 / (W - 1)
    coord[:, :8, 0] = torch.tensor([1 + 0.5 * cell, 1 + 0.25 * cell, 1.0, 0.0, -0.5 * cell, 0.5, 1 + 0.9 * cell, 0.3])
    ih = torch.tensor([375.0, 368.0])
    hn = _f32(1.0) / ih
    coord[:, 8, 4], coord[:, 8, 5] = hn, 0.0
    coord[:, 9, 4], coord[:, 9, 5] = torch.nextafter(hn, _f32(0)), 0.0
    coord[:, 10, 4:] = 1e-4
    size3d = torch.randn(B, N, 3, generator=g) + 1.5
    reg = torch.randn(B, N, 2, generator=g)
    wd = torch.rand(B, H, W, generator=g) * 60
    calibs = torch.zeros(B, 3, 4)
    calibs[:, 0, 0] = torch.tensor([700.0, 713.5])
    sizes = torch.stack((torch.full((B,), 1242.0), ih), -1)
    dout = torch.randn(B, N, 2, generator=g)
    return coord, size3d, reg, wd, calibs, sizes, dout


def _taps32(coord, H, W, loose=False):
    u = em.head_xy32(coord[..., :2])
    x, y = u[..., 0] * float(W - 1), u[..., 1] * float(H - 1)
    xf, yf = torch.floor(x), torch.floor(y)
    x0, y0, lx, ly = xf.long(), yf.long(), x - xf, y - yf
    xmax = W if loose else W - 1
    out = []
    for dy_, dx_, w in ((0, 0, (1 - ly) * (1 - lx)), (0, 1, (1 - ly) * lx), (1, 0, ly * (1 - lx)), (1, 1, ly * lx)):
        xx, yy = x0 + dx_, y0 + dy_
        ok = (xx >= 0) & (xx <= xmax) & (yy >= 0) & (yy <= H - 1)
        out.append((torch.where(ok, yy * W + xx, torch.full_like(xx, -1)), w))
    return out


def _hd_fwd32(coord, size3d, reg, wd, calibs, sizes, loose=False):
    B, N = coord.shape[:2]
    H, W = wd.shape[1:]
    h = torch.clamp((coord[..., 4] + coord[..., 5]) * sizes[:, 1:2], min=1)
    geo = size3d[..., 0] / h * calibs[:, 0, 0:1]
    dr = 1 / (torch.sigmoid(reg[..., 0]) + _f32(1e-6)) - 1
    d = torch.cat((wd.reshape(B, -1), torch.zeros(B, 1)), 1)           # a read past the map's end sees 0
    dm = torch.zeros(B, N)
    for idx, w in _taps32(coord, H, W, loose):
        dm = dm + torch.gather(d, 1, torch.where(idx >= 0, idx, torch.full_like(idx, H * W))) * w
    return (dr + geo + dm) / 3


def _hd_bwd32(dout, coord, size3d, calibs, sizes, H, W, clamp_grad=True, third=True):
    B = coord.shape[0]
    g = dout[..., 0] / 3 if third else dout[..., 0]
    ih, fu = sizes[:, 1:2], calibs[:, 0, 0:1]
    hraw = (coord[..., 4] + coord[..., 5]) * ih
    h = torch.clamp(hraw, min=1)
    dh = -g * size3d[..., 0] * fu / (h * h)
    dhn = torch.where(hraw >= 1, dh * ih, torch.zeros_like(dh)) if clamp_grad else dh * ih
    dmap = torch.zeros(B, H * W + 1)
    for idx, w in _taps32(coord, H, W):
        dmap.scatter_add_(1, torch.where(idx >= 0, idx, torch.full_like(idx, H * W)), w * g)
    return dhn, dmap[:, :-1].reshape(B, H, W)


def test_head_depth_mutants():
    coord, size3d, reg, wd, calibs, sizes, dout = _hd_inputs()
    H, W = wd.shape[1:]
    ref, mag = em.head_depth_fwd(coord, size3d, reg, wd, calibs, sizes)
    assert _meets("C_HD_FWD", _hd_fwd32(coord, size3d, reg, wd, calibs, sizes), ref, mag)
    assert not _meets("C_HD_FWD", _hd_fwd32(coord, size3d, reg, wd, calibs, sizes, loose=True), ref, mag)   # x0 + 1 <= W
    r = em.head_depth_bwd(dout, coord, size3d, reg, calibs, sizes, H, W)
    dhn, dmap = _hd_bwd32(dout, coord, size3d, calibs, sizes, H, W)
    assert _meets("C_HD_BWD", dhn, *r["dhn"]) and _meets("C_HD_MAP", dmap, *r["dmap"])
    assert not _meets("C_HD_BWD", _hd_bwd32(dout, coord, size3d, calibs, sizes, H, W, clamp_grad=False)[0], *r["dhn"])
    assert not _meets("C_HD_MAP", _hd_bwd32(dout, coord, size3d, calibs, sizes, H, W, third=False)[1], *r["dmap"])


# ---- depth predictor tail -------------------------------------------------------------------------------------------------------
def _butterfly(v, op):
    """v (P, 32) per-lane values -> the xor-shuffle reduction every lane ends with (lane 0's copy)."""
    for o in (16, 8, 4, 2, 1):
        v = op(v, v[:, torch.arange(32) ^ o])
    return v[:, 0]


def _wd32(logits, bins, fma=False):
    """The kernels' weighted depth: lane l holds bins l, l + 32, l + 64; per-lane sums in that order, then the butterfly."""
    P, nb = logits.shape
    v = torch.full((P, 96), -float("inf"))
    v[:, :nb] = logits
    b = torch.zeros(96)
    b[:nb] = bins
    v, b = v.view(P, 3, 32), b.view(3, 32)
    mx = _butterfly(v.max(1).values, torch.maximum)
    e = torch.exp(v - mx[:, None, None])
    se = torch.zeros(P, 32)
    sw = torch.zeros(P, 32)
    for k in range(3):
        se = se + e[:, k]
        sw = _fma32(e[:, k], b[k].expand(P, 32), sw) if fma else sw + e[:, k] * b[k]
    se, sw = _butterfly(se, torch.add), _butterfly(sw, torch.add)
    return sw / se, e.reshape(P, 96)[:, :nb], se


def _cell32(wd, E, dmax, clamp_ci=True):
    x = wd.clamp(min=0, max=float(_f32(dmax)))
    f = torch.floor(x)
    fi = f.long()
    ci = (fi + 1).clamp(max=E - 1) if clamp_ci else fi + 1
    return fi, ci, x - f


def _tail_bwd32(logits, bins, emb_pad, E, d_ip, d_ext, dmax, fma=False, clamp_ci=True, mask=True):
    """emb_pad: (E + 1, C), the row past the end standing in for what an unclamped ceil index would read."""
    wd, e, se = _wd32(logits, bins, fma)
    fi, ci, d = _cell32(wd, E, dmax, clamp_ci)
    e0, e1 = emb_pad[fi], emb_pad[ci]
    dd = (d_ip * (e1 - e0)).sum(-1)
    inside = (wd >= 0) & (wd <= float(_f32(dmax)))
    dwd = torch.where(inside, dd, torch.zeros_like(dd)) if mask else dd
    dwd = dwd + d_ext
    dlog = e / se[:, None] * (bins[None] - wd[:, None]) * dwd[:, None]
    demb = torch.zeros_like(emb_pad)
    demb.index_add_(0, fi, d_ip * (1 - d)[:, None])
    demb.index_add_(0, ci, d_ip * d[:, None])
    return dlog, demb[:E]


def _model_bins(nb, dmax):
    idx = torch.linspace(0, nb - 2, nb - 1)
    bs = 2 * (dmax - 1e-3) / ((nb - 1) * nb)
    return torch.cat(((idx + 0.5).pow(2) * bs / 2 - bs / 8 + 1e-3, torch.tensor([dmax])))


def _tail_case(logits, bins, E, C, dmax, seed):
    g = torch.Generator().manual_seed(seed)
    P = logits.shape[0]
    emb = torch.randn(E + 1, C, generator=g)
    d_ip, d_ext = torch.randn(P, C, generator=g), torch.randn(P, generator=g)
    wd, _, _ = _wd32(logits, bins)
    fi, ci, d = _cell32(wd, E, dmax)
    ip = emb[fi] * (1 - d)[:, None] + emb[ci] * d[:, None]
    (w64, wm), (i64, im) = em.depth_tail_fwd(logits, bins, emb[:E], wd, dmax)
    assert _meets("C_DT_WD", wd, w64, wm) and _meets("C_DT_IP", ip, i64, im)
    ref = em.depth_tail_bwd(logits, bins, emb[:E], d_ip, d_ext, wd, dmax)

    def meets(**mut):
        dl, de = _tail_bwd32(logits, bins, emb, E, d_ip, d_ext, dmax, **mut)
        return _meets("C_DT_DLOGITS", dl, *ref[0]) and _meets("C_DT_DEMB", de, *ref[1])

    return meets


def test_depth_tail_shipped_and_mutants():
    E, C, dmax, nb = 61, 8, 60.0, 81
    bins = _model_bins(nb, dmax)
    meets = _tail_case(em.edge_logits(bins, dmax), bins, E, C, dmax, 0)
    assert meets()
    assert not meets(fma=True)                 # an FMA-contracted softmax sum in the backward moves the cell near integers
    assert not meets(clamp_ci=False)           # ceil index past E - 1 at wd == dmax
    assert meets(mask=False)                   # the model's bins keep wd in [0, dmax]: the mask never acts


def test_depth_tail_own_bins_exercise_the_clamp_mask():
    E, C, nb = 61, 8, 96
    dmax = E - 1.5
    bins = torch.linspace(-5.0, dmax + 5.0, nb)[torch.randperm(nb, generator=torch.Generator().manual_seed(nb))]
    logits = torch.randn(512, nb, generator=torch.Generator().manual_seed(3)) * 8
    wd = _wd32(logits, bins)[0]
    assert bool((wd < 0).any()) and bool((wd > dmax).any())
    meets = _tail_case(logits, bins, E, C, dmax, 1)
    assert meets()
    assert not meets(mask=False)


# ---- column sums ------------------------------------------------------------------------------------------------------------------
def _colsum32(x, prior, reproducible, use_prior=True):
    """colsum_kernel: gy slabs of `rows` rows; in a slab, lane ty adds rows r0 + ty, r0 + ty + 8, ... in order; the 8 lane sums
    are added in order and the slab's sum added to the output (slab order: atomics; here in order)."""
    M, N = x.shape
    gx = (N + 31) // 32
    gy = (M + 511) // 512
    gy = min(gy, (NUM_SMS * 8 + gx - 1) // gx)
    if gy < 1 or reproducible:
        gy = 1
    rows = (M + gy - 1) // gy
    out = prior.copy() if use_prior else np.zeros(N, np.float32)
    for s in range(gy):
        r0, r1 = s * rows, min(M, s * rows + rows)
        if r0 >= r1:
            continue
        slab = x[r0:r1]
        pad = (-slab.shape[0]) % 8
        slab = np.concatenate((slab, np.zeros((pad, N), np.float32))).reshape(-1, 8, N)
        acc = np.zeros((8, N), np.float32)
        for t in range(slab.shape[0]):
            acc += slab[t]
        part = np.float32(0) + np.zeros(N, np.float32)
        for k in range(8):
            part += acc[k]
        out = out + part
    return out


def test_colsum_chains_both_modes():
    rng = np.random.default_rng(0)
    for M, N in ((81600, 64), (513, 33), (7, 1)):
        x = (rng.standard_normal((M, N)) + 1.0).astype(np.float32)
        prior = (rng.standard_normal(N) * 100).astype(np.float32)
        ref, mag = em.colsum(torch.from_numpy(x), torch.from_numpy(prior))
        for rep in (False, True):
            assert _meets("C_COLSUM", torch.from_numpy(_colsum32(x, prior, rep)), ref, mag), (M, N, rep)
            assert not _meets("C_COLSUM", torch.from_numpy(_colsum32(x, prior, rep, use_prior=False)), ref, mag)


# ---- resize -------------------------------------------------------------------------------------------------------------------------
def _src_np(Hi, Ho, fma=True, clamp=True):
    sc = np.float32(Hi) / np.float32(Ho)
    o = np.arange(Ho, dtype=np.float32) + np.float32(0.5)
    s = (o.astype(np.float64) * np.float64(sc) - 0.5).astype(np.float32) if fma else o * sc - np.float32(0.5)
    if clamp:
        s = np.maximum(s, np.float32(0))
    i0 = s.astype(np.int64)
    return sc, i0, i0 + (i0 < Hi - 1), s


def _window_np(h, sc, Ho, upper=1.5):
    hf = h.astype(np.float32)
    lo = np.floor((hf - np.float32(0.5)) / sc - np.float32(0.5)).astype(np.int64) - 2
    lo = np.where(h <= 1, 0, np.maximum(lo, 0))
    hi = np.minimum(np.ceil((hf + np.float32(upper)) / sc - np.float32(0.5)).astype(np.int64) + 2, Ho - 1)
    return lo, hi


def _covered(Hi, Ho, fma=True, upper=1.5):
    """Every output whose source window touches input row h lies in h's window [ylo, yhi]."""
    sc, i0, i1, _ = _src_np(Hi, Ho, fma)
    o = np.arange(Ho)
    for h in (i0, i1):
        lo, hi = _window_np(h, sc, Ho, upper)
        if not ((lo <= o) & (o <= hi)).all():
            return False
    return True


def test_resize_window_covers_every_source_exhaustive():
    for fma in (True, False):
        misses = [(Hi, Ho) for Hi in range(1, 201) for Ho in range(1, 201) if not _covered(Hi, Ho, fma)]
        assert misses == [], misses[:10]
    assert not all(_covered(Hi, Ho, upper=0.5) for Hi in range(1, 49) for Ho in range(1, 49))


def test_resize_src_matches_the_emulation():
    for Hi, Ho in ((12, 24), (6, 12), (7, 3), (48, 1), (1, 48), (37, 41)):
        i0, i1, l0, l1 = em.resize_src(Hi, Ho)
        _, j0, j1, s = _src_np(Hi, Ho)
        assert i0.tolist() == j0.tolist() and i1.tolist() == j1.tolist()
        assert torch.equal(l1, torch.from_numpy(s.astype(np.float64) - j0))


def _resize_1d32(x, Ho, clamp=True):
    """Forward along one axis in fp32: x (Hi,) -> (Ho,)."""
    Hi = x.numel()
    _, i0, i1, s = _src_np(Hi, Ho, clamp=clamp)
    l1 = torch.from_numpy(s - i0.astype(np.float32))
    return (1 - l1) * x[torch.from_numpy(i0)] + l1 * x[torch.from_numpy(i1)]


def _resize_bwd_1d32(dy, Hi, upper=1.5):
    """The gather backward along one axis in fp32: dy (Ho,) -> (Hi,), walking each row's window in order."""
    Ho = dy.numel()
    sc, i0, i1, s = _src_np(Hi, Ho)
    l1 = s - i0.astype(np.float32)
    l0 = np.float32(1) - l1
    d = dy.numpy()
    out = np.zeros(Hi, np.float32)
    lo, hi = _window_np(np.arange(Hi), sc, Ho, upper)
    for h in range(Hi):
        acc = np.float32(0)
        for o in range(lo[h], hi[h] + 1):
            if i0[o] == h:
                acc += l0[o] * d[o]
            if i1[o] == h:
                acc += l1[o] * d[o]
        out[h] = acc
    return torch.from_numpy(out)


def test_resize_shipped_and_mutants():
    g = torch.Generator().manual_seed(2)
    fwd_bad = bwd_bad = False
    for Hi, Ho in ((4, 48), (3, 40), (12, 24), (6, 12), (40, 7), (5, 33)):
        x, dy = torch.randn(Hi, generator=g), torch.randn(Ho, generator=g)
        ref, mag = em.resize_fwd(x.view(1, Hi, 1, 1), Ho, 1)
        assert _meets("C_RESIZE_FWD", _resize_1d32(x, Ho).view(1, Ho, 1, 1), ref, mag)
        fwd_bad |= not _meets("C_RESIZE_FWD", _resize_1d32(x, Ho, clamp=False).view(1, Ho, 1, 1), ref, mag)
        ref, mag = em.resize_bwd(dy.view(1, Ho, 1, 1), Hi, 1)
        assert _meets("C_RESIZE_BWD", _resize_bwd_1d32(dy, Hi).view(1, Hi, 1, 1), ref, mag)
        bwd_bad |= not _meets("C_RESIZE_BWD", _resize_bwd_1d32(dy, Hi, upper=0.5).view(1, Hi, 1, 1), ref, mag)
    assert fwd_bad and bwd_bad


# ---- exact operations --------------------------------------------------------------------------------------------------------------
def test_round_tf32_emulation():
    def i32(b):
        return b - (1 << 32) if b >= 1 << 31 else b
    pairs = [(0x3F800FFF, 0x3F800000), (0x3F801000, 0x3F802000), (0x3F801001, 0x3F802000), (0x3FFFF000, 0x40000000),
             (0x00001000, 0x00002000), (0x7F7FF000, 0x7F800000), (0xBF801000, 0xBF802000), (0xFF7FFFFF, 0xFF800000)]
    bits = torch.tensor([i32(a) for a, _ in pairs], dtype=torch.int32)
    assert em.round_tf32(bits.view(F32)).view(torch.int32).tolist() == [i32(b) for _, b in pairs]
