"""Error model of the LayerNorm and GroupNorm kernels (csrc/norm.cu), shared by the GPU tests that hold the kernels to it
(tests/test_norm_edges_gpu.py) and by the CPU test that checks the bounds are sharp (tests/test_norm_error_model_host_logic.py).

Every reference is float64, computed from the kernel's fp32 inputs: z = x + drop(res) for LayerNorm, the fp32 sum (and
fp32 product drop(res)) the kernel forms, as x + res in PyTorch would; z = x for GroupNorm.  A normalisation group is a row
of LayerNorm or one (image, group) of GroupNorm; mu, rstd and xhat = (z - mu) * rstd are its float64 statistics, and m = mean |z| over the group.  u = 2^-24.
Per element:

    forward   |y - y64|         <= C_FWD  * u * (|gamma| * rstd * (|z| + m) + |beta|)      (fused ReLU on both sides)
              |mu' - mu|        <= C_MU   * u * m                                           (the kernel's `mean` output)
              |rstd'/rstd - 1|  <= C_RSTD * u                                               (the kernel's `rstd` output)
    dx        |dx - dx64|       <= C_BWD  * u * rstd * (|g| + mean|g| + |xhat| mean|g xhat| + a (mean|g xhat| + |xhat| mean|g|))
    dgamma    |dg - dg64|       <= C_PAR  * u * sum |dy| (|xhat| + a)
    dbeta     |db - db64|       <= C_PAR  * u * sum |dy|

with g = dy * gamma (dy masked by the fused ReLU) and a = rstd * m.  The sums run over rows, or over images and pixels; a
prior value the kernel accumulates onto is added to both sides.  `m` rather than |mu| sets the scale of the mean's error:
a float32 sum of values of mixed sign cannot fix the mean better than u * mean|z|, and a float32 mean cannot be nearer than
u * |mu|/2.  `a` carries that error into xhat, where the backward passes meet it.  Bounds on rstd rather than on the
variance cover a constant group: var64 = 0, rstd64 = eps^-1/2, and the kernel must give y == beta there bit for bit.

The constants are twice the worst ratio measured on an H100 over every element of the GPU tests' cases.  A GroupNorm that
sums raw x and x^2 (no shift) exceeds them at a group offset of 30; tests/test_norm_error_model_host_logic.py checks both
directions on an emulation of the kernels' accumulation order.
"""
import torch

from tc_error_model import assert_rel  # noqa: F401  (re-exported: |y - ref| <= c * mag per element)

F64 = torch.float64
U32 = 2.0 ** -24

# Twice the worst ratio measured on an H100 80GB HBM3 (700 W power limit) over every element of tests/test_norm_edges_gpu.py,
# both modes.  The unshifted GroupNorm statistics measure y 40 and rstd 552 at offset 30 (default mode, emulated).
C_FWD = 7.3    # worst 3.62: LayerNorm y, M = 81600, C = 1024, with res
C_MU = 4.8     # worst 2.37: LayerNorm mean, M = 81600, C = 1024, near-constant rows
C_RSTD = 6.6   # worst 3.28: LayerNorm rstd, M = 81600, C = 1024, with res
C_BWD = 7.1    # worst 3.50: LayerNorm dx, M = 81600, C = 256, dropout 0.1
C_PAR = 5.1    # worst 2.54: GroupNorm dbeta, C = 1024, G = 256, HW = 257, reproducible mode


def eps64(eps):
    """The fp32 eps the kernel adds, as a float64."""
    return float(torch.tensor(eps, dtype=torch.float32))


def view4(t, G=None):
    """LayerNorm (M, C) -> (M, 1, 1, C); GroupNorm (B, HW, C) -> (B, HW, G, C/G).  Groups reduce over dims (1, 3)."""
    if G is None:
        return t.reshape(t.shape[0], 1, 1, t.shape[-1])
    return t.reshape(t.shape[0], -1, G, t.shape[-1] // G)


def param4(p, G=None):
    """gamma / beta (C,) -> broadcastable against view4."""
    return p.reshape(1, 1, 1, -1) if G is None else p.reshape(1, 1, G, -1)


def stats(z4, eps):
    """float64 mu, rstd, m = mean|z| per group (keepdim), and xhat."""
    z4 = z4.to(F64)
    mu = z4.mean((1, 3), keepdim=True)
    var = ((z4 - mu) ** 2).mean((1, 3), keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps64(eps))
    m = z4.abs().mean((1, 3), keepdim=True)
    return mu, rstd, m, (z4 - mu) * rstd


def forward(z4, g4, b4, eps):
    """(y64 before ReLU, its magnitude for C_FWD, mu, rstd, m, xhat)."""
    mu, rstd, m, xh = stats(z4, eps)
    g4, b4 = g4.to(F64), b4.to(F64)
    y = xh * g4 + b4
    mag = U32 * (g4.abs() * rstd * (z4.to(F64).abs() + m) + b4.abs())
    return y, mag, mu, rstd, m, xh


def backward(dy4, g4, rstd, m, xh):
    """dy4: dy with the fused ReLU's mask applied.  (dx64, its magnitude for C_BWD, per-element d*xhat and its magnitude
    for C_PAR, per-element |dy|) -- sum the last three over the group's rows / images and pixels for dgamma / dbeta."""
    d = dy4.to(F64)
    gy = d * g4.to(F64)
    m1, m2 = gy.mean((1, 3), keepdim=True), (gy * xh).mean((1, 3), keepdim=True)
    dx = rstd * (gy - m1 - xh * m2)
    a1, a2 = gy.abs().mean((1, 3), keepdim=True), (gy * xh).abs().mean((1, 3), keepdim=True)
    a = rstd * m
    mag_dx = U32 * rstd * (gy.abs() + a1 + xh.abs() * a2 + a * (a2 + xh.abs() * a1))
    return dx, mag_dx, d * xh, U32 * d.abs() * (xh.abs() + a), U32 * d.abs()


def param_sum(t4):
    """Sum a per-element (view4) tensor over rows / images and pixels -> (C,)."""
    return t4.sum((0, 1)).reshape(-1)


def check_stats(name, mean, rstd, mu, rstd64, m):
    """The kernel's per-group mean / rstd outputs against the float64 statistics."""
    r1 = assert_rel(name + " mean", mean.reshape(mu.shape), mu, U32 * m, C_MU)
    r2 = assert_rel(name + " rstd", rstd.reshape(rstd64.shape).to(F64) / rstd64, torch.ones_like(rstd64),
                    torch.full_like(rstd64, U32), C_RSTD)
    return r1, r2
