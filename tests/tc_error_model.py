"""Error model of the tensor-core GEMM family (csrc/conv_gemm.cu) and of the attention core (csrc/attention.cu), shared by
the GPU tests that hold the kernels to it and by the CPU test that checks the bound is sharp.

GEMM family.  A kernel of precision mode `mode` splits every operand x the documented way (`split`) and sums a fixed set of
products of the parts (`target`, computed in float64).  What is left between the kernel and that target is fp32
accumulation only, so per output element

    |y - T| <= C[mode] * S + EPI * (|T| + |bias| + |residual|),     S = sum_k |a_k| |b_k|   (float64),

where the second term is the epilogue's rounding of the bias and residual additions.  Elements with S == 0 (padding,
a dgrad parity class no tap reaches) must come out as the epilogue of an exact zero.

Attention.  The forward (3xTF32 scores and P.V) is held per element to C_ATT_FWD * sum_j p_ij |v_jd|; the backward
(single-pass TF32 gradient contractions, round-to-nearest operands) to C_ATT_BWD times the float64 magnitudes of the same
contractions.

The constants are twice the worst ratio measured on an H100 over every element of the GPU tests' cases.  A kernel that
loses one compensation product in one k-block exceeds them: tests/test_error_model_host_logic.py checks both directions on
a simulated kernel.
"""
import torch

# float32 unit roundoff
U32 = 2.0 ** -24
# epilogue: two fp32 additions (bias, then residual) after the accumulator
EPI = 4 * U32

# |y - T| / S: twice the worst ratio measured on an H100 80GB HBM3 (700 W) over every element of
# tests/test_tc_error_model_gpu.py.  Worst measured: bf16x3 6.9e-6, tf32x3 1.4e-5, tf32 4.6e-6, each in the reproducible
# (unsplit) weight gradient over 81600 rows.  The error grows with the length of one accumulation chain: 2e-7..3e-7 for
# the split neck conv (32 k-blocks per slice), 2.4e-6..7.8e-6 for the same conv unsplit (576 k-blocks).
C = {"bf16x3": 1.4e-5, "tf32x3": 2.8e-5, "tf32": 9.2e-6}
# attention: forward per element relative to sum_j p_ij |v_jd| (worst measured 8.6e-6, peaked logits, Lk = 1920);
# backward relative to the fp64 magnitude contractions (worst measured 9.4e-4, dV at Lq = 1, Lk = 1920).  Twice those.
C_ATT_FWD = 1.7e-5
C_ATT_BWD = 1.9e-3


def bf16_rn(x):
    return x.to(torch.bfloat16).to(x.dtype)


def trunc_tf32(x):
    """Clear the 13 low mantissa bits (what the kernels' trunc_tf32 and the tensor core's TF32 operand read do)."""
    return (x.contiguous().view(torch.int32) & -8192).view(torch.float32)


def rn_tf32(x):
    """cvt.rna.tf32.f32: round to nearest TF32, ties away from zero."""
    return ((x.contiguous().view(torch.int32) + 0x1000) & -8192).view(torch.float32)


def split(x, mode):
    """fp32 operand -> the parts the kernel multiplies: (hi, lo) for the compensated modes, (x_tf32, None) for 'tf32'."""
    x = x.float()
    if mode == "bf16x3":
        hi = bf16_rn(x)
        return hi, bf16_rn(x - hi)
    if mode == "tf32x3":
        hi = trunc_tf32(x)
        return hi, trunc_tf32(x - hi)       # the tensor core reads lo as TF32 too
    if mode == "tf32":
        return trunc_tf32(x), None
    raise ValueError(mode)


def target(f, a, b, mode):
    """T = f(A_hi, B_hi) + f(A_lo, B_hi) + f(A_hi, B_lo) in float64 (f bilinear), or f(A_tf32, B_tf32) for 'tf32'; and
    S = f(|a|, |b|) in float64."""
    ah, al = split(a, mode)
    bh, bl = split(b, mode)
    d = torch.float64
    t = f(ah.to(d), bh.to(d))
    if al is not None:
        t = t + f(al.to(d), bh.to(d)) + f(ah.to(d), bl.to(d))
    s = f(a.to(d).abs(), b.to(d).abs())
    return t, s


def epi_mag(t, bias=None, residual=None):
    """|T| + |bias| + |residual| in float64: what the epilogue's two fp32 additions round."""
    m = t.abs()
    if bias is not None:
        m = m + bias.to(torch.float64).abs()
    if residual is not None:
        m = m + residual.to(torch.float64).abs()
    return m


def gemm_excess(y, t, s, epi=None):
    """Per-element |y - t| minus the epilogue allowance EPI * epi, over S.  Returns (worst ratio over S > 0, mask S > 0).

    y: the kernel's output; t: its float64 target including bias / residual (and ReLU / mask: 1-Lipschitz, or exact);
    epi: epi_mag of the target before ReLU / mask, or None when the epilogue adds nothing."""
    err = (y.to(torch.float64) - t).abs()
    if epi is not None:
        err = err - EPI * epi
    pos = s > 0
    ratio = float((err[pos] / s[pos]).max()) if bool(pos.any()) else 0.0
    return ratio, pos


def assert_gemm(name, y, t, s, mode, epi=None, exact_zero=None):
    """Assert the GEMM bound per element.  exact_zero: what the kernel must give bit for bit where S == 0 (the fp32
    epilogue applied to an exact 0: bias + residual, ReLU, mask), or None to skip that check."""
    ratio, pos = gemm_excess(y, t, s, epi)
    print(f"{name} [{mode}]: worst |y-T|/S = {ratio:.3e} (bound {C[mode]:.1e})")
    assert torch.isfinite(y).all(), name
    assert ratio <= C[mode], f"{name} [{mode}]: |y - T| / S = {ratio:.3e} > {C[mode]:.1e}"
    if exact_zero is not None and not bool(pos.all()):
        z = ~pos
        assert torch.equal(y[z], exact_zero.expand_as(y)[z]), f"{name} [{mode}]: S == 0 elements are not the exact epilogue"
    return ratio


def assert_rel(name, y, ref, mag, c):
    """|y - ref| <= c * mag per element (all float64 except y)."""
    y = y.to(torch.float64)
    assert torch.isfinite(y).all(), name
    err = (y - ref).abs()
    pos = mag > 0
    ratio = float((err[pos] / mag[pos]).max()) if bool(pos.any()) else 0.0
    print(f"{name}: worst |y-ref|/mag = {ratio:.3e} (bound {c:.1e})")
    assert ratio <= c, f"{name}: {ratio:.3e} > {c:.1e}"
    assert bool((err[~pos] == 0).all()), f"{name}: elements with zero magnitude are not exact"
    return ratio
