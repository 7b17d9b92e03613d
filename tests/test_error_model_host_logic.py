"""The error-model bounds of tests/tc_error_model.py are sharp, checked without a GPU: a float32 simulation of the kernels'
arithmetic (documented operand split, exact products within one tensor-core k-step, one fp32 rounding per k-step into the
accumulator, k-blocks in order, fixed-order split-K reduction; online softmax over 64-key tiles for attention) meets the
bounds, and each arithmetic mutant of the kernels -- one compensation product lost, a split-K slice skipped, a lo term of
the attention P.V dropped, an unguarded rescale -- breaks them."""
import math

import pytest
import torch

import tc_error_model as em

F64 = torch.float64


def _round32(x):
    return x.to(torch.float32)


def sim_gemm(a, b, mode, bias=None, mutant=None, kb_per_slice=None):
    """y[M,N] = a[M,K] b[N,K]^T as the wgmma kernel computes it.  Mutants:
    'skip_lo_hi_ks1'  A_lo*B_hi not issued for k-step 1 of every k-block (bf16x3);
    'skip_lo_hi_kb0'  the same in k-block 0 only;
    'skip_hi_lo'      A_hi*B_lo never issued (3xTF32);
    'reduce_from_1'   the split-K reduction starts at slice 1."""
    M, K = a.shape
    nkb = -(-K // 32)
    pad = nkb * 32 - K
    ah, al = em.split(torch.nn.functional.pad(a, (0, pad)), mode)
    bh, bl = em.split(torch.nn.functional.pad(b, (0, pad)), mode)
    step = 16 if mode == "bf16x3" else 8
    kb_per_slice = kb_per_slice or nkb
    parts = []
    for z in range(-(-nkb // kb_per_slice)):
        acc = torch.zeros(M, b.shape[0])
        for kb in range(z * kb_per_slice, min(nkb, (z + 1) * kb_per_slice)):
            for ks in range(32 // step):
                sl = slice(kb * 32 + ks * step, kb * 32 + (ks + 1) * step)
                prods = [(ah, bh)]
                if al is not None:
                    if not ((mutant == "skip_lo_hi_ks1" and ks == 1) or (mutant == "skip_lo_hi_kb0" and ks == 1 and kb == 0)):
                        prods.append((al, bh))
                    if mutant != "skip_hi_lo":
                        prods.append((ah, bl))
                for x, y in prods:
                    acc = _round32(acc.to(F64) + x[:, sl].to(F64) @ y[:, sl].to(F64).t())
        parts.append(acc)
    y = bias.expand(M, -1).clone() if bias is not None else torch.zeros(M, b.shape[0])
    for z, p in enumerate(parts):
        if mutant == "reduce_from_1" and z == 0:
            continue
        y = y + p
    return y


def _gemm_case(M, N, K, seed, bias):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g)
    b = torch.randn(N, K, generator=g) / K ** 0.5
    bb = torch.randn(N, generator=g) if bias else None
    return a, b, bb


def _gemm_ratio(mode, M, N, K, seed, bias=False, **kw):
    a, b, bb = _gemm_case(M, N, K, seed, bias)
    y = sim_gemm(a, b, mode, bb, **kw)
    t, s = em.target(lambda x, w: x @ w.t(), a, b, mode)
    if bb is not None:
        t_full, epi = t + bb.to(F64), em.epi_mag(t, bb)
    else:
        t_full, epi = t, None
    return em.gemm_excess(y, t_full, s, epi)[0]


@pytest.mark.parametrize("mode", ["bf16x3", "tf32x3", "tf32"])
@pytest.mark.parametrize("K", [4, 36, 100, 260])
def test_simulated_gemm_meets_bound(mode, K):
    for M, N, seed in ((16, 8, 1), (5, 13, 2)):
        for bias in (False, True):
            r = _gemm_ratio(mode, M, N, K, seed + K, bias)
            assert r <= em.C[mode], (mode, K, M, N, bias, r)


def test_simulated_splitk_meets_bound():
    for mode in ("bf16x3", "tf32x3"):
        r = _gemm_ratio(mode, 8, 8, 32 * 70 + 12, 3, bias=True, kb_per_slice=32)     # 71 k-blocks: slices 32, 32, 7
        assert r <= em.C[mode], (mode, r)


@pytest.mark.parametrize("mutant,mode,kw", [
    ("skip_lo_hi_ks1", "bf16x3", {}),
    ("skip_lo_hi_kb0", "bf16x3", {}),
    ("skip_hi_lo", "tf32x3", {}),
    ("reduce_from_1", "bf16x3", {"kb_per_slice": 32}),
])
def test_gemm_mutants_break_bound(mutant, mode, kw):
    K = 32 * 70 + 12 if mutant == "reduce_from_1" else 256
    r = _gemm_ratio(mode, 16, 8, K, 4, bias=True, mutant=mutant, **kw)
    assert r > em.C[mode], (mutant, r)


# ---- attention forward -----------------------------------------------------------------------------------------------------
def sim_attention(q, k, v, dead=None, mutant=None):
    """One head, q (Lq, 32), k / v (Lk, 32): scores accurate to fp32 (3xTF32), online softmax over 64-key tiles with
    fp32 exp, P.V as 3xTF32 with round-to-nearest splits, one fp32 rounding per 8-key step.  Mutants:
    'drop_lo_last_u'    the P_lo * V_hi product of the last 8-key step of each 32-key half is dropped;
    'unguarded_rescale' c = exp(m_old - m_new) without the -inf guard."""
    Lq, Lk = q.shape[0], k.shape[0]
    s_all = _round32((q.to(F64) @ k.to(F64).t()) / math.sqrt(32))
    if dead is not None:
        s_all = s_all.masked_fill(dead[None, :], float("-inf"))
    m = torch.full((Lq,), float("-inf"))
    l = torch.zeros(Lq)
    acc = torch.zeros(Lq, 32)
    for k0 in range(0, Lk, 64):
        s = torch.full((Lq, 64), float("-inf"))
        n = min(64, Lk - k0)
        s[:, :n] = s_all[:, k0:k0 + n]
        vt = torch.zeros(64, 32)
        vt[:n] = v[k0:k0 + n]
        mn = torch.maximum(m, s.max(1).values)
        if mutant == "unguarded_rescale":
            c = torch.exp(m - mn)
        else:
            c = torch.where(mn == float("-inf"), torch.ones_like(mn), torch.exp(m - mn))
        l = l * c
        acc = acc * c[:, None]
        p = torch.where(mn[:, None] == float("-inf"), torch.zeros_like(s), torch.exp(s - mn[:, None]))
        l = l + p.sum(1)
        m = mn
        ph, pl = em.rn_tf32(p), em.rn_tf32(p - em.rn_tf32(p))
        vh, vl = em.rn_tf32(vt), em.rn_tf32(vt - em.rn_tf32(vt))
        for u8 in range(8):
            sl = slice(8 * u8, 8 * u8 + 8)
            terms = [(ph, vh), (ph, vl)]
            if not (mutant == "drop_lo_last_u" and u8 % 4 == 3):
                terms.append((pl, vh))
            for x, y in terms:
                acc = _round32(acc.to(F64) + x[:, sl].to(F64) @ y[sl].to(F64))
    inv = torch.where(l > 0, 1.0 / l, torch.zeros_like(l))
    return acc * inv[:, None]


def _attn_ref(q, k, v, dead=None):
    s = (q.to(F64) @ k.to(F64).t()) / math.sqrt(32)
    if dead is not None:
        s = s.masked_fill(dead[None, :], float("-inf"))
    p = torch.softmax(s, 1)
    return p @ v.to(F64), p @ v.to(F64).abs()


def _attn_case(Lq, Lk, seed, dominant=None):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(Lq, 32, generator=g)
    k = torch.randn(Lk, 32, generator=g)
    v = torch.randn(Lk, 32, generator=g)
    if dominant is not None:                       # row i's largest logit (~4) at key dominant(i)
        for i in range(Lq):
            k[dominant(i)] = q[i] * (4 * math.sqrt(32) / float(q[i] @ q[i]))
        k = k.clone()
    return q, k, v


def _attn_ratio(q, k, v, dead=None, mutant=None):
    y = sim_attention(q, k, v, dead, mutant)
    if not bool(torch.isfinite(y).all()):
        return math.inf
    ref, mag = _attn_ref(q, k, v, dead)
    return float(((y.to(F64) - ref).abs() / mag).max())


def test_simulated_attention_meets_bound():
    q, k, v = _attn_case(16, 129, 1)
    assert _attn_ratio(q, k, v) <= em.C_ATT_FWD
    dead = torch.zeros(129, dtype=torch.bool)
    dead[:64] = True                               # first key tile fully masked
    assert _attn_ratio(q, k, v, dead) <= em.C_ATT_FWD
    q, k, v = _attn_case(16, 129, 2, dominant=lambda i: 64 + 24 + (i % 8))
    assert _attn_ratio(q, k, v) <= em.C_ATT_FWD


def test_attention_mutants_break_bound():
    # a dominant key (p ~ 0.5, so its lo part is not zero) in the last 8-key step of a 32-key half
    q, k, v = _attn_case(16, 129, 2, dominant=lambda i: 64 + 24 + (i % 8))
    assert _attn_ratio(q, k, v, mutant="drop_lo_last_u") > em.C_ATT_FWD
    dead = torch.zeros(129, dtype=torch.bool)
    dead[:64] = True
    assert _attn_ratio(q, k, v, dead, mutant="unguarded_rescale") == math.inf
