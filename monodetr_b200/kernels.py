"""Raw host wrappers (no autograd) of the attention / normalisation C ABI.  fp32 CUDA tensors only; no fallback."""
import torch

from . import _lib


# ---- dropout seed ------------------------------------------------------------------------------------------
# Masks are a counter-based hash of (seed, site, element) -- csrc/rng.cuh -- so nothing but the seed is stored.  The seed
# lives in device memory (a captured CUDA graph re-reads it at every replay).  There is one MASTER seed per device,
# initialised from torch.initial_seed() (so torch.manual_seed controls it) and the process rank (so data-parallel ranks draw
# different masks); `begin_forward` advances it and takes a SNAPSHOT that every dropout site of that forward -- and of
# its backward, which gets the snapshot through ctx -- uses.  A second forward before the first backward, or any other
# change of the master seed, therefore cannot desynchronise forward and backward masks.
_master = {}
_current = {}


def _rank():
    import torch.distributed as dist
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def master_seed(device):
    key = str(torch.device(device))
    if key not in _master:
        init = (torch.initial_seed() * 0x9E3779B97F4A7C15 + _rank() * 0xD1B54A32D192ED03 + 0x1234567) & 0x7FFFFFFFFFFFFFFF
        _master[key] = torch.tensor([init], dtype=torch.int64, device=device)
    return _master[key]


def reseed(device, value):
    """Set the master seed explicitly (tests / reproducibility across runs)."""
    master_seed(device).fill_(int(value) & 0x7FFFFFFFFFFFFFFF)
    _current.pop(str(torch.device(device)), None)


def begin_forward(device):
    """Advance the master seed and snapshot it for one forward/backward pair.  MonoDETR.forward calls this in train()
    mode; both operations are device-side (graph-safe).  Returns the snapshot."""
    m = master_seed(device)
    m.add_(0x632BE5AB)
    snap = m.clone()
    _current[str(torch.device(device))] = snap
    return snap


def seed_tensor(device):
    """The seed snapshot the dropout sites of the forward in flight use (the master seed itself before any begin_forward)."""
    snap = _current.get(str(torch.device(device)))
    return snap if snap is not None else master_seed(device)


# ---- attention ------------------------------------------------------------------------------------------
def _heads(E, heads):
    """(H, head width): heads=None means width-32 heads (H = E // 32)."""
    if heads is None:
        return E // 32, 32
    if heads <= 0 or E % heads:
        raise ValueError(f"attention: {heads} heads do not divide the embedding width {E}")
    return heads, E // heads


def attention_forward(q, k, v, key_padding_mask=None, drop_p=0.0, site=0, seed=None, heads=None):
    """q (B, Lq, H*d), k/v (B, Lk, H*d) with H = heads and head width d = E / H (16, 32 or 64; heads=None: d = 32): last
    dim contiguous, token stride arbitrary (views of packed buffers ok)."""
    B, Lq, E = q.shape
    Lk = k.shape[1]
    H, hd = _heads(E, heads)
    for t in (q, k, v):
        assert t.dtype == torch.float32 and t.stride(2) == 1 and t.stride(0) == t.shape[1] * t.stride(1)
    out = torch.empty((B, Lq, E), dtype=torch.float32, device=q.device)
    lse = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device)
    kpm = None
    if key_padding_mask is not None:
        kpm = key_padding_mask.to(torch.uint8).contiguous()
    seed = (seed if seed is not None else seed_tensor(q.device)) if drop_p > 0 else None
    _lib.call("mdb_attention_forward_f32", q, k, v, kpm, out, lse, B, H, Lq, Lk, hd, q.stride(1), k.stride(1), v.stride(1), E,
              float(drop_p), seed, site)
    return out, lse, kpm


def attention_backward(q, k, v, kpm, out, lse, dout, drop_p=0.0, site=0, seed=None, heads=None):
    B, Lq, E = q.shape
    Lk = k.shape[1]
    H, hd = _heads(E, heads)
    dout = dout.contiguous()
    dq = torch.empty((B, Lq, E), dtype=torch.float32, device=q.device)
    dk = torch.empty((B, Lk, E), dtype=torch.float32, device=q.device)
    dv = torch.empty((B, Lk, E), dtype=torch.float32, device=q.device)
    ws = torch.empty((B, H, Lq), dtype=torch.float32, device=q.device)
    seed = (seed if seed is not None else seed_tensor(q.device)) if drop_p > 0 else None
    _lib.call("mdb_attention_backward_f32", q, k, v, kpm, out, lse, dout, ws, dq, dk, dv, B, H, Lq, Lk, hd, q.stride(1),
              k.stride(1), v.stride(1), E, E, E, E, float(drop_p), seed, site, launches=3)
    return dq, dk, dv


# ---- layer norm ----------------------------------------------------------------------------------------
def add_layernorm_forward(x, res, gamma, beta, eps=1e-5, drop_p=0.0, site=0, seed=None):
    C = x.shape[-1]
    M = x.numel() // C
    assert x.is_contiguous() and (res is None or (res.is_contiguous() and res.shape == x.shape))
    y = torch.empty_like(x)
    mean = torch.empty((M,), dtype=torch.float32, device=x.device)
    rstd = torch.empty((M,), dtype=torch.float32, device=x.device)
    seed = (seed if seed is not None else seed_tensor(x.device)) if drop_p > 0 else None
    _lib.call("mdb_add_layernorm_forward_f32", x, res, gamma, beta, y, mean, rstd, M, C, eps, float(drop_p), seed, site)
    return y, mean, rstd


def add_layernorm_backward(dy, x, res, gamma, mean, rstd, drop_p=0.0, site=0, seed=None):
    C = x.shape[-1]
    M = x.numel() // C
    dy = dy.contiguous()
    dx = torch.empty_like(x)
    dres = torch.empty_like(x) if (res is not None and drop_p > 0) else None
    dgamma = torch.empty((C,), dtype=torch.float32, device=x.device)
    dbeta = torch.empty((C,), dtype=torch.float32, device=x.device)
    seed = (seed if seed is not None else seed_tensor(x.device)) if drop_p > 0 else None
    # reproducible mode: a second, fixed-order launch computes dgamma / dbeta
    _lib.call("mdb_add_layernorm_backward_f32", dy, x, res, gamma, mean, rstd, dx, dres, dgamma, dbeta, M, C, float(drop_p), seed,
              site, 0, launches=2 if _lib.deterministic() else 1)
    return dx, (dres if dres is not None else dx), dgamma, dbeta


# ---- group norm (NHWC) -----------------------------------------------------------------------------------
def groupnorm_forward(x, gamma, beta, G=32, eps=1e-5, relu=False):
    """x (B, ..., C) channels-last contiguous."""
    assert x.is_contiguous()
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C)
    y = torch.empty_like(x)
    mean = torch.empty((B, G), dtype=torch.float32, device=x.device)
    rstd = torch.empty((B, G), dtype=torch.float32, device=x.device)
    ws = torch.empty((B, G, 2), dtype=torch.float64, device=x.device)
    _lib.call("mdb_groupnorm_forward_f32", x, gamma, beta, y, mean, rstd, ws, B, HW, C, G, eps, int(relu), launches=2)
    return y, mean, rstd


def groupnorm_backward(dy, x, y, gamma, mean, rstd, G=32, relu=False):
    dy = dy.contiguous()
    B, C = x.shape[0], x.shape[-1]
    HW = x.numel() // (B * C)
    dx = torch.empty_like(x)
    dgamma = torch.empty((C,), dtype=torch.float32, device=x.device)
    dbeta = torch.empty((C,), dtype=torch.float32, device=x.device)
    ws = torch.empty((B, G, 2), dtype=torch.float64, device=x.device)
    _lib.call("mdb_groupnorm_backward_f32", dy, x, y if relu else None, gamma, mean, rstd, dx, dgamma, dbeta, ws, B, HW, C, G,
              int(relu), launches=2)
    return dx, dgamma, dbeta
