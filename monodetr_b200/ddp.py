"""Data-parallel gradient exchange: ONE NCCL all-reduce per step over a flat fp32 bucket (SURVEY.md 8e).

Every gradient-receiving parameter's `.grad` is a view into one contiguous buffer, so backward accumulates
straight into the bucket and the step ends with a single `all_reduce(bucket) / world_size` over NVLink.  The 15
tensors that never receive a gradient (sa_v_proj, query_scale, ref_point_head, label_enc -- SURVEY.md appendix C.2)
are left out of the bucket (their .grad stays None, exactly as in the reference).  With use_dab, query_scale and
ref_point_head are on the path and in the bucket; the never-called query_scale_bbox is left out instead.
"""
import torch
import torch.distributed as dist

_NEVER_USED = ("sa_v_proj", "decoder.query_scale", "decoder.ref_point_head", "label_enc")
_NEVER_USED_DAB = ("sa_v_proj", "decoder.query_scale_bbox", "label_enc")


class FlatGradBucket:
    """Two modes.  `views=True`: every .grad IS a view of the flat buffer (backward accumulates in place; one
    `zero()` per step; costs one small add kernel per parameter in AccumulateGrad).  `views=False` (default): backward
    produces ordinary gradients and `all_reduce()` first packs them with ONE multi-tensor copy, reduces the flat buffer
    and leaves `.grad` pointing at the reduced views -- ~4 launches instead of 313.

    CUDA-graph mode (`freeze_sources()` right after capturing fwd+bwd, views=False): every replay rewrites the captured
    gradient tensors (`static_grads`); `all_reduce()` packs from THOSE and, like the eager mode, leaves `.grad` pointing
    at the reduced views, so an optimizer stepping on `p.grad` always sees the rank-mean gradients.  The captured
    tensors are remembered separately, so re-pointing `.grad` never changes what the next replay's pack reads."""

    ALIGN = 32

    def __init__(self, model, views=False):
        never = _NEVER_USED_DAB if getattr(model, "use_dab", False) else _NEVER_USED
        named = [(n, p) for n, p in model.named_parameters() if p.requires_grad and not any(s in n for s in never)]
        # Bucket order = weight-decay tensors first, then the tensors with 'bias' in their name (the reference's optimizer
        # grouping, lib/helpers/optimizer_helper.py:9-16): the fused AdamW (monodetr_b200.optim) then needs one boundary
        # index (`n_decay`, in elements) instead of a per-tensor table.
        named = [(n, p) for n, p in named if "bias" not in n] + [(n, p) for n, p in named if "bias" in n]
        self.names = [n for n, _ in named]
        self.params = [p for _, p in named]
        # Every tensor starts on a 128-byte boundary of the flat buffer (ALIGN elements): the fused AdamW turns the parameters
        # themselves into views at the same offsets, and the kernels read parameters with 16-byte vector loads and TMA.  The
        # padding elements stay zero in every flat buffer (zero gradient -> zero moments -> zero update).
        self.offsets, off = [], 0
        for _, p in named:
            self.offsets.append(off)
            off += -(-p.numel() // self.ALIGN) * self.ALIGN
        n_bias = sum(1 for n, _ in named if "bias" in n)
        self.n_decay = self.offsets[len(named) - n_bias] if n_bias else off      # elements [0, n_decay) get weight decay
        self.param_numel = sum(p.numel() for p in self.params)
        dev = self.params[0].device
        self.flat = torch.zeros(off, dtype=torch.float32, device=dev)
        self.views = [self.flat[o:o + p.numel()].view_as(p) for o, p in zip(self.offsets, self.params)]
        self.numel = off                             # length of the flat buffers (incl. alignment padding)
        self.use_views = views
        self.static_grads = None     # CUDA-graph mode: the gradient tensors the captured backward writes every replay
        if views:
            for p, v in zip(self.params, self.views):
                p.grad = v

    def zero(self):
        if self.use_views:
            self.flat.zero_()
        else:
            for p in self.params:
                p.grad = None

    def freeze_sources(self):
        """Call once right after capturing fwd+bwd in a CUDA graph: replays rewrite these very tensors."""
        if not self.use_views:
            flat_lo, flat_hi = self.flat.data_ptr(), self.flat.data_ptr() + self.flat.numel() * 4
            for p in self.params:
                if p.grad is not None and flat_lo <= p.grad.data_ptr() < flat_hi:
                    raise RuntimeError("freeze_sources(): .grad already aliases the flat bucket (an eager all_reduce ran "
                                       "before the capture); call bucket.zero() and capture again")
            self.static_grads = [p.grad if p.grad is not None else torch.zeros_like(v) for p, v in zip(self.params, self.views)]

    def _distributed(self):
        return dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1

    def all_reduce(self):
        if not self._distributed():
            return
        if not self.use_views:
            grads = self.static_grads or [p.grad if p.grad is not None else torch.zeros_like(v) for p, v in zip(self.params, self.views)]
            torch._foreach_copy_(self.views, grads)
        dist.all_reduce(self.flat, op=dist.ReduceOp.SUM)
        self.flat.div_(dist.get_world_size())
        if not self.use_views:
            for p, v in zip(self.params, self.views):
                if p.grad is not v:
                    p.grad = v                               # the optimizer sees the reduced gradients (graph mode too)


def rank_world():
    """(rank, world size) of the default process group; (0, 1) without torch.distributed."""
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def broadcast_parameters(model, src=0):
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        for t in list(model.parameters()) + list(model.buffers()):
            dist.broadcast(t.data, src)
