"""Optimizer of the training step (SURVEY.md 8f-2): the reference's AdamW (lib/helpers/optimizer_helper.py:30-129) as ONE
fused kernel over flat buffers, and `build_optimizer` with the reference's signature / grouping rule (:7-27).

Layout.  The parameters the step updates are the gradient-receiving tensors of `FlatGradBucket` (monodetr_b200.ddp), in the
bucket's order: weight-decay tensors first, then every tensor with 'bias' in its name (weight_decay 0 -- the reference's
rule, :9-16).  At construction the optimizer moves those parameters INTO one flat fp32 buffer (`p.data` becomes a view of
it; values, names, shapes and state_dict are unchanged), keeps exp_avg / exp_avg_sq as two more flat buffers, and takes the
bucket's flat gradient buffer as `g`.  `step()` is then a single HBM-bound launch (`mdb_adamw_step_f32`, 28 bytes per
parameter) instead of ~10 elementwise kernels per tensor; with `device_step=True` the bias-correction factor is computed
on the device so the whole step can live inside a CUDA graph.

Parameters that never receive a gradient (SURVEY.md appendix C.2: sa_v_proj, query_scale, ref_point_head, label_enc; with
use_dab sa_v_proj, query_scale_bbox, label_enc) are not in the bucket and are left untouched, exactly as the reference's `if p.grad is None: continue` (:95-96) leaves them.
"""
import math

import torch

from . import _lib
from .ddp import FlatGradBucket


class FusedAdamW(torch.optim.Optimizer):
    """Same constructor arguments, `param_groups` keys and update rule as the reference's AdamW; amsgrad is not supported."""

    def __init__(self, model, bucket: FlatGradBucket = None, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, device_step=False):
        if lr < 0.0 or eps < 0.0 or not (0.0 <= betas[0] < 1.0) or not (0.0 <= betas[1] < 1.0):
            raise ValueError("invalid AdamW hyper-parameters")
        self.bucket = bucket if bucket is not None else FlatGradBucket(model)
        b = self.bucket
        if not b.params[0].is_cuda:
            raise RuntimeError("FusedAdamW: CUDA parameters required (there is no CPU path)")
        nd = next(i for i, n in enumerate(b.names + ["bias"]) if "bias" in n)          # first no-decay tensor
        groups = [{"params": b.params[nd:], "weight_decay": 0}, {"params": b.params[:nd], "weight_decay": weight_decay}]
        super().__init__([g for g in groups if g["params"]], dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False))
        # parameters -> views of one flat buffer, in bucket order
        self.flat_p = torch.zeros_like(b.flat)
        with torch.no_grad():
            for off, p in zip(b.offsets, b.params):          # 128-byte aligned offsets: vector loads / TMA on parameters keep working
                v = self.flat_p[off:off + p.numel()].view_as(p)
                v.copy_(p)
                p.data = v
        self.exp_avg = torch.zeros_like(b.flat)
        self.exp_avg_sq = torch.zeros_like(b.flat)
        self.step_count = 0
        self.device_step = device_step
        if device_step:
            self._t = torch.zeros((), dtype=torch.float64, device=b.flat.device)
            self._step_size = torch.zeros((), dtype=torch.float32, device=b.flat.device)

    def _grads_in_bucket(self):
        b = self.bucket
        lo, hi = b.flat.data_ptr(), b.flat.data_ptr() + b.flat.numel() * 4
        if all(p.grad is not None and lo <= p.grad.data_ptr() < hi for p in b.params):
            return
        src = b.static_grads or [p.grad if p.grad is not None else torch.zeros_like(v) for p, v in zip(b.params, b.views)]
        torch._foreach_copy_(b.views, src)            # single-GPU use without bucket.all_reduce(): pack the gradients once

    @torch.no_grad()
    def step(self, closure=None):
        loss = closure() if closure is not None else None
        b = self.bucket
        self._grads_in_bucket()
        g0 = self.param_groups[-1]                    # lr / betas / eps are kept equal across the two groups (as the reference builds them)
        lr, (beta1, beta2), eps = g0["lr"], g0["betas"], g0["eps"]
        wd = max(g["weight_decay"] for g in self.param_groups)
        self.step_count += 1
        step_dev = None
        if self.device_step:                          # graph-safe: t and the bias corrections live on the device
            self._t += 1
            self._step_size.copy_(lr * torch.sqrt(1 - beta2 ** self._t) / (1 - beta1 ** self._t))
            step_size, step_dev = 0.0, self._step_size
        else:
            step_size = lr * math.sqrt(1 - beta2 ** self.step_count) / (1 - beta1 ** self.step_count)
        _lib.call("mdb_adamw_step_f32", self.flat_p, b.flat, self.exp_avg, self.exp_avg_sq, b.numel, b.n_decay, beta1, 1 - beta1, beta2,
                  1 - beta2, eps, wd, step_size, step_dev)
        return loss

    def zero_grad(self, set_to_none=True):
        self.bucket.zero()


def build_optimizer(cfg_optimizer, model, bucket=None):
    """lib/helpers/optimizer_helper.py:7-27 with `adamw` served by the fused kernel; sgd / adam fall back to torch.optim with
    the same 'bias'-in-name grouping."""
    if cfg_optimizer["type"] == "adamw":
        return FusedAdamW(model, bucket, lr=cfg_optimizer["lr"], weight_decay=cfg_optimizer["weight_decay"])
    weights = [p for n, p in model.named_parameters() if "bias" not in n]
    biases = [p for n, p in model.named_parameters() if "bias" in n]
    groups = [{"params": biases, "weight_decay": 0}, {"params": weights, "weight_decay": cfg_optimizer["weight_decay"]}]
    if cfg_optimizer["type"] == "sgd":
        return torch.optim.SGD(groups, lr=cfg_optimizer["lr"], momentum=0.9)
    if cfg_optimizer["type"] == "adam":
        return torch.optim.Adam(groups, lr=cfg_optimizer["lr"])
    raise NotImplementedError("%s optimizer is not supported" % cfg_optimizer["type"])
